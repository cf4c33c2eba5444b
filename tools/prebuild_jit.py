"""Build ahead of time the on-demand fast-path libraries the GPU tests ask for (pympc_b200/_jit/, git-ignored but shipped to the
GPU box with the snapshot), so that `pytest -m gpu` does not spend its first minutes in nvcc (about a minute per shape, built
in parallel here).  The tests build them themselves when they are missing."""
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pympc_b200 import build  # noqa: E402

if __name__ == "__main__":
    jobs = [(build.jit_shape, (3, 1, 12, 9))]                           # test_any_single_input_shape_gets_the_fast_path
    g = np.load(os.path.join(ROOT, "tests", "golden", "shapes.npz"))     # tests/test_gpu_shapes.py (the supported ones)
    jobs += [(build.jit_shape, (int(nx), 1, int(Np), int(Nc))) for nx, Np, Nc, _ in g["shapes"]
             if build.tpi_shape_supported(int(nx), 1, int(Np), int(Nc))]
    A = np.ones((3, 3)); A[2, 0] = 0.0                                  # test_multi_input_fast_path_built_on_demand_for_a_dense_system
    jobs.append((build.jit_multi_input_shape, (3, 2, 10, 6, A, np.ones((3, 2)))))
    # tests/test_gpu_mimo_shapes.py: every supported shape with its golden system (and so its sparsity pattern), and the
    # non-symmetric pattern's shape dense as well
    g = np.load(os.path.join(ROOT, "tests", "golden", "mimo_shapes.npz"))
    for nx, nu, Np, Nc in (tuple(int(v) for v in s[:4]) for s in g["shapes"]):
        if build.tpm_shape_supported(nx, nu, Np, Nc) and not build.tpi_shape_supported(nx, nu, Np, Nc):
            tag = f"{nx}_{nu}_{Np}_{Nc}_"
            jobs.append((build.jit_multi_input_shape, (nx, nu, Np, Nc, g[tag + "Ad"], g[tag + "Bd"])))
    jobs.append((build.jit_multi_input_shape, tuple(int(v) for v in g["pattern"])))
    with ThreadPoolExecutor(min(len(jobs), os.cpu_count() or 1)) as ex:
        for lib in ex.map(lambda j: j[0](*j[1]), jobs):
            print(lib)
