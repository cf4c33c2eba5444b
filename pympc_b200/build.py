"""In-tree build of libbmpc.so for sm_90a (nvcc cross-compiles without a GPU)."""
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "csrc", "bmpc.cu")
SHAPES = os.path.join(_HERE, "csrc", "tpi_shapes.inc")
import glob
# every header / table the translation unit includes, and this file (NVCC_FLAGS: the target architecture): an edit to any of them
# makes the library and the per-shape builds under _jit/ stale
DEPS = sorted(set([SRC, SHAPES, os.path.abspath(__file__), os.path.join(_HERE, "..", "include", "bmpc.h")] + glob.glob(os.path.join(_HERE, "csrc", "*.cuh")) +
                  glob.glob(os.path.join(_HERE, "csrc", "*.inc"))))
LIB = os.path.join(_HERE, "libbmpc.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def build(force=False, verbose=False):
    stale = force or not os.path.exists(LIB) or any(os.path.getmtime(LIB) < os.path.getmtime(p) for p in DEPS)
    if stale:
        cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [SRC, "-o", LIB]
        subprocess.check_call(cmd)
    return LIB


TPI_DOMAIN = "fast-path shapes need nu == 1, nx <= 13, Np*nx <= 128, Np < 32, 1 <= Nc <= Np"


def tpi_shape_supported(nx, nu, Np, Nc=None):
    """True when the single-input fast path (thread-per-instance ADMM + Riccati polish, csrc/bmpc_tpi.cuh) can hold the shape:
    nu == 1; Np*nx <= 128 and Np < 32 (the register-resident sweeps); nx <= 13 (a stage's working set is one code word of
    2 nx + 6 bits, at most 32).  Every such shape also fits the polish's shared memory with at least one warp per CTA.
    Other shapes run on the team kernels."""
    Nc = Np if Nc is None else Nc
    return nu == 1 and 1 <= nx <= 13 and Np * nx <= 128 and Np < 32 and 1 <= Nc <= Np


def add_shape(nx, nu, Np, Nc=None):
    """Register one more compile-time fast-path shape (tpi_shape_supported, default Nc = Np) and rebuild."""
    Nc = Np if Nc is None else Nc
    if not tpi_shape_supported(nx, nu, Np, Nc):
        raise ValueError(TPI_DOMAIN)
    line = f"BMPC_TPI_SHAPE({nx}, {nu}, {Np}, {Nc})"
    txt = open(SHAPES).read()
    if line not in txt:
        open(SHAPES, "a").write(line + "\n")
    return build(force=True)


def jit_shape(nx, nu, Np, Nc=None, verbose=False):
    """Build (once; cached under pympc_b200/_jit/) a copy of the library whose fast-path table holds exactly the shape
    (nx, 1, Np, Nc) and return its path: lets a controller of ANY single-input shape run on the thread-per-instance kernels
    without editing csrc/tpi_shapes.inc.  Raises on shapes the fast path cannot hold or when nvcc is not available."""
    Nc = Np if Nc is None else Nc
    if not tpi_shape_supported(nx, nu, Np, Nc):
        raise ValueError(TPI_DOMAIN)
    jdir = os.path.join(_HERE, "_jit"); os.makedirs(jdir, exist_ok=True)
    tag = f"{nx}_{nu}_{Np}_{Nc}"
    inc = os.path.join(jdir, f"shape_{tag}.inc"); lib = os.path.join(jdir, f"libbmpc_{tag}.so")
    if not os.path.exists(inc):
        open(inc, "w").write(f"BMPC_TPI_SHAPE({nx}, {nu}, {Np}, {Nc})\n")
    deps = [p for p in DEPS if p != SHAPES]
    if not os.path.exists(lib) or any(os.path.getmtime(lib) < os.path.getmtime(p) for p in deps):
        cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [f'-DBMPC_TPI_SHAPES_FILE="{inc}"', SRC, "-o", lib + ".tmp"]
        subprocess.check_call(cmd)
        os.replace(lib + ".tmp", lib)
    return lib


TPM_DOMAIN = "multi-input fast-path shapes need nu >= 1, 1 <= nx <= 13, 2 nx + 10 nu <= 64, Np <= 64, 1 <= Nc <= Np"


def tpm_shape_supported(nx, nu, Np, Nc=None):
    """True when the multi-input fast path (thread-per-instance Riccati polish over the scalar delta-u chain, csrc/bmpc_tpm.cuh)
    can hold the shape:
      * 2 nx + 10 nu <= 64: a stage's working set is one 64-bit code word (2 soft-row bits per state, 10 bits per channel);
      * nx <= 13 and Np <= 64: the per-thread stack frame of k_tpm_pol stays at a few KB.  The cost-to-go of order nx + nu and the
        nx x nx state map are unrolled into registers, the working sets are three arrays of Np words.  sm_90a builds: at most
        1.5 KB up to nx = 9 and at (2,1,64,64), 2.5-3.8 KB at nx = 10-11, 4-7 KB at nx = 12-13.  From nx = 14 on, ptxas
        falls back to 64 registers and the frame jumps to 18 KB at (14,1,7,7), 35 KB at (18,2,6,6) and 68 KB at (22,2,6,6).
        The driver reserves a frame for every thread the GPU can hold (270 336 on an H100 SXM): 7 KB is 1.9 GB of device
        memory, 68 KB would be 18 GB;
      * 1 <= Nc <= Np.
    Other shapes run on the team kernels.  (A single-input shape inside build.tpi_shape_supported takes the single-input fast path
    instead.)"""
    Nc = Np if Nc is None else Nc
    return nu >= 1 and 1 <= nx <= 13 and 2 * nx + 10 * nu <= 64 and 2 <= Np <= 64 and 1 <= Nc <= Np


def jit_multi_input_shape(nx, nu, Np, Nc=None, Ad=None, Bd=None, verbose=False):
    """Build (once; cached under pympc_b200/_jit/) a copy of the library whose multi-input fast-path table holds the shape
    (nx, nu, Np, Nc) — with the sparsity pattern of (Ad, Bd) fixed at compile time when they are given and small enough for the
    pattern masks (the sweeps then skip the structural zeros) — and return its path.  Per-instance systems (Ad of shape
    (batch, nx, nx), Bd (batch, nx, nu)) compile the union of the instances' patterns.  Raises on shapes outside
    tpm_shape_supported."""
    import numpy as np
    Nc = Np if Nc is None else Nc
    if not tpm_shape_supported(nx, nu, Np, Nc):
        raise ValueError(TPM_DOMAIN)
    line = f"BMPC_TPM_SHAPE({nx}, {nu}, {Np}, {Nc})"; tag = f"m{nx}_{nu}_{Np}_{Nc}"
    if Ad is not None and Bd is not None and nx * nx <= 64 and nx * nu <= 32:
        A = (np.asarray(Ad, float).reshape(-1, nx, nx) != 0.0).any(axis=0); Bm = (np.asarray(Bd, float).reshape(-1, nx, nu) != 0.0).any(axis=0)
        am = sum(1 << i for i, v in enumerate(A.ravel()) if v); bm = sum(1 << i for i, v in enumerate(Bm.ravel()) if v)
        if am != (1 << (nx * nx)) - 1 or bm != (1 << (nx * nu)) - 1:
            line = f"BMPC_TPM_SPARSE_SHAPE({nx}, {nu}, {Np}, {Nc}, 0x{am:x}ull, 0x{bm:x}u)\n" + line      # the dense entry stays behind it
            tag += f"_{am:x}_{bm:x}"
    jdir = os.path.join(_HERE, "_jit"); os.makedirs(jdir, exist_ok=True)
    inc = os.path.join(jdir, f"shape_{tag}.inc"); lib = os.path.join(jdir, f"libbmpc_{tag}.so")
    if not os.path.exists(inc):
        open(inc, "w").write(line + "\n")
    deps = [p for p in DEPS if not p.endswith("tpm_shapes.inc")]
    if not os.path.exists(lib) or any(os.path.getmtime(lib) < os.path.getmtime(p) for p in deps):
        cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [f'-DBMPC_TPM_SHAPES_FILE="{inc}"', SRC, "-o", lib + ".tmp"]
        subprocess.check_call(cmd)
        os.replace(lib + ".tmp", lib)
    return lib


if __name__ == "__main__":
    import sys
    if len(sys.argv) == 3 and sys.argv[1] == "--add-shape":          # nx,nu,Np[,Nc]
        print(add_shape(*[int(v) for v in sys.argv[2].split(",")]))
    else:
        print(build(force=True, verbose=True))
