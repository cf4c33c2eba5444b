"""CPU: the launch configuration of the team / tile kernels (pympc_b200/csrc/bmpc_launch.cuh: bmpc_plan_launch, bmpc_round_launch),
which libbmpc.so and the host emulation share, pinned at an H100's opt-in shared memory (232 448 bytes per block) and 132 SMs for
the shapes of tests/golden/team_shapes.npz and the shared-memory edges; and host twins of the GPU capacity tests: the device core
compiled for the CPU (tests/hostemu) replays the device's polish tiers on golden instances whose optimal working sets are known."""
import numpy as np
import pytest

from conftest import golden
from emu import EmuSystem, plan_launch, launch_tiers, round_launch

SYS_KEYS = ("Ad", "Bd", "Qx", "QxN", "Qu", "QDu", "xmin", "xmax", "umin", "umax", "Dumin", "Dumax", "uref")

# (shape, options) -> team, warps per CTA, main tier, small tier, CTA tier of a warp team, overflow, tile size
PLANS = [
    # A: mc = 188, warp team: 64 per warp, overflow to a CTA tier of all 188 rows (153 KB)
    ((7, 1, 20, 20), {}, dict(team=32, wpb=8, rmax=64, rmax_small=0, fb_rmax=188, overflow=1, tile_T=0)),
    # B: mc = 232, the full tier holds every row; the MIMO shape, where shared memory caps it at 222 of 652
    ((5, 2, 25, 25), {}, dict(team=256, wpb=8, rmax=232, rmax_small=80, fb_rmax=0, overflow=0, tile_T=8)),
    ((8, 4, 40, 40), {}, dict(team=256, wpb=8, rmax=222, rmax_small=80, fb_rmax=0, overflow=0, tile_T=8)),
    # C: mc = 192 is the largest warp-team shape, 193 a CTA team; NU = 64 a warp team, NU = 65 a CTA team
    ((9, 1, 18, 10), {}, dict(team=32, wpb=8, rmax=64, rmax_small=0, fb_rmax=192, overflow=1, tile_T=0)),
    ((8, 1, 19, 16), {}, dict(team=256, wpb=8, rmax=193, rmax_small=80, fb_rmax=0, overflow=0, tile_T=8)),
    ((1, 2, 32, 32), {}, dict(team=32, wpb=8, rmax=64, rmax_small=0, fb_rmax=163, overflow=1, tile_T=0)),
    ((1, 5, 13, 13), {}, dict(team=256, wpb=8, rmax=149, rmax_small=80, fb_rmax=0, overflow=0, tile_T=8)),
    # D: the smallest shapes: every row fits one tier, no overflow
    ((1, 1, 2, 2), {}, dict(team=32, wpb=8, rmax=8, rmax_small=0, fb_rmax=8, overflow=0, tile_T=0)),
    ((2, 3, 5, 1), {}, dict(team=32, wpb=8, rmax=21, rmax_small=0, fb_rmax=21, overflow=0, tile_T=0)),
    # E / G: hard state rows use the same tiers; per-instance systems have no tiles
    ((5, 2, 25, 25), {"n_sys": 333}, dict(team=256, wpb=8, rmax=232, rmax_small=80, fb_rmax=0, overflow=0, tile_T=0)),
    ((7, 1, 20, 20), {"n_sys": 333}, dict(team=32, wpb=8, rmax=64, rmax_small=0, fb_rmax=188, overflow=1, tile_T=0)),
    # F: tiles of 8 stop fitting at (8, 4, 50), of 4 at (8, 4, 83), of 2 at (8, 4, 122); at (8, 4, 261) the full tier is shrunk to
    # 96 rows and there is no small tier; (8, 4, 313) is the last shape that fits at all
    ((8, 4, 49, 49), {}, dict(team=256, wpb=8, rmax=218, rmax_small=80, fb_rmax=0, overflow=0, tile_T=8)),
    ((8, 4, 50, 50), {}, dict(team=256, wpb=8, rmax=218, rmax_small=80, fb_rmax=0, overflow=0, tile_T=4)),
    ((8, 4, 83, 83), {}, dict(team=256, wpb=8, rmax=204, rmax_small=80, fb_rmax=0, overflow=0, tile_T=2)),
    ((8, 4, 122, 122), {}, dict(team=256, wpb=8, rmax=185, rmax_small=80, fb_rmax=0, overflow=0, tile_T=0)),
    ((8, 4, 261, 261), {}, dict(team=256, wpb=8, rmax=96, rmax_small=0, fb_rmax=0, overflow=0, tile_T=0)),
    # options: rmax > 0 caps the main tier (a CTA team then has one tier); team_threads = 256 forces a CTA team without tiles
    ((7, 1, 20, 20), {"team_threads": 256, "rmax": 40}, dict(team=256, wpb=8, rmax=40, rmax_small=0, fb_rmax=0, overflow=0, tile_T=0)),
    ((7, 1, 20, 20), {"rmax": 32}, dict(team=32, wpb=8, rmax=32, rmax_small=0, fb_rmax=188, overflow=1, tile_T=0)),
    ((4, 1, 20, 20), {}, dict(team=32, wpb=8, rmax=64, rmax_small=0, fb_rmax=125, overflow=1, tile_T=0)),
]


@pytest.mark.parametrize("shape,opts,want", PLANS, ids=[f"{'-'.join(map(str, s))}{''.join(f'-{k}{v}' for k, v in o.items())}" for s, o, w in PLANS])
def test_launch_plan_at_h100_shared_memory(shape, opts, want):
    L = plan_launch(*shape, **opts)
    assert L["ok"] == 1
    assert {k: L[k] for k in want} == want
    budget = 232448 - 1024
    for k in ("smem_admm", "smem_polish", "smem_polish_small", "fb_smem_polish"):
        assert L[k] <= budget, k
    if L["fb_rmax"]:                                   # the CTA tier is the largest that fits: one row more does not
        nx, nu, Np, Nc = shape
        mc = (Np + 1) * nx + (2 * Nc + 1) * nu
        assert L["fb_rmax"] == mc or plan_launch(*shape, team_threads=256, rmax=L["fb_rmax"] + 1)["rmax"] == L["fb_rmax"]


def test_first_shape_beyond_shared_memory_is_refused():
    assert plan_launch(8, 4, 313)["ok"] == 1
    assert plan_launch(8, 4, 314)["ok"] == 0
    assert plan_launch(12, 6, 208)["ok"] == 1 and plan_launch(12, 6, 209)["ok"] == 0


def _cta(count, *caps, threads=256):
    return [(0, count, threads, c) for c in caps]


# (shape, options, open instances, straggler round) -> ADMM (kind, tile size, grid, threads), polish tiers (warp, grid, threads,
# capacity), smallest capacity first
ROUNDS = [
    # warp team: a straggler list of at most 4 096 runs one warp per CTA and the CTA tier alone; anything else the warp tier with
    # its overflow to the CTA tier
    ((7, 1, 20, 20), {}, 65536, False, ("warp", 0, 8192, 256), [(1, 8192, 256, 64)] + _cta(65536, 188, threads=128)),
    ((7, 1, 20, 20), {}, 333, False, ("warp", 0, 42, 256), [(1, 42, 256, 64)] + _cta(333, 188, threads=128)),
    ((7, 1, 20, 20), {}, 4096, True, ("lone_warp", 0, 4096, 32), _cta(4096, 188, threads=128)),
    ((7, 1, 20, 20), {}, 4097, True, ("warp", 0, 513, 256), [(1, 513, 256, 64)] + _cta(4097, 188, threads=128)),
    ((7, 1, 20, 20), {"n_sys": 333}, 333, True, ("lone_warp", 0, 333, 32), _cta(333, 188, threads=128)),
    ((1, 1, 2, 2), {}, 5000, False, ("warp", 0, 625, 256), [(1, 625, 256, 8)]),
    # tiles of 8 while the open instances fill the 132 SMs twice over (more than 2 112), then of 4 while they fill them with
    # tiles of 2 (more than 528), then of 2
    ((5, 2, 25, 25), {}, 2113, False, ("tile", 8, 265, 160), _cta(2113, 80, 232)),
    ((5, 2, 25, 25), {}, 2112, True, ("tile", 4, 528, 160), _cta(2112, 80, 232)),
    ((5, 2, 25, 25), {}, 529, True, ("tile", 4, 133, 160), _cta(529, 80, 232)),
    ((5, 2, 25, 25), {}, 528, True, ("tile", 2, 264, 160), _cta(528, 80, 232)),
    ((8, 4, 40, 40), {}, 16384, False, ("tile", 8, 2048, 352), _cta(16384, 80, 222)),
    # shapes where tiles of 8 (or of 4) do not fit: the tile size never exceeds the largest that does
    ((8, 4, 50, 50), {}, 100000, False, ("tile", 4, 25000, 416), _cta(100000, 80, 218)),
    ((8, 4, 50, 50), {}, 528, True, ("tile", 2, 264, 416), _cta(528, 80, 218)),
    ((8, 4, 83, 83), {}, 100000, False, ("tile", 2, 50000, 512), _cta(100000, 80, 204)),
    # CTA team without tiles: per-instance systems, shapes beyond the tiles, a forced team size; rmax > 0 leaves one tier
    ((5, 2, 25, 25), {"n_sys": 333}, 333, False, ("cta", 0, 333, 256), _cta(333, 80, 232)),
    ((8, 4, 261, 261), {}, 5000, True, ("cta", 0, 5000, 256), _cta(5000, 96)),
    ((7, 1, 20, 20), {"team_threads": 256, "rmax": 40}, 300, True, ("cta", 0, 300, 256), _cta(300, 40)),
]


def _bytes(shape, rmax=None):
    """shared memory per instance of k_admm (rmax None) or of k_polish at capacity rmax"""
    nx, nu, Np, Nc = shape
    NX, NU = (Np + 1) * nx, Nc * nu
    mc = NX + NU + (Nc + 1) * nu
    if rmax is None:
        return 8 * (4 * NU + NX + 2 * mc + nu + 8)
    return 8 * (3 * NU + NX + 4 * mc + rmax * (rmax + 1) // 2 + rmax + nu + 2 + (mc + rmax + 3) // 2)


@pytest.mark.parametrize("shape,opts,count,given,admm,tiers", ROUNDS,
                         ids=[f"{'-'.join(map(str, s))}{''.join(f'-{k}{v}' for k, v in o.items())}-{c}{'-list' if g else ''}"
                              for s, o, c, g, *_ in ROUNDS])
def test_round_launch_at_h100(shape, opts, count, given, admm, tiers):
    R = round_launch(*shape, count=count, list_given=given, **opts)
    assert (R["admm"], R["tile_T"], R["admm_grid"], R["admm_threads"]) == admm
    assert [(t["warp"], t["grid"], t["threads"], t["rmax"]) for t in R["tiers"]] == tiers
    # shared memory: the kernels' per-instance carve-up (at the tier's capacity) times the instances per CTA
    wpb = plan_launch(*shape, **opts)["wpb"]
    assert R["admm_smem"] <= 232448 - 1024
    if R["admm"] != "tile":
        assert R["admm_smem"] == (wpb if R["admm"] == "warp" else 1) * _bytes(shape)
    for t in R["tiers"]:
        assert t["smem"] == (wpb if t["warp"] else 1) * _bytes(shape, t["rmax"])
    assert launch_tiers(*shape, count=count, **opts)[int(given)] == tuple(c for *_, c in tiers)


@pytest.mark.parametrize("shape", [(7, 1, 20, 20), (9, 1, 18, 10), (1, 2, 32, 32), (5, 2, 25, 25), (8, 4, 40, 40)])
def test_polish_capacity_does_not_depend_on_batch_size(shape):
    """The largest capacity an instance can reach in a round is the same whatever the number of open instances: a straggler
    round of 333 takes the CTA tier directly, one of 5 000 the warp tier and then, for the working sets it cannot hold, the CTA
    tier in the same round."""
    caps = {c: launch_tiers(*shape, count=c) for c in (1, 333, 4096, 4097, 5000, 65536)}
    top = {max(t) for first, later in caps.values() for t in (first, later)}
    assert len(top) == 1, caps


def _case(name):
    g = golden("team_shapes.npz"); tag = name + "_"
    nx, nu, Np, Nc = (int(v) for v in g[tag + "shape"])
    cfg = {k: g[tag + k] for k in SYS_KEYS}
    cfg.update(Np=Np, Nc=Nc, eps_feas=float(g[tag + "eps_feas"]))
    return cfg, g[tag + "X"], g[tag + "useq"], g[tag + "Xref"], g[tag + "ws"]


def _cold(cfg, x0, xref, **kw):
    E = EmuSystem(cfg)
    U, st, it, ps, res = E.solve(x0, np.zeros(cfg["Bd"].shape[1]), xref, first_iters=0, **kw)
    return U, st


def test_golden_working_sets_reach_every_capacity_edge():
    """team_shapes.npz holds optimal working sets on both sides of every tier the GPU tests exercise"""
    ws = _case("warp_cap")[-1]
    for lo, hi in ((30, 64), (64, 80), (100, 128), (128, 188)):
        assert ((ws > lo) & (ws <= hi)).any(), (lo, hi)
    ws = _case("cta_cap")[-1]
    for lo, hi in ((0, 80), (80, 232)):
        assert ((ws > lo) & (ws <= hi)).any(), (lo, hi)
    ws = _case("cta_hard")[-1]
    assert ws.max() > 50                               # more active rows than inputs (NU = 50): degenerate vertices


@pytest.mark.parametrize("name", ["warp_cap", "cta_cap"])
def test_host_twin_of_the_capacity_tiers(name):
    """Cold solves of the golden first states in host emulation.  The library's tiers (launch_tiers) verify every instance that an
    unlimited capacity verifies, with the same answer, at any batch size.  The fixed caps they replace did not: on a warp team 64
    alone (the straggler rounds of a batch of more than 4 096) and 64 then 128 (a batch of up to 4 096); the CTA team's small tier
    of 80 without its overflow handoff."""
    cfg, GX, GS, GXref, WS = _case(name)
    nx, nu, Np, Nc = cfg["Bd"].shape[0], cfg["Bd"].shape[1], cfg["Np"], cfg["Nc"]
    mc = (Np + 1) * nx + (2 * Nc + 1) * nu
    old = {"warp_cap": {"batch > 4096": ((64,), (64,)), "batch <= 4096": ((64,), (128,))},
           "cta_cap": {"small tier alone": ((80,), (80,))}}[name]
    failed = {k: 0 for k in old}
    for b in range(GX.shape[1]):
        x0, xref = GX[0][b], GXref[b]
        U_inf, st_inf = _cold(cfg, x0, xref, rmax=mc)
        assert st_inf == 1, b
        scale = 1.0 + np.abs(GS[0][b]).max()
        assert np.abs(U_inf - GS[0][b]).max() < 1e-6 * scale, b
        for count in (333, 5000):
            U, st = _cold(cfg, x0, xref, tiers=launch_tiers(nx, nu, Np, Nc, count=count))
            assert st == 1 and np.array_equal(U, U_inf), (b, count, st)
        for k, tiers in old.items():
            U, st = _cold(cfg, x0, xref, tiers=tiers)
            if WS[0][b] > max(max(t) for t in tiers):
                assert st != 1, (b, k)                 # a working set beyond every tier cannot be verified
                failed[k] += 1
            elif st == 1:
                assert np.array_equal(U, U_inf), (b, k)
    assert all(v > 0 for v in failed.values()), failed
