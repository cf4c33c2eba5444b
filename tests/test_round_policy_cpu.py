"""The solver's round policy (pympc_b200/csrc/bmpc_rounds.cuh), through tools/round_plan.py, which compiles the same header: the full
schedule of every kernel family, cold and warm, round by round — which ADMM and which polish run, chunk, caps, working sets, exchange
mode, reset and infeasibility check — until the Schur-form polish takes over or the iteration budget is spent.  Each solve is
enumerated as if every round left instances open."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
from round_plan import plan_round  # noqa: E402


def schedule(family, cold, **opts):
    rows, r, total = [], 0, 0
    while (p := plan_round(family, r, total, cold, **opts)) is not None:
        rows.append(p)
        if p["polish"] == "schur" and family != "team":
            break
        total += p["chunk"]; r += 1
    return rows


def tpi(admm, chunk, ws, capA, capB, reset=0, infeas=0):
    return dict(admm=admm, chunk=chunk, polish="tpi", ws=ws, capA=capA, capB=capB, cap=0, exchange=0, reset=reset, infeas=infeas)


def tpm(admm, chunk, ws, cap, exchange, reset=0, infeas=0):
    return dict(admm=admm, chunk=chunk, polish="tpm", ws=ws, capA=0, capB=0, cap=cap, exchange=exchange, reset=reset, infeas=infeas)


def schur(chunk, cap, reset=0, infeas=0):
    return dict(admm="team", chunk=chunk, polish="schur", ws=None, capA=0, capB=0, cap=cap, exchange=0, reset=reset, infeas=infeas)


def check(chunk, reset=0, infeas=0):
    return dict(admm="team", chunk=chunk, polish="check", ws=None, capA=0, capB=0, cap=0, exchange=0, reset=reset, infeas=infeas)


def tpi_stragglers(capB, chunks=(25, 25, 50, 100), total=0):
    """straggler rounds of the single-input families: team ADMM, k_tpi_pol from v, then the Schur-form polish after 200 iterations"""
    rows = []
    for c in chunks:
        rows.append(tpi("team", c, "from_v", 2, capB, infeas=int(total >= 25))); total += c
    return rows + [schur(200, 30, infeas=1)]


def test_single_input_shared_warm():
    rows = tpi_stragglers(6)
    assert schedule("tpi", cold=False, codes_valid=True) == [tpi("none", 0, "shifted", 1, 7, reset=1)] + rows
    assert schedule("tpi", cold=False, codes_valid=True, shift_warm=0) == [tpi("none", 0, "stored", 1, 7, reset=1)] + rows
    assert schedule("tpi", cold=False, codes_valid=False) == [tpi("none", 0, "from_v", 1, 7, reset=1)] + rows


def test_single_input_shared_cold():
    want = [tpi("tpi", 25, "from_v", 1, 15, reset=1)] + tpi_stragglers(14, chunks=(25, 50, 100), total=25)
    assert schedule("tpi", cold=True) == want
    assert schedule("tpi", cold=True, codes_valid=True) == want
    assert schedule("tpi", cold=True, cold_iters=40) == want                        # cold_iters is a team / multi-input option


def test_single_input_per_instance():
    assert schedule("tpi_view", cold=False, codes_valid=True) == [tpi("none", 0, "shifted", 1, 7, reset=1)] + tpi_stragglers(6)
    assert schedule("tpi_view", cold=True) == [tpi("team", 25, "from_v", 2, 14, reset=1)] + tpi_stragglers(14, chunks=(25, 50, 100), total=25)
    assert schedule("tpi_view", cold=False, codes_valid=True, first_iters=5) == \
        [tpi("team", 5, "from_v", 2, 6, reset=1)] + tpi_stragglers(6, chunks=(20, 25, 50, 100), total=5)


def test_single_input_first_iters():
    assert schedule("tpi", cold=False, codes_valid=True, first_iters=5) == \
        [tpi("tpi", 5, "from_v", 1, 7, reset=1)] + tpi_stragglers(6, chunks=(20, 25, 50, 100), total=5)
    assert schedule("tpi", cold=True, first_iters=5) == \
        [tpi("tpi", 5, "from_v", 1, 15, reset=1)] + tpi_stragglers(14, chunks=(20, 25, 50, 100), total=5)


def test_multi_input_warm():
    assert schedule("tpm", cold=False) == [
        tpm("none", 0, "record", 12, 0, reset=1),
        tpm("team", 100, "from_v", 12, 1),
        tpm("team", 100, "from_v", 12, 1, infeas=1),
        schur(200, 30, infeas=1)]


def test_multi_input_cold():
    assert schedule("tpm", cold=True) == [
        tpm("team", 25, "from_v", 24, 0, reset=1),
        tpm("team", 25, "from_v", 24, 1, infeas=1),
        tpm("team", 50, "from_v", 24, 1, infeas=1),
        tpm("team", 100, "from_v", 24, 1, infeas=1),
        schur(200, 30, infeas=1)]
    assert schedule("tpm", cold=True, cold_iters=40) == [
        tpm("team", 40, "from_v", 24, 0, reset=1),
        tpm("team", 40, "from_v", 24, 1, infeas=1),
        tpm("team", 80, "from_v", 24, 1, infeas=1),
        schur(160, 30, infeas=1)]


def test_multi_input_first_iters():
    # (round 0 runs the ADMM in a warm solve too, and the next chunk follows the 25 / doubling rule, not the first straggler chunk)
    for cold, cap, exchange in ((False, 12, 1), (True, 24, 0)):
        assert schedule("tpm", cold=cold, first_iters=5) == [
            tpm("team", 5, "from_v", cap, exchange, reset=1), tpm("team", 20, "from_v", cap, 1),
            tpm("team", 25, "from_v", cap, 1, infeas=1), tpm("team", 50, "from_v", cap, 1, infeas=1),
            tpm("team", 100, "from_v", cap, 1, infeas=1), schur(200, 30, infeas=1)], cold


def test_multi_input_caps_knob(monkeypatch):
    """BMPC_TPM_CAPS = first-launch cap, straggler cap, first straggler chunk, cold cap (a tuning knob of the multi-input family)"""
    monkeypatch.setenv("BMPC_TPM_CAPS", "8,6,25,16")
    assert schedule("tpm", cold=False)[:3] == [tpm("none", 0, "record", 8, 0, reset=1), tpm("team", 25, "from_v", 6, 1),
                                               tpm("team", 25, "from_v", 6, 1, infeas=1)]
    assert schedule("tpm", cold=True)[0] == tpm("team", 25, "from_v", 16, 0, reset=1)
    assert schedule("team", cold=False)[0] == schur(10, 10, reset=1)


def test_team():
    # warm: 10 iterations, then up to 25 and doubling; 10 Schur steps in rounds 0 and 1, 30 from round 2; the last chunk clamped
    warm = [schur(10, 10, reset=1), schur(15, 10)] + [schur(c, 30, infeas=1) for c in (25, 50, 100, 200, 400, 800, 1600, 800)]
    assert schedule("team", cold=False) == warm
    cold = [schur(50, 10, reset=1), schur(50, 10, infeas=1)] + [schur(c, 30, infeas=1) for c in (100, 200, 400, 800, 1600, 800)]
    assert schedule("team", cold=True) == cold
    assert schedule("team", cold=True, cold_iters=30)[:3] == [schur(30, 10, reset=1), schur(30, 10, infeas=1), schur(60, 30, infeas=1)]
    assert schedule("team", cold=True, first_iters=7)[:3] == [schur(7, 10, reset=1), schur(18, 10), schur(25, 30, infeas=1)]
    assert schedule("team", cold=False, pdas_steps=4)[:3] == [schur(10, 4, reset=1), schur(15, 4), schur(25, 12, infeas=1)]


@pytest.mark.parametrize("family", ["tpi", "tpi_view", "tpm", "team"])
@pytest.mark.parametrize("cold", [False, True])
def test_pure_admm(family, cold):
    """polish = 0: 25 iterations per round (OSQP's check_termination) and k_check_converged, to the end of the budget"""
    want = [check(25, reset=1)] + [check(25, infeas=1)] * 159
    assert schedule(family, cold=cold, codes_valid=True, polish=0) == want
    assert schedule(family, cold=cold, polish=0, first_iters=5, max_iter=60) == [check(25, reset=1), check(25, infeas=1), check(10, infeas=1)]


def test_max_iter_clamps_the_chunk():
    assert schedule("tpi", cold=False, codes_valid=True, max_iter=60) == [
        tpi("none", 0, "shifted", 1, 7, reset=1), tpi("team", 25, "from_v", 2, 6), tpi("team", 25, "from_v", 2, 6, infeas=1),
        tpi("team", 10, "from_v", 2, 6, infeas=1)]
    assert schedule("tpi", cold=True, max_iter=20) == [tpi("tpi", 20, "from_v", 1, 15, reset=1)]
    assert schedule("tpm", cold=False, max_iter=50) == [tpm("none", 0, "record", 12, 0, reset=1), tpm("team", 50, "from_v", 12, 1)]
    assert schedule("team", cold=False, max_iter=5) == [schur(5, 10, reset=1)]
    assert schedule("team", cold=True, max_iter=120) == [schur(50, 10, reset=1), schur(50, 10, infeas=1), schur(20, 30, infeas=1)]
