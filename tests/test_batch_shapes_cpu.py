"""
CPU check (no GPU) that the shape matrix of tests/test_gpu_batch_shapes.py reaches every tile edge it is there for.  The tile
sizes are read from the kernel sources: if a kernel is retiled, this fails until the matrix moves with it.

    logits_tc_kernel     kLgBM-row M tiles          a last tile of 1 row and of kLgBM - 1 rows, a partial tile after 7 full ones
    wv_gather_kernel     kBandWins-window groups    a last group of 1 and of kBandWins - 1 windows
    launch_sgemm         32 / 64-row tiles          both variants, with a partial tile on each side of the switch
    multi-step calls                                a last step whose group count differs from the steps before it
    conv_t / layer1_wv   kUnitsPerWin / kFuUnitsPerWin units per window on persistent CTAs: more than one round, last partial
"""
import re

import pytest

import test_gpu_batch_shapes as S
from genomad_b200 import build as B

H100_SMS = 132                               # SMs of an H100 SXM: the persistent kernels' grid


def _const(name, text, env):
    m = re.search(r"constexpr int\s+(?:\w+\s*=\s*[^,;]+,\s*)*" + name + r"\s*=\s*([^,;]+)[,;]", text)
    assert m, f"{name} not found"
    return int(eval(m.group(1), {"__builtins__": {}}, env))


@pytest.fixture(scope="module")
def k():
    src = {p.name: p.read_text() for p in B.CSRC.iterdir() if p.suffix in (".cuh", ".cu")}
    env = {}
    env["kTok"] = _const("kTok", src["common.cuh"], env)
    env["kTileM"] = _const("kTileM", src["conv_t.cuh"], env)
    env["kFuUnit"] = _const("kFuUnit", src["layer1_wv.cuh"], env)
    out = {"kLgBM": _const("kLgBM", src["logits_tc.cuh"], env), "kBandWins": _const("kBandWins", src["wv_gather.cuh"], env),
           "kUnitsPerWin": _const("kUnitsPerWin", src["conv_t.cuh"], env),
           "kFuUnitsPerWin": _const("kFuUnitsPerWin", src["layer1_wv.cuh"], env)}
    body = re.search(r"static int launch_sgemm\(.*?\n}\n", src["api.cu"], re.S)
    assert body, "launch_sgemm not found in api.cu"
    m = re.search(r"if \(M >= (\d+)\) \{.*?sgemm_epi_kernel<(\d+)>.*?\} else \{.*?sgemm_epi_kernel<(\d+)>", body.group(0), re.S)
    assert m, "launch_sgemm's row-tile switch not found"
    out["sgemm_switch"], out["sgemm_big"], out["sgemm_small"] = map(int, m.groups())
    return out


def test_constants_match_the_test_file(k):
    assert (S.TILE, S.GROUP) == (k["kLgBM"], k["kBandWins"])
    assert all(S.head_tile(n, 1) == (k["sgemm_big"] if n >= k["sgemm_switch"] else k["sgemm_small"]) for n in S.FFMA_SHAPES)


def test_last_m_tiles(k):
    t = k["kLgBM"]
    last = {n % t for n in S.TC_SHAPES}
    assert 1 in last and t - 1 in last, last
    assert any(n // t >= 7 and n % t for n in S.TC_SHAPES), "no partial M tile after several full ones"
    last_steps = [n % mb or mb for mb, n in S.MULTI_STEP]
    assert any(m > t and m % t for m in last_steps), f"no multi-step call whose last step ends in a partial second tile: {last_steps}"


def test_last_window_groups(k):
    g = k["kBandWins"]
    last = {n % g for n in S.TC_SHAPES}
    assert 1 in last and g - 1 in last, last
    assert any(n % g == 0 for n in S.TC_SHAPES), "no batch of whole groups"


def test_both_sgemm_variants_with_partial_tiles(k):
    sw, big, small = k["sgemm_switch"], k["sgemm_big"], k["sgemm_small"]
    below, above = [n for n in S.FFMA_SHAPES if n < sw], [n for n in S.FFMA_SHAPES if n >= sw]
    assert any(n % small for n in below), "no partial 32-row tile below the switch"
    assert any(n % big for n in above), "no partial 64-row tile above the switch"
    assert sw in S.FFMA_SHAPES


def test_multistep_last_step_changes_the_group_count(k):
    g = k["kBandWins"]
    for mb, n in S.MULTI_STEP:
        steps = [min(mb, n - o) for o in range(0, n, mb)]
        assert len(steps) >= 2 and -(-steps[-1] // g) != -(-steps[-2] // g), (mb, n, steps)


def test_persistent_kernels_run_a_partial_last_round(k):
    for units in (k["kUnitsPerWin"], k["kFuUnitsPerWin"]):
        assert any(n * units > H100_SMS and n * units % H100_SMS for n in S.TC_SHAPES + S.FFMA_SHAPES), units


def test_samples_straddle_the_tile_edges(k):
    t, g = k["kLgBM"], k["kBandWins"]
    for n in S.TC_SHAPES + S.FFMA_SHAPES + tuple(n % mb or mb for mb, n in S.MULTI_STEP):
        idx = set(S.sample_rows(n))
        edges = [e for e in (t, 2 * t, (n - 1) // t * t) if 0 < e < n]
        for e in edges:
            assert {e - 1, e} <= idx, (n, e, sorted(idx))
        assert {0, n - 1} <= idx and (n < g + 1 or {g - 1, g} <= idx), (n, sorted(idx))
    assert set(S.SINGLES) <= set(range(S.POOL)) and {t - 1, t} <= set(S.SINGLES)
    assert all(mb < S.POOL for mb in S.INVARIANCE_BATCHES if mb != 1024) and 1 in S.INVARIANCE_BATCHES
    assert S.ATTR_CHUNK > t and {t - 1, t} <= set(S.ATTR_SAMPLE) and S.ATTR_CHUNK <= S.ATTR_CTX
    rows = S.IG_WINDOWS * S.IG_STEPS
    assert t < rows <= S.ATTR_CTX and any(w * S.IG_STEPS <= t < (w + 1) * S.IG_STEPS for w in S.IG_CHECK)
