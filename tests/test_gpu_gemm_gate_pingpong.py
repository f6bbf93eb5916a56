"""Gate/residual launches and second outputs on the GEMM's ping-pong schedule (single-CTA tiles at block_n 64 and 128,
more tiles than CTAs).  A ping-pong gate/residual tile stages its residual and its gate (table and temb slices over the
tile's columns) in shared memory during the main loop, and the second output (the GELU / SiLU pre-activation, or the
gate2 copy of the gated residual) leaves by TMA store through the same tile.  Launches whose tiles can straddle samples
(rows_per_sample neither a multiple of 128 nor >= M), and launches with both gate and gate2, keep the cooperative
schedule; their cases hold that choice to the same results.

Every case runs the single-CTA launch on several grids (max_ctas 1, 2, 3, 5 and the full device) and a repeat of the
first, and compares each bit for bit with the cooperative launch (one tile per CTA: max_ctas at least the tile count),
which issues the same MMAs in the same k-order for every output element.  Every output lives in a sentinel-filled buffer
whose elements outside the output windows must survive."""
import pytest

from _gemm_case import Case, assert_same, load_ops

pytestmark = pytest.mark.gpu

COOP = 1 << 20  # max_ctas at or above the tile count: one tile per CTA, the cooperative schedule
GRIDS = (1, 2, 3, 5, 0)


@pytest.fixture(scope="module")
def ops():
    return load_ops()


def _check(ops, case, epi, bn, grids=GRIDS, **epi_kw):
    """Single-CTA launches on every grid in `grids`, and a repeat of the first, against the cooperative launch."""
    want = case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=COOP, **epi_kw)
    first = case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=grids[0], **epi_kw)
    assert_same(first, want, f"{epi} bn{bn} max_ctas={grids[0]} vs cooperative")
    assert_same(case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=grids[0], **epi_kw), first,
                f"{epi} bn{bn} repeat")
    for mc in grids[1:]:
        assert_same(case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=mc, **epi_kw), want,
                    f"{epi} bn{bn} max_ctas={mc}")


GATES = {"none": {}, "gate": dict(gate=True), "gate2": dict(gate2=True), "both": dict(gate=True, gate2=True)}


# M = 600: 5 row tiles, the last ragged; N = 264: 3 tiles of 128 columns (5 of 64), the last 8 columns wide.
# rows_per_sample 1 and 64: every tile spans many / two samples; 197: sample boundaries inside tiles; 128 and 256: tiles
# inside one sample; 2688 >= M: one sample.
@pytest.mark.parametrize("rps", [1, 64, 128, 197, 256, 2688])
@pytest.mark.parametrize("gates", list(GATES))
@pytest.mark.parametrize("bn", [64, 128])
def test_rows_per_sample(ops, rps, gates, bn):
    case = Case(600, 264, 200, rps=rps, seed=rps + bn)
    _check(ops, case, "GATE_RES", bn, **GATES[gates])


# N % 128 = 8, 64, 120 with a ragged M: the clamped gate copies and the ragged TMA stores of out and out2
@pytest.mark.parametrize("N", [136, 192, 248])
@pytest.mark.parametrize("gates", ["gate", "gate2"])
@pytest.mark.parametrize("bn", [64, 128])
def test_ragged_n(ops, N, gates, bn):
    case = Case(300, N, 136, rps=256, seed=N)
    _check(ops, case, "GATE_RES", bn, **GATES[gates])


@pytest.mark.parametrize("gates", ["none", "gate", "gate2"])
@pytest.mark.parametrize("bn", [64, 128])
def test_batched_gaps(ops, gates, bn):
    """Batched launch: every batch's out and out2 at its own c_boff, the gaps between the slices untouched."""
    case = Case(300, 200, 192, batch=3, rps=128, seed=3)
    _check(ops, case, "GATE_RES", bn, grids=(3, 5, 0), **GATES[gates])


@pytest.mark.parametrize("bn", [64, 128])
def test_in_place_residual_many_tiles(ops, bn):
    """out == res with a gate over at least ten tiles per CTA: each tile's residual is loaded before its out is stored,
    and no other tile touches its rows."""
    case = Case(640, 512, 128, rps=128, seed=5)
    _check(ops, case, "GATE_RES", bn, grids=(2, 1, 0), in_place=True, gate=True)


# K2 = 384: six extension k-blocks after four main ones, more than the 5 ring stages of block_n 128
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("K2", [128, 384])
@pytest.mark.parametrize("gates", ["gate", "gate2"])
def test_lora_extension_groups(ops, b_mn, K2, gates):
    """The K2 extension with per-group A2 slices on gate/residual launches."""
    case = Case(300, 768, 200, b_mn=b_mn, K2=K2, group=256, rps=2688, seed=7)
    _check(ops, case, "GATE_RES", 128, grids=(1, 2, 5, 0), **GATES[gates])


# K = 16 and 64: one k-block, fewer than the ring stages; 1000: sixteen.  M = 600, N = 520: 5 x 5 tiles at block_n 128,
# 5 x 9 at 64, so a CTA has several tiles on every grid but the full one.
@pytest.mark.parametrize("K", [16, 64, 1000])
@pytest.mark.parametrize("epi", ["GELU", "SILU"])
@pytest.mark.parametrize("bn", [64, 128])
def test_activation_out2(ops, K, epi, bn):
    case = Case(600, 520, K, seed=K + bn)
    _check(ops, case, epi, bn, out2=True)
    _check(ops, case, epi, bn, grids=(3, 0))


# The step's five fused launches at M = 2688 (one 49x512x768 sample; D = 2048, LoRA rank 64), as in tools/gemm_bench.py
STEP = {
    "to_out": dict(N=2048, K=2048, K2=64, epi="GATE_RES", kw=dict(gate=True)),
    "to_out2": dict(N=2048, K=2048, K2=64, epi="GATE_RES", kw={}),
    "ffn_down": dict(N=2048, K=8192, K2=0, epi="GATE_RES", kw=dict(gate=True)),
    "to_q2.dX": dict(N=2048, K=2048, K2=64, epi="GATE_RES", b_mn=True, kw=dict(gate2=True)),
    "ffn_up": dict(N=8192, K=2048, K2=0, epi="GELU", kw=dict(out2=True)),
}


@pytest.mark.parametrize("name", list(STEP))
def test_step_shapes(ops, name):
    s = STEP[name]
    b_mn = s.get("b_mn", False)
    case = Case(2688, s["N"], s["K"], b_mn=b_mn, K2=s["K2"], rps=2688, seed=13)
    _check(ops, case, s["epi"], 128, grids=(0,), bias=not b_mn, **s["kw"])
