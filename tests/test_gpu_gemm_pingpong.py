"""The GEMM's ping-pong schedule (single-CTA tiles at block_n 64 and 128, more tiles than CTAs): the two math warpgroups
take alternate tiles of a CTA's work list, so the edges are in how many tiles a CTA gets and how many k-blocks each tile
has.  The gates here have samples of 197 rows, which start inside tiles, so gated launches take the cooperative
schedule and their cases hold that choice to the same results; residual launches without a gate ping-pong.

Every case is bitwise equal to a repeat of itself, to the launch on the full grid and, at block_n 128 with a K-major A,
to the CTA-pair launch on the full grid.  These shapes have fewer pair items (at most 15) than that grid has clusters,
so the pair launch runs cooperative M-pairs, which issue the same MMAs in the same k-order for every element.  Every
output lives in a sentinel-filled buffer whose elements outside the output windows must survive."""
import pytest

from _gemm_case import Case, assert_same, load_ops

pytestmark = pytest.mark.gpu

RPS = 197  # rows per sample of the per-sample gates: sample boundaries fall inside tiles


@pytest.fixture(scope="module")
def ops():
    return load_ops()


def _check(ops, case, epi, bn, max_ctas_list=(0,), pair=True, **epi_kw):
    """Ping-pong launches on every grid in max_ctas_list, and a repeat of the first, against the CTA-pair launch (or,
    at block_n 64, where pairs do not exist, against the first)."""
    first = case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=max_ctas_list[0], **epi_kw)
    want = case.launch(ops, epi, block_n=bn, cta_pair=2, **epi_kw) if pair else first
    assert_same(first, want, f"{epi} bn{bn} max_ctas={max_ctas_list[0]} vs pair")
    assert_same(case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=max_ctas_list[0], **epi_kw), first,
                f"{epi} bn{bn} repeat")
    for mc in max_ctas_list[1:]:
        assert_same(case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=mc, **epi_kw), want,
                    f"{epi} bn{bn} max_ctas={mc}")


# M = 300: 3 tiles of 128 rows (the last ragged); N = 200 / 328: 2 / 3 tiles of 128 columns (4 / 6 of 64).  Over
# max_ctas 1, 2, 3, 5 a CTA gets an odd or even number of tiles, one tile (warpgroup 1 idle) or none beyond its first.
@pytest.mark.parametrize("N", [200, 328])
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
def test_tiles_per_cta(ops, N, bn, a_mn, b_mn):
    case = Case(300, N, 200, a_mn=a_mn, b_mn=b_mn, rps=RPS, seed=N + bn)
    pair = bn == 128 and not a_mn
    _check(ops, case, "GATE_RES", bn, (1, 2, 3, 5, 0), pair=pair, out2=True, gate=True, gate2=True)
    _check(ops, case, "F32_STORE", bn, (1, 2, 3, 5, 0), pair=pair)


# Fewer k-blocks than ring stages (K = 16 and 64: one k-block; 200: four), and more (1000: sixteen), with many tiles
# per CTA so that each warpgroup's ring position skips the other's k-blocks many times over.
@pytest.mark.parametrize("K", [16, 64, 200, 1000])
@pytest.mark.parametrize("bn", [64, 128])
def test_few_kblocks(ops, K, bn):
    case = Case(600, 520, K, seed=K)
    _check(ops, case, "GELU", bn, (1, 3, 0), pair=bn == 128, out2=True)


# K2 = 384: six extension k-blocks after four main ones, more than the 5 ring stages of block_n 128
@pytest.mark.parametrize("b_mn,K2", [pytest.param(False, 128, id="False"), pytest.param(True, 128, id="True"),
                                     pytest.param(False, 384, id="k2_384-False"), pytest.param(True, 384, id="k2_384-True")])
def test_lora_extension_groups(ops, b_mn, K2):
    """The K2 extension with per-group A2 slices: the other warpgroup's tiles pass main and extension k-blocks."""
    case = Case(300, 768, 200, b_mn=b_mn, K2=K2, group=256, rps=RPS, seed=7)
    _check(ops, case, "GATE_RES", 128, (1, 2, 5, 0), out2=True, gate=True, gate2=True)


@pytest.mark.parametrize("bn", [64, 128])
def test_batched_gaps(ops, bn):
    """Batched launch: every batch's out and out2 at its own c_boff, the gaps between the slices untouched."""
    case = Case(300, 200, 192, batch=3, rps=RPS, seed=3)
    _check(ops, case, "GELU", bn, (2, 5, 0), pair=bn == 128, out2=True)
    _check(ops, case, "GATE_RES", bn, (3, 0), pair=bn == 128, gate=True)


def test_in_place_residual_many_tiles(ops):
    """out == res over ten tiles per CTA: each element's residual is read before it is overwritten."""
    case = Case(640, 512, 128, rps=RPS, seed=5)
    _check(ops, case, "GATE_RES", 128, (2, 1, 0), in_place=True, gate=True)


@pytest.mark.parametrize("epi,kw", [
    ("STORE", {}), ("GELU", {}), ("GELU", dict(out2=True)), ("SILU", {}), ("SILU", dict(out2=True)),
    ("GATE_RES", {}), ("GATE_RES", dict(gate=True)), ("GATE_RES", dict(gate2=True, out2=True)),
    ("GATE_RES", dict(gate=True, gate2=True, out2=True)), ("MUL_DGELU", {})],
    ids=["store", "gelu", "gelu-out2", "silu", "silu-out2", "res", "gate", "gate2-out2", "gate-gate2-out2", "dgelu"])
@pytest.mark.parametrize("bn", [64, 128])
def test_every_bf16_epilogue(ops, epi, kw, bn):
    case = Case(300, 328, 200, b_mn=True, K2=64, rps=RPS, seed=11)
    _check(ops, case, epi, bn, (3, 0), pair=bn == 128, **kw)
