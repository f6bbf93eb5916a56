"""Ping-pong epilogues that read and write their shared-memory tile as 8 x 8 matrices (ldmatrix / stmatrix) and load
the tile's bias before its first column chunk.

Each case runs every bf16 epilogue path of the ping-pong schedule (plain store, bias, GELU with its pre-activation
copy, residual, gate and gate2 copy, GELU') at ragged edges and at the step shapes, on single CTAs and on 2-CTA
clusters, with 2 and 3 tiles per CTA, and compares each output bit for bit with the same launch on the cooperative
schedule (one tile per CTA) or at block_n 64.  Every output lives in a sentinel-filled buffer whose elements past M and
N must survive."""
import pytest

from _gemm_case import Case, assert_same, load_ops

pytestmark = pytest.mark.gpu

COOP = 1 << 20  # max_ctas at or above the tile count: one tile per CTA, the cooperative schedule

KINDS = {
    "store": ("STORE", dict(bias=False)),
    "bias": ("STORE", {}),
    "gelu2": ("GELU", dict(out2=True)),
    "res": ("GATE_RES", dict(bias=False)),
    "gate": ("GATE_RES", dict(gate=True)),
    "gate2": ("GATE_RES", dict(gate2=True, bias=False)),
    "dgelu": ("MUL_DGELU", dict(bias=False)),
}


@pytest.fixture(scope="module")
def ops():
    return load_ops()


def _launch(ops, case, kind, **launch):
    epi, kw = KINDS[kind]
    return case.launch(ops, epi, **kw, **launch)


def _tiles(M, N, bn):
    return ((M + 127) // 128) * ((N + bn - 1) // bn)


# M = 300 and 600: a ragged last row tile; N % 128 = 64 (320, 448): the last 128-wide tile's second 64-column box lies
# wholly outside N; N = 264: the last tile is 8 columns wide, its first box partly outside.  max_ctas gives each CTA 2
# and then 3 tiles.
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("M,N", [(300, 320), (600, 448), (600, 264)])
@pytest.mark.parametrize("per_cta", [2, 3])
@pytest.mark.parametrize("b_mn", [False, True])
def test_ragged_edges_single_cta(ops, kind, M, N, per_cta, b_mn):
    case = Case(M, N, 192, b_mn=b_mn, seed=M + N + per_cta)
    want = _launch(ops, case, kind, block_n=128, cta_pair=1, max_ctas=COOP)
    grid = (_tiles(M, N, 128) + per_cta - 1) // per_cta
    assert_same(_launch(ops, case, kind, block_n=128, cta_pair=1, max_ctas=grid), want,
                f"{kind} M={M} N={N} {per_cta} tiles per CTA vs cooperative")
    grid64 = (_tiles(M, N, 64) + per_cta - 1) // per_cta
    assert_same(_launch(ops, case, kind, block_n=64, cta_pair=1, max_ctas=grid64), want,
                f"{kind} M={M} N={N} block_n 64, {per_cta} tiles per CTA")


# 2-CTA clusters (N-pairs sharing A): N = 512 and 768 (4 and 6 tiles of 128), a ragged M, 2 and 3 pair items per cluster
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("M,N", [(600, 512), (300, 768)])
@pytest.mark.parametrize("per_cta", [2, 3])
def test_ragged_m_cta_pairs(ops, kind, M, N, per_cta):
    case = Case(M, N, 256, seed=M + N)
    want = _launch(ops, case, kind, block_n=128, cta_pair=1, max_ctas=COOP)
    items = ((M + 127) // 128) * (N // 256)
    grid = 2 * ((items + per_cta - 1) // per_cta)
    assert_same(_launch(ops, case, kind, block_n=128, cta_pair=2, max_ctas=grid), want,
                f"{kind} M={M} N={N} pairs, {per_cta} items per cluster vs cooperative")


# The step's fused launches at M = 2688 (one 49x512x768 sample, D = 2048) with the library's automatic schedule (2-CTA
# ping-pong) against the cooperative one; K is cut to 512 to keep the test short (the epilogue does not see K).
STEP = {
    "to_out": (2048, False, "gate"),
    "to_out2": (2048, False, "res"),
    "ffn_up": (8192, False, "gelu2"),
    "ffn_down": (2048, False, "gate"),
    "to_q2.dX": (2048, True, "gate2"),
    "ffn_down.dX": (8192, True, "dgelu"),
    "qkv": (6144, False, "bias"),
}


@pytest.mark.parametrize("name", list(STEP))
def test_step_shapes(ops, name):
    N, b_mn, kind = STEP[name]
    case = Case(2688, N, 512, b_mn=b_mn, seed=17)
    want = _launch(ops, case, kind, block_n=128, cta_pair=1, max_ctas=COOP)
    assert_same(_launch(ops, case, kind), want, f"{name} automatic vs cooperative")
