"""Ping-pong epilogues that read and write their shared-memory tile as 8 x 8 matrices (ldmatrix / stmatrix) and load
the tile's bias before its first column chunk.

Each case runs every bf16 epilogue path of the ping-pong schedule (plain store, bias, GELU with its pre-activation
copy, residual, gate and gate2 copy, GELU') at ragged edges and at the step shapes, on single CTAs and on 2-CTA
clusters, with 2 and 3 tiles per CTA, and compares each output bit for bit with the same launch on the cooperative
schedule (one tile per CTA) or at block_n 64.  Every output lives in a sentinel-filled buffer whose elements past M and
N must survive."""
import pytest
import torch

from _util import check_sentinel, sentinel_buffer, window

pytestmark = pytest.mark.gpu

EPI = dict(STORE=0, GELU=1, GATE_RES=3, MUL_DGELU=4)
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
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


class Case:
    def __init__(self, M, N, K, b_mn=False, seed=0):
        self.M, self.N, self.K, self.b_mn = M, N, K, b_mn
        g = torch.Generator(device="cuda").manual_seed(seed)

        def rnd(*shape, s=1.0):
            return (torch.randn(*shape, device="cuda", generator=g) * s).bfloat16()

        self.A = rnd(M, K)
        self.B = rnd(K, N, s=K ** -0.5) if b_mn else rnd(N, K, s=K ** -0.5)
        self.bias = rnd(N, s=0.5)
        self.ldc, self.ldc2, self.ldx = N + 24, N + 40, N + 56
        self.x = rnd(M, self.ldx)  # residual or GELU' aux
        self.tab = rnd(N, s=0.5)
        self.temb = rnd(1, N + 8, s=0.5)

    def _buffer(self, ld):
        buf = sentinel_buffer(self.M * ld + 32, torch.bfloat16)
        return buf, window(buf, 0, self.M, self.N, ld)

    def launch(self, ops, kind, **launch):
        epi, kw0 = KINDS[kind]
        buf, win = self._buffer(self.ldc)
        kw = dict(M=self.M, N=self.N, K=self.K, ldc=self.ldc, b_mn=self.b_mn, epi=EPI[epi], alpha=0.75,
                  bias=None if kw0.get("bias") is False else self.bias, **launch)
        out2 = kw0.get("out2", False)
        if epi == "GATE_RES":
            kw.update(res=self.x, ldres=self.ldx)
            if kw0.get("gate") or kw0.get("gate2"):
                kw.update(temb_stride=self.temb.stride(0), rows_per_sample=self.M)
            if kw0.get("gate"):
                kw.update(gate_table=self.tab, gate_temb=self.temb)
            if kw0.get("gate2"):
                kw.update(gate2_table=self.tab, gate2_temb=self.temb)
                out2 = True
        if epi == "MUL_DGELU":
            kw.update(aux=self.x, ldaux=self.ldx)
        buf2 = win2 = None
        if out2:
            buf2, win2 = self._buffer(self.ldc2)
            kw.update(out2=buf2, ldc2=self.ldc2)
        ops.gemm(self.A, self.B, buf, **kw)
        check_sentinel(buf, [win], f"{kind} out")
        outs = [win.clone()]
        if out2:
            check_sentinel(buf2, [win2], f"{kind} out2")
            outs.append(win2.clone())
        return outs


def _assert_same(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        neq = g.view(torch.int16) != w.view(torch.int16)
        if neq.any():
            j = tuple(int(v) for v in neq.nonzero()[0])
            raise AssertionError(f"{what} [output {i}]: {int(neq.sum())} element(s) differ, first at {j}: "
                                 f"got {g[j].item()!r} want {w[j].item()!r}")


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
    want = case.launch(ops, kind, block_n=128, cta_pair=1, max_ctas=COOP)
    grid = (_tiles(M, N, 128) + per_cta - 1) // per_cta
    _assert_same(case.launch(ops, kind, block_n=128, cta_pair=1, max_ctas=grid), want,
                 f"{kind} M={M} N={N} {per_cta} tiles per CTA vs cooperative")
    grid64 = (_tiles(M, N, 64) + per_cta - 1) // per_cta
    _assert_same(case.launch(ops, kind, block_n=64, cta_pair=1, max_ctas=grid64), want,
                 f"{kind} M={M} N={N} block_n 64, {per_cta} tiles per CTA")


# 2-CTA clusters (N-pairs sharing A): N = 512 and 768 (4 and 6 tiles of 128), a ragged M, 2 and 3 pair items per cluster
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("M,N", [(600, 512), (300, 768)])
@pytest.mark.parametrize("per_cta", [2, 3])
def test_ragged_m_cta_pairs(ops, kind, M, N, per_cta):
    case = Case(M, N, 256, seed=M + N)
    want = case.launch(ops, kind, block_n=128, cta_pair=1, max_ctas=COOP)
    items = ((M + 127) // 128) * (N // 256)
    grid = 2 * ((items + per_cta - 1) // per_cta)
    _assert_same(case.launch(ops, kind, block_n=128, cta_pair=2, max_ctas=grid), want,
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
    want = case.launch(ops, kind, block_n=128, cta_pair=1, max_ctas=COOP)
    _assert_same(case.launch(ops, kind), want, f"{name} automatic vs cooperative")
