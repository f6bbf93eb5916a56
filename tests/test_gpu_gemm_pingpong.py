"""The GEMM's ping-pong schedule (single-CTA tiles at block_n 64 and 128, more tiles than CTAs): the two math warpgroups
take alternate tiles of a CTA's work list, so the edges are in how many tiles a CTA gets and how many k-blocks each tile
has.  Gate/residual launches take the cooperative schedule; their cases hold that choice to the same results.

Every case is bitwise equal to the CTA-pair launch at the same block_n (the cooperative schedule, which runs the same
MMAs in the same k-order for every element), to a repeat of itself, and to the launch on the full grid; every output
lives in a sentinel-filled buffer whose elements outside the output windows must survive."""
import pytest
import torch

from _util import check_sentinel, sentinel_buffer, window

pytestmark = pytest.mark.gpu

EPI = dict(STORE=0, GELU=1, SILU=2, GATE_RES=3, MUL_DGELU=4, F32_STORE=7)
RPS = 197  # rows per sample of the per-sample gates: sample boundaries fall inside tiles


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


def _up8(x):
    return (x + 7) // 8 * 8


class Case:
    """Operands of one GEMM with every epilogue input it may use; launch() returns the output windows."""

    def __init__(self, M, N, K, a_mn=False, b_mn=False, K2=0, group=0, batch=1, seed=0):
        self.M, self.N, self.K, self.K2, self.group, self.batch = M, N, K, K2, group, batch
        self.a_mn, self.b_mn = a_mn, b_mn
        g = torch.Generator(device="cuda").manual_seed(seed)

        def rnd(r, c, s=1.0):
            return (torch.randn(r, _up8(c), device="cuda", generator=g) * s).bfloat16()

        z = batch - 1
        # batch z: rows z * 8 further down A (or columns of an MN-major A), B rows / columns z * 16 further in
        self.a_boff = (0, 8) if a_mn else (8, 0)
        self.b_boff = (0, 16) if b_mn else (16, 0)
        self.A = rnd(K, M + 8 * z) if a_mn else rnd(M + 8 * z, K)
        self.B = rnd(K, N + 16 * z, K ** -0.5) if b_mn else rnd(N + 16 * z, K, K ** -0.5)
        groups = (N + group - 1) // group if group else 1
        if K2:
            self.A2 = rnd(M, K2 * groups)
            self.B2 = rnd(K2, N, K2 ** -0.5) if b_mn else rnd(N, K2, K2 ** -0.5)
        self.bias = rnd(1, N)[0]
        self.ldc, self.ldc2, self.ldres, self.ldaux = N + 24, N + 40, N + 56, N + 72
        self.c_boff = M * self.ldc2 + 40 if batch > 1 else 0  # out and out2 share it; gaps between the batch slices
        self.res = rnd(M, self.ldres)
        self.aux = rnd(M, self.ldaux)
        nsmp = (M + RPS - 1) // RPS
        self.tab = rnd(2, N, 0.5)
        self.temb = rnd(nsmp, 2 * N + 8, 0.5)

    def _buffer(self, ld, boff, dtype):
        n = (self.batch - 1) * boff + self.M * ld + 32
        buf = sentinel_buffer(n, dtype)
        return buf, [window(buf, z * boff, self.M, self.N, ld) for z in range(self.batch)]

    def launch(self, ops, epi, out2=False, gate=False, gate2=False, in_place=False, **launch):
        dtype = torch.float32 if epi == "F32_STORE" else torch.bfloat16
        buf, wins = self._buffer(self.ldc, self.c_boff, dtype)
        kw = dict(M=self.M, N=self.N, K=self.K, ldc=self.ldc, a_mn=self.a_mn, b_mn=self.b_mn, batch=self.batch,
                  a_boff=self.a_boff, b_boff=self.b_boff, c_boff=self.c_boff, epi=EPI[epi], alpha=0.75,
                  bias=self.bias, **launch)
        if self.K2:
            kw.update(A2=self.A2, B2=self.B2, K2=self.K2, a2_group_n=self.group)
        if epi == "GATE_RES":
            if in_place:
                wins[0].copy_(self.res[:, :self.N])
                kw.update(res=buf, ldres=self.ldc)
            else:
                kw.update(res=self.res, ldres=self.ldres)
            if gate or gate2:
                kw.update(temb_stride=self.temb.stride(0), rows_per_sample=RPS)
            if gate:
                kw.update(gate_table=self.tab[0], gate_temb=self.temb)
            if gate2:
                kw.update(gate2_table=self.tab[1], gate2_temb=self.temb[:, self.N:])
        if epi == "MUL_DGELU":
            kw.update(aux=self.aux, ldaux=self.ldaux)
        buf2 = wins2 = None
        if out2:
            buf2, wins2 = self._buffer(self.ldc2, self.c_boff, torch.bfloat16)
            kw.update(out2=buf2, ldc2=self.ldc2)
        ops.gemm(self.A, self.B, buf, **kw)
        check_sentinel(buf, wins, f"{epi} out")
        if out2:
            check_sentinel(buf2, wins2, f"{epi} out2")
        return wins + (wins2 or [])


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _assert_same(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        neq = _bits(g) != _bits(w)
        if neq.any():
            j = tuple(int(v) for v in neq.nonzero()[0])
            raise AssertionError(f"{what} [window {i}]: {int(neq.sum())} element(s) differ, first at {j}: "
                                 f"got {g[j].item()!r} want {w[j].item()!r}")


def _check(ops, case, epi, bn, max_ctas_list=(0,), pair=True, **epi_kw):
    """Ping-pong launches on every grid in max_ctas_list, and a repeat of the first, against the CTA-pair launch (or,
    at block_n 64, where pairs do not exist, against the first)."""
    first = case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=max_ctas_list[0], **epi_kw)
    want = case.launch(ops, epi, block_n=bn, cta_pair=2, **epi_kw) if pair else first
    _assert_same(first, want, f"{epi} bn{bn} max_ctas={max_ctas_list[0]} vs pair")
    _assert_same(case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=max_ctas_list[0], **epi_kw), first,
                 f"{epi} bn{bn} repeat")
    for mc in max_ctas_list[1:]:
        _assert_same(case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=mc, **epi_kw), want,
                     f"{epi} bn{bn} max_ctas={mc}")


# M = 300: 3 tiles of 128 rows (the last ragged); N = 200 / 328: 2 / 3 tiles of 128 columns (4 / 6 of 64).  Over
# max_ctas 1, 2, 3, 5 a CTA gets an odd or even number of tiles, one tile (warpgroup 1 idle) or none beyond its first.
@pytest.mark.parametrize("N", [200, 328])
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
def test_tiles_per_cta(ops, N, bn, a_mn, b_mn):
    case = Case(300, N, 200, a_mn=a_mn, b_mn=b_mn, seed=N + bn)
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
    case = Case(300, 768, 200, b_mn=b_mn, K2=K2, group=256, seed=7)
    _check(ops, case, "GATE_RES", 128, (1, 2, 5, 0), out2=True, gate=True, gate2=True)


@pytest.mark.parametrize("bn", [64, 128])
def test_batched_gaps(ops, bn):
    """Batched launch: every batch's out and out2 at its own c_boff, the gaps between the slices untouched."""
    case = Case(300, 200, 192, batch=3, seed=3)
    _check(ops, case, "GELU", bn, (2, 5, 0), pair=bn == 128, out2=True)
    _check(ops, case, "GATE_RES", bn, (3, 0), pair=bn == 128, gate=True)


def test_in_place_residual_many_tiles(ops):
    """out == res over ten tiles per CTA: each element's residual is read before it is overwritten."""
    case = Case(640, 512, 128, seed=5)
    _check(ops, case, "GATE_RES", 128, (2, 1, 0), in_place=True, gate=True)


@pytest.mark.parametrize("epi,kw", [
    ("STORE", {}), ("GELU", {}), ("GELU", dict(out2=True)), ("SILU", {}), ("SILU", dict(out2=True)),
    ("GATE_RES", {}), ("GATE_RES", dict(gate=True)), ("GATE_RES", dict(gate2=True, out2=True)),
    ("GATE_RES", dict(gate=True, gate2=True, out2=True)), ("MUL_DGELU", {})],
    ids=["store", "gelu", "gelu-out2", "silu", "silu-out2", "res", "gate", "gate2-out2", "gate-gate2-out2", "dgelu"])
@pytest.mark.parametrize("bn", [64, 128])
def test_every_bf16_epilogue(ops, epi, kw, bn):
    case = Case(300, 328, 200, b_mn=True, K2=64, seed=11)
    _check(ops, case, epi, bn, (3, 0), pair=bn == 128, **kw)
