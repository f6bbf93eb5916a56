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
import torch

from _util import check_sentinel, sentinel_buffer, window

pytestmark = pytest.mark.gpu

EPI = dict(GELU=1, SILU=2, GATE_RES=3)
COOP = 1 << 20  # max_ctas at or above the tile count: one tile per CTA, the cooperative schedule
GRIDS = (1, 2, 3, 5, 0)


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


def _up8(x):
    return (x + 7) // 8 * 8


class Case:
    """Operands of one GEMM with the gate/residual and second-output inputs; launch() returns the output windows."""

    def __init__(self, M, N, K, b_mn=False, K2=0, group=0, batch=1, rps=128, bias=True, seed=0):
        self.M, self.N, self.K, self.K2, self.group, self.batch, self.rps = M, N, K, K2, group, batch, rps
        self.b_mn = b_mn
        g = torch.Generator(device="cuda").manual_seed(seed)

        def rnd(r, c, s=1.0):
            return (torch.randn(r, _up8(c), device="cuda", generator=g) * s).bfloat16()

        z = batch - 1
        self.a_boff, self.b_boff = (8, 0), ((0, 16) if b_mn else (16, 0))
        self.A = rnd(M + 8 * z, K)
        self.B = rnd(K, N + 16 * z, K ** -0.5) if b_mn else rnd(N + 16 * z, K, K ** -0.5)
        groups = (N + group - 1) // group if group else 1
        if K2:
            self.A2 = rnd(M, K2 * groups)
            self.B2 = rnd(K2, N, K2 ** -0.5) if b_mn else rnd(N, K2, K2 ** -0.5)
        self.bias = rnd(1, N)[0] if bias else None
        self.ldc, self.ldc2, self.ldres = N + 24, N + 40, N + 56
        self.c_boff = M * self.ldc2 + 40 if batch > 1 else 0  # out and out2 share it; gaps between the batch slices
        self.res = rnd(M, self.ldres)
        nsmp = (M + rps - 1) // rps
        # gate vectors of exactly N elements each; the temb rows hold gate then gate2, one row per sample
        self.tab = [rnd(1, N, 0.5)[0, :N].contiguous() for _ in range(2)]
        self.temb = rnd(nsmp, 2 * N + 8, 0.5)

    def _buffer(self, ld, boff):
        buf = sentinel_buffer((self.batch - 1) * boff + self.M * ld + 32, torch.bfloat16)
        return buf, [window(buf, z * boff, self.M, self.N, ld) for z in range(self.batch)]

    def launch(self, ops, epi, out2=False, gate=False, gate2=False, in_place=False, **launch):
        buf, wins = self._buffer(self.ldc, self.c_boff)
        kw = dict(M=self.M, N=self.N, K=self.K, ldc=self.ldc, b_mn=self.b_mn, batch=self.batch, a_boff=self.a_boff,
                  b_boff=self.b_boff, c_boff=self.c_boff, epi=EPI[epi], alpha=0.75, bias=self.bias, **launch)
        if self.K2:
            kw.update(A2=self.A2, B2=self.B2, K2=self.K2, a2_group_n=self.group)
        if epi == "GATE_RES":
            if in_place:
                wins[0].copy_(self.res[:, :self.N])
                kw.update(res=buf, ldres=self.ldc)
            else:
                kw.update(res=self.res, ldres=self.ldres)
            if gate or gate2:
                kw.update(temb_stride=self.temb.stride(0), rows_per_sample=self.rps)
            if gate:
                kw.update(gate_table=self.tab[0], gate_temb=self.temb)
            if gate2:
                kw.update(gate2_table=self.tab[1], gate2_temb=self.temb[:, self.N:])
                out2 = True
        buf2 = wins2 = None
        if out2:
            buf2, wins2 = self._buffer(self.ldc2, self.c_boff)
            kw.update(out2=buf2, ldc2=self.ldc2)
        ops.gemm(self.A, self.B, buf, **kw)
        check_sentinel(buf, wins, f"{epi} out")
        if out2:
            check_sentinel(buf2, wins2, f"{epi} out2")
        return wins + (wins2 or [])


def _assert_same(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        neq = g.view(torch.int16) != w.view(torch.int16)
        if neq.any():
            j = tuple(int(v) for v in neq.nonzero()[0])
            raise AssertionError(f"{what} [window {i}]: {int(neq.sum())} element(s) differ, first at {j}: "
                                 f"got {g[j].item()!r} want {w[j].item()!r}")


def _check(ops, case, epi, bn, grids=GRIDS, **epi_kw):
    """Single-CTA launches on every grid in `grids`, and a repeat of the first, against the cooperative launch."""
    want = case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=COOP, **epi_kw)
    first = case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=grids[0], **epi_kw)
    _assert_same(first, want, f"{epi} bn{bn} max_ctas={grids[0]} vs cooperative")
    _assert_same(case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=grids[0], **epi_kw), first,
                 f"{epi} bn{bn} repeat")
    for mc in grids[1:]:
        _assert_same(case.launch(ops, epi, block_n=bn, cta_pair=1, max_ctas=mc, **epi_kw), want,
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
    case = Case(2688, s["N"], s["K"], b_mn=b_mn, K2=s["K2"], rps=2688, bias=not b_mn, seed=13)
    _check(ops, case, s["epi"], 128, grids=(0,), **s["kw"])
