"""The GEMM's ping-pong schedule on 2-CTA clusters: the two CTAs of a cluster compute N tiles (m, 2 np) and (m, 2 np + 1)
and each loads half of the shared A tile (and LoRA A2 slice), which the TMA multicasts into both.  Each output element
still gets the same MMAs in the same k-order as on a single CTA, so every case here is bitwise equal to the single-CTA
ping-pong launch (cta_pair = 1), and every output lives in a sentinel-filled buffer whose elements outside the output
windows must survive.

cta_pair = 2 takes the ping-pong pairs when block_n is 128, the launch can ping-pong at all, there are more pair items
(m tile, pair of N tiles, batch) than max_ctas / 2, and a2_group_n is a multiple of 256; otherwise it runs the
cooperative M-pairs, which give the same bits.  So every pair launch here is also checked, by the kernel name the
profiler records, to have run the ping-pong pair instantiation gemm_kernel<128, 0, B_MN, true, true>."""
import re

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from _util import check_sentinel, sentinel_buffer, window

pytestmark = pytest.mark.gpu

EPI = dict(STORE=0, GELU=1, SILU=2, GATE_RES=3, MUL_DGELU=4, F32_STORE=7)


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


def _up8(x):
    return (x + 7) // 8 * 8


class Case:
    """Operands of one GEMM with every epilogue input it may use; launch() returns the output windows.  Samples of the
    per-sample gates are `rps` rows long (a multiple of 128, or all of M: ping-pong tiles lie inside one sample)."""

    def __init__(self, M, N, K, b_mn=False, K2=0, group=0, batch=1, rps=None, seed=0):
        self.M, self.N, self.K, self.K2, self.group, self.batch = M, N, K, K2, group, batch
        self.b_mn, self.rps = b_mn, rps or M
        g = torch.Generator(device="cuda").manual_seed(seed)

        def rnd(r, c, s=1.0):
            return (torch.randn(r, _up8(c), device="cuda", generator=g) * s).bfloat16()

        z = batch - 1
        # batch z: rows z * 8 further down A, B rows / columns z * 16 further in
        self.a_boff = (8, 0)
        self.b_boff = (0, 16) if b_mn else (16, 0)
        self.A = rnd(M + 8 * z, K)
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
        nsmp = (M + self.rps - 1) // self.rps
        self.tab = rnd(2, N, 0.5)
        self.temb = rnd(nsmp, 2 * N + 8, 0.5)

    def _buffer(self, ld, boff, dtype):
        n = (self.batch - 1) * boff + self.M * ld + 32
        buf = sentinel_buffer(n, dtype)
        return buf, [window(buf, z * boff, self.M, self.N, ld) for z in range(self.batch)]

    def launch(self, ops, epi, out2=False, gate=False, gate2=False, **launch):
        dtype = torch.float32 if epi == "F32_STORE" else torch.bfloat16
        buf, wins = self._buffer(self.ldc, self.c_boff, dtype)
        kw = dict(M=self.M, N=self.N, K=self.K, ldc=self.ldc, b_mn=self.b_mn, batch=self.batch,
                  a_boff=self.a_boff, b_boff=self.b_boff, c_boff=self.c_boff, epi=EPI[epi], alpha=0.75,
                  bias=self.bias, block_n=128, **launch)
        if self.K2:
            kw.update(A2=self.A2, B2=self.B2, K2=self.K2, a2_group_n=self.group)
        if epi == "GATE_RES":
            kw.update(res=self.res, ldres=self.ldres)
            if gate or gate2:
                kw.update(temb_stride=self.temb.stride(0), rows_per_sample=self.rps)
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


PAIR_PP = re.compile(r"gemm_kernel<128, 0, [01], true, true>")
SINGLE_PP = re.compile(r"gemm_kernel<128, 0, [01], false, true>")


def _profiled(fn):
    """fn()'s result and the names of the GEMM kernels it launched."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e.name for e in prof.events() if "gemm_kernel" in e.name]


def _launch_pair(ops, case, epi, **kw):
    """A launch that must run the ping-pong pair kernel: its output windows."""
    out, names = _profiled(lambda: case.launch(ops, epi, **kw))
    assert len(names) == 1 and PAIR_PP.search(names[0]), f"{epi} {kw}: ran {names}, not the ping-pong pair kernel"
    return out


def _check(ops, case, epi, max_ctas_list, **epi_kw):
    """Pair ping-pong launches on every grid in max_ctas_list, and a repeat of the first, against single-CTA
    ping-pong."""
    want = case.launch(ops, epi, cta_pair=1, max_ctas=max_ctas_list[0], **epi_kw)
    for mc in max_ctas_list:
        _assert_same(_launch_pair(ops, case, epi, cta_pair=2, max_ctas=mc, **epi_kw), want, f"{epi} pair max_ctas={mc}")
    _assert_same(case.launch(ops, epi, cta_pair=2, max_ctas=max_ctas_list[0], **epi_kw), want, f"{epi} pair repeat")


EPILOGUES = [("STORE", {}), ("GELU", {}), ("GELU", dict(out2=True)), ("SILU", {}), ("SILU", dict(out2=True)),
             ("GATE_RES", {}), ("GATE_RES", dict(gate=True)), ("GATE_RES", dict(gate2=True, out2=True)),
             ("MUL_DGELU", {}), ("F32_STORE", {})]
EPI_IDS = ["store", "gelu", "gelu-out2", "silu", "silu-out2", "res", "gate", "gate2-out2", "dgelu", "f32"]


# M = 300: 3 ragged M tiles; N = 584: 5 N tiles (the last 72 columns wide), so the last pair's second CTA has no tile;
# K = 200: a ragged last k-block.  9 pair items; max_ctas 2, 3 (one cluster), 6 and 10 give a cluster 9, 9, 3 and 2
# items (odd and even counts per warpgroup).  Gates: samples of 256 rows, so the second M tile's gate is sample 0's and
# the third's sample 1's.
@pytest.mark.parametrize("epi,kw", EPILOGUES, ids=EPI_IDS)
@pytest.mark.parametrize("b_mn", [False, True])
def test_every_epilogue_ragged(ops, epi, kw, b_mn):
    case = Case(300, 584, 200, b_mn=b_mn, K2=64, rps=256, seed=11)
    _check(ops, case, epi, (2, 3, 6, 10), **kw)


# LoRA extension with per-group A2 slices (a2_group_n 256 and 512: both tiles of a pair read one slice, multicast), and
# more extension k-blocks (K2 = 384: six) than the 5 ring stages
@pytest.mark.parametrize("group,K2", [(256, 64), (512, 128), (256, 384), (0, 128)])
@pytest.mark.parametrize("b_mn", [False, True])
def test_lora_extension_groups(ops, group, K2, b_mn):
    case = Case(520, 1024, 192, b_mn=b_mn, K2=K2, group=group, seed=7)
    _check(ops, case, "GELU", (4, 10), out2=True)
    _check(ops, case, "GATE_RES", (6,), gate=True)


# Fewer k-blocks than ring stages (K = 16 and 64: one; 200: four) and many (1000: sixteen), with many items per cluster
@pytest.mark.parametrize("K", [16, 64, 200, 1000])
def test_few_kblocks(ops, K):
    case = Case(600, 1160, K, seed=K)  # 5 x 10 tiles (the last 8 columns wide), 25 pair items
    _check(ops, case, "STORE", (2, 8))
    _check(ops, case, "MUL_DGELU", (6,))


@pytest.mark.parametrize("b_mn", [False, True])
def test_batched_gaps(ops, b_mn):
    """Batched launch: every batch's out and out2 at its own c_boff, the gaps between the slices untouched."""
    case = Case(300, 328, 192, b_mn=b_mn, batch=3, seed=3)  # 3 M tiles x 2 pairs (3 N tiles) x 3 batches
    _check(ops, case, "GELU", (4, 6, 12), out2=True)
    _check(ops, case, "GATE_RES", (6,), gate=True)


# The step's twelve GEMMs (tools/gemm_bench.py) at M = 2688, each with its step epilogue, on the full grid: the automatic
# choice (cta_pair = 0) and forced pairs against single-CTA ping-pong.
D, RP = 2048, 64
STEP = [  # name, N, K, MN-major B, epilogue, K2, a2_group_n
    ("qkv", 3 * D, D, False, "store", RP, D), ("to_out", D, D, False, "gate", RP, 0),
    ("to_q2", D, D, False, "store", RP, 0), ("to_out2", D, D, False, "res", RP, 0),
    ("ffn_up", 4 * D, D, False, "gelu2", 0, 0), ("ffn_down", D, 4 * D, False, "gate", 0, 0),
    ("qkv.dX", D, 3 * D, True, "store", 3 * RP, 0), ("to_out.dX", D, D, True, "store", RP, 0),
    ("to_q2.dX", D, D, True, "gate2", RP, 0), ("to_out2.dX", D, D, True, "store", RP, 0),
    ("ffn_down.dX", 4 * D, D, True, "dgelu", 0, 0), ("ffn_up.dX", D, 4 * D, True, "store", 0, 0)]
STEP_EPI = dict(store=("STORE", {}), gate=("GATE_RES", dict(gate=True)), res=("GATE_RES", {}),
                gelu2=("GELU", dict(out2=True)), gate2=("GATE_RES", dict(gate2=True, out2=True)),
                dgelu=("MUL_DGELU", {}))


@pytest.mark.parametrize("name,N,K,b_mn,epi,K2,group", STEP, ids=[s[0] for s in STEP])
def test_step_shapes(ops, name, N, K, b_mn, epi, K2, group):
    case = Case(2688, N, K, b_mn=b_mn, K2=K2, group=group, seed=N + K)
    e, kw = STEP_EPI[epi]
    want = case.launch(ops, e, cta_pair=1, **kw)
    _assert_same(_launch_pair(ops, case, e, cta_pair=0, **kw), want, f"{name} auto")
    _assert_same(_launch_pair(ops, case, e, cta_pair=2, **kw), want, f"{name} pair")


# The automatic choice keeps single-CTA ping-pong where pairs were not measured: an odd N-tile count (the last pair
# would have an empty tile), a single N tile (the rank-128 LoRA du launch), batched launches (the block-batched LoRA
# and kv2 projections), and launches with at most one tile per CTA.
@pytest.mark.parametrize("M,N,K,batch,max_ctas", [
    pytest.param(2688, 1152, 256, 1, 0, id="odd-n-tiles"),       # 21 x 9 tiles
    pytest.param(20000, 128, 256, 1, 0, id="one-n-tile"),        # 157 x 1 tiles
    pytest.param(600, 1024, 256, 4, 0, id="batched"),            # 5 x 8 x 4 tiles
    pytest.param(600, 1024, 256, 1, 40, id="one-tile-per-cta")])  # 40 tiles on 40 CTAs: cooperative
def test_automatic_choice_keeps_single_cta(ops, M, N, K, batch, max_ctas):
    case = Case(M, N, K, batch=batch, seed=N)
    want = case.launch(ops, "STORE", cta_pair=1, max_ctas=max_ctas)
    got, names = _profiled(lambda: case.launch(ops, "STORE", cta_pair=0, max_ctas=max_ctas))
    assert len(names) == 1 and "true, true>" not in names[0], f"automatic choice ran {names}"
    if max_ctas == 0:
        assert SINGLE_PP.search(names[0]), f"automatic choice ran {names}, not single-CTA ping-pong"
    _assert_same(got, want, "auto")
