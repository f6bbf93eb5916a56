"""The GEMM's ping-pong schedule on 2-CTA clusters: the two CTAs of a cluster compute N tiles (m, 2 np) and (m, 2 np + 1)
and each loads half of the shared A tile (and LoRA A2 slice), which the TMA multicasts into both.  Each output element
still gets the same MMAs in the same k-order as on a single CTA, so every case here is bitwise equal to the same launch
with cta_pair = 1 (single-CTA ping-pong, or the cooperative schedule where a CTA gets one tile), and every output lives
in a sentinel-filled buffer whose elements outside the output windows must survive.

cta_pair = 2 takes the ping-pong pairs when block_n is 128, the launch can ping-pong at all, there are more pair items
(m tile, pair of N tiles, batch) than max_ctas / 2, and a2_group_n is a multiple of 256; otherwise it runs the
cooperative M-pairs, which give the same bits.  So every pair launch here is also checked, by the kernel name the
profiler records, to have run the ping-pong pair instantiation gemm_kernel<128, 0, B_MN, true, true>."""
import re
import time

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from _gemm_case import Case, assert_same, load_ops

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    return load_ops()


PAIR_PP = re.compile(r"gemm_kernel<128, 0, [01], true, true>")
SINGLE_PP = re.compile(r"gemm_kernel<128, 0, [01], false, true>")
PROFILE_PAD_S = 0.02


def _launch(ops, case, epi, **kw):
    """Every launch here is at block_n 128, the tile width of the ping-pong pairs."""
    return case.launch(ops, epi, block_n=128, **kw)


def _profiled(fn):
    """fn()'s result and the names of the GEMM kernels it launched.  The profiler keeps a kernel only if its device
    timestamps, converted to host time, fall inside the capture window, and that conversion drifts in a long-running
    process: a launch issued right after the window opens can be dropped.  A pause on each side keeps fn's launches
    well inside."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(PROFILE_PAD_S)
        out = fn()
        torch.cuda.synchronize()
        time.sleep(PROFILE_PAD_S)
    return out, [e.name for e in prof.events() if "gemm_kernel" in e.name]


def _launch_pair(ops, case, epi, **kw):
    """A launch that must run the ping-pong pair kernel: its output windows."""
    out, names = _profiled(lambda: _launch(ops, case, epi, **kw))
    assert len(names) == 1 and PAIR_PP.search(names[0]), f"{epi} {kw}: ran {names}, not the ping-pong pair kernel"
    return out


def _check(ops, case, epi, max_ctas_list, **epi_kw):
    """Pair ping-pong launches on every grid in max_ctas_list, and a repeat of the first, against single-CTA
    ping-pong."""
    want = _launch(ops, case, epi, cta_pair=1, max_ctas=max_ctas_list[0], **epi_kw)
    for mc in max_ctas_list:
        assert_same(_launch_pair(ops, case, epi, cta_pair=2, max_ctas=mc, **epi_kw), want, f"{epi} pair max_ctas={mc}")
    assert_same(_launch(ops, case, epi, cta_pair=2, max_ctas=max_ctas_list[0], **epi_kw), want, f"{epi} pair repeat")


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
    want = _launch(ops, case, e, cta_pair=1, **kw)
    assert_same(_launch_pair(ops, case, e, cta_pair=0, **kw), want, f"{name} auto")
    assert_same(_launch_pair(ops, case, e, cta_pair=2, **kw), want, f"{name} pair")


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
    want = _launch(ops, case, "STORE", cta_pair=1, max_ctas=max_ctas)
    got, names = _profiled(lambda: _launch(ops, case, "STORE", cta_pair=0, max_ctas=max_ctas))
    assert len(names) == 1 and "true, true>" not in names[0], f"automatic choice ran {names}"
    if max_ctas == 0:
        assert SINGLE_PP.search(names[0]), f"automatic choice ran {names}, not single-CTA ping-pong"
    assert_same(got, want, "auto")
