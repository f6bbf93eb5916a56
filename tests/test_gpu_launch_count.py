"""GPU: ops.LAUNCH_COUNT, the library's own count of the kernels it enqueued, equals the number of libb2d kernels the
device ran, as torch.profiler records them (every libb2d kernel is in namespace b2d): over an eager LTX training step
whose self- and cross-attention backward split their dK/dV pass, over an eager Wan image-to-video step with the
two-context backward, and over ops.attn_bwd alone on either side of the dK/dV split."""
import time

import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

from _util import SMALL, build_pair, run_b200_micro
from test_gpu_wan_i2v import SMALL64, _batch, _micro, _pair

pytestmark = pytest.mark.gpu


def _counted(fn):
    """-> (libb2d kernels the profiler saw run during fn, the increase of ops.LAUNCH_COUNT over fn).  The profiler keeps
    a kernel only if its device timestamps, converted to host time, fall inside the capture window, and that conversion
    drifts in a long-running process: a pause on each side keeps fn's launches well inside."""
    from finetrainers_b200 import ops
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.02)
        n0 = ops.LAUNCH_COUNT
        fn()
        torch.cuda.synchronize()
        n1 = ops.LAUNCH_COUNT
        time.sleep(0.02)
    ran = sum(1 for e in prof.events()
              if e.device_type == DeviceType.CUDA and e.name.removeprefix("void ").startswith("b2d::"))
    return ran, n1 - n0


def test_ltx_step_launch_count():
    """B = 1, 512 latent tokens, L = 128 text tokens, 4 heads: 4 (self) and 16 (cross) key-tile CTAs and 8 query tiles,
    so both attention backwards take the split dK/dV pass and its reduce."""
    from oracle import ltx_oracle as O
    _, om, bm = build_pair(SMALL, 16)
    batch = O.make_synthetic_batch(om.cfg, 1, 2, 16, 16, text_len=128, seed=7)

    def step():
        st, _, _ = run_b200_micro(bm, batch)
        st.optimizer_step()

    ran, counted = _counted(step)
    assert ran > 0 and counted == ran, (counted, ran)


def test_wan_i2v_step_launch_count():
    """Two blocks at head_dim 64, 512 latent tokens, 512 text + 257 image keys: the two-context backward with a split
    dK/dV pass for the text keys."""
    _, bm = _pair(2, **SMALL64)
    bt = _batch(F=2, H=32, W=32)
    from finetrainers_b200.trainer import SFTTrainStep
    st = SFTTrainStep(bm, flow_weighting_scheme="none")
    ran, counted = _counted(lambda: _micro(st, bt))
    assert ran > 0 and counted == ran, (counted, ran)


@pytest.mark.parametrize("below", [True, False])
def test_attn_bwd_launch_count_either_side_of_the_split(below):
    """One key tile per head and 16 query tiles: the dK/dV pass splits its query range while the (key tile, head) CTAs
    number fewer than the SMs (delta, split dK/dV, reduce, dQ), and runs whole from as many CTAs as SMs (delta, dK/dV,
    dQ)."""
    from finetrainers_b200 import ops
    nsm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    B, H, Sq, Sk = 1, nsm - 1 if below else nsm, 1024, 128
    torch.manual_seed(0)
    q = torch.randn(B, H, Sq, 64, device="cuda").bfloat16()
    k, v = torch.randn(B, H, Sk, 64, device="cuda").bfloat16(), torch.randn(B, H, Sk, 64, device="cuda").bfloat16()
    out = torch.empty(B, Sq, H * 64, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, Sq, device="cuda")
    ops.attn_fwd(q, k, v, None, out, lse, B, H, Sq, Sk, 0.125)
    dout = torch.randn_like(out)
    ws = torch.empty(ops.attn_bwd_ws_floats(B, H, Sq, Sk), device="cuda")
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    ran, counted = _counted(lambda: ops.attn_bwd(q, k, v, None, out, dout, lse, ws, dq, dk, dv, B, H, Sq, Sk, 0.125))
    assert counted == ran == (4 if below else 3), (counted, ran)
