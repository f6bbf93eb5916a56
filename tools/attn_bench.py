"""Attention kernels, by default self-attention at the BASELINE shape ([1, 32, 2688, 64] bf16): device time of forward
and backward next to PyTorch SDPA (cuDNN / flash backends) measured in the SAME run, plus a quick correctness check
against math SDPA.
  python tools/attn_bench.py [--no-sdpa] [--head-dim 64|128] [--heads H] [--seq Sq] [--kv-seq Sk] [--bias]
                             [--lib PATH]
Wan-2.1 T2V-1.3B self-attention: --head-dim 128 --heads 12 --seq 32760; its text cross-attention: add --kv-seq 512.
LTX text cross-attention as the step runs it: --kv-seq 128 --bias (an additive key bias of -10000 on the padded keys,
the last 51 of 128 as in the step's 77-token prompts, which times the masked path).
--lib PATH times another build of the library, so that two builds can be alternated in one session."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from finetrainers_b200 import lib  # noqa: E402

if "--lib" in sys.argv:  # time another build of the library (tools/micro/poly_exp_variants.py)
    lib.LIB_PATH = sys.argv[sys.argv.index("--lib") + 1]
from finetrainers_b200 import ops  # noqa: E402



def _arg(name, default):
    return int(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


dev = "cuda"
torch.manual_seed(0)
B, H, S, HD = 1, _arg("--heads", 32), _arg("--seq", 2688), _arg("--head-dim", 64)
SK = _arg("--kv-seq", S)
D = H * HD
rnd = lambda *s: torch.randn(*s, device=dev).bfloat16()  # noqa: E731
q, k, v = rnd(B, H, S, HD), rnd(B, H, SK, HD), rnd(B, H, SK, HD)
ao = torch.empty(B, S, D, device=dev, dtype=torch.bfloat16)
lse = torch.empty(B, H, S, device=dev)
dout = rnd(B, S, D)
dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
delta = torch.empty(ops.attn_bwd_ws_floats(B, H, S, SK, head_dim=HD), device=dev)
kb = None
if "--bias" in sys.argv:  # keys at and past 77/128 of Sk are padding: bias -10000, like the step's encoder mask
    kb = ((torch.arange(SK, device=dev) >= (SK * 77 + 127) // 128).float() * -10000.0).expand(B, SK).contiguous()


def t(fn, n=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


fwd = lambda: ops.attn_fwd(q, k, v, kb, ao, lse, B, H, S, SK, 0.125, head_dim=HD)  # noqa: E731
bwd = lambda: ops.attn_bwd(q, k, v, kb, ao, dout, lse, delta, dq, dk, dv, B, H, S, SK, 0.125, head_dim=HD)  # noqa: E731
fwd()
bwd()
torch.cuda.synchronize()
# correctness vs fp32 math attention on 4 heads (1 head when the score matrix is long)
NC = 4 if S * SK <= 2688 * 2688 else 1
qf, kf, vf = (x[:, :NC].float().requires_grad_(True) for x in (q, k, v))
ref = F.scaled_dot_product_attention(qf, kf, vf, attn_mask=None if kb is None else kb[:, None, None, :], scale=0.125)
ref.backward(dout.view(B, S, H, HD)[:, :, :NC].transpose(1, 2).float())
rel = lambda a, b: ((a.float() - b.float()).abs().max() / b.float().abs().max()).item()  # noqa: E731
print("err fwd %.2e dq %.2e dk %.2e dv %.2e" % (rel(ao.view(B, S, H, HD)[:, :, :NC].transpose(1, 2), ref), rel(dq[:, :NC], qf.grad),
                                                  rel(dk[:, :NC], kf.grad), rel(dv[:, :NC], vf.grad)), flush=True)
del qf, kf, vf, ref
tf, tb = t(fwd), t(bwd)
gf = 4.0 * S * SK * HD * H * B / 1e6
print("b200  fwd %7.1f us (%6.1f TFLOP/s)   bwd %7.1f us (%6.1f TFLOP/s at 2.5x fwd flops)" % (tf, gf / tf, tb, 2.5 * gf / tb), flush=True)
if "--long" in sys.argv:
    # ~1 s of back-to-back launches of each direction with NVML clock / power samples: shows whether a number is
    # taken at the power cap (SM clock well below its maximum) rather than at full clocks
    import threading
    import time
    import pynvml
    pynvml.nvmlInit()
    hnd = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
    for name, fn, n in (("fwd", fwd, 10000), ("bwd", bwd, 4000)):
        samples, stop = [], threading.Event()

        def sampler():
            while not stop.is_set():
                samples.append((pynvml.nvmlDeviceGetClockInfo(hnd, pynvml.NVML_CLOCK_SM), pynvml.nvmlDeviceGetPowerUsage(hnd) / 1e3))
                time.sleep(0.02)
        th = threading.Thread(target=sampler)
        th.start()
        us = t(fn, n)
        stop.set()
        th.join()
        half = samples[len(samples) // 2:]
        print("long %s: %7.1f us over %d launches; SM clock median %d MHz, power median %.0f W (second half of the loop)" % (
            name, us, n, sorted(c for c, _ in half)[len(half) // 2], sorted(w for _, w in half)[len(half) // 2]), flush=True)
if "--no-sdpa" not in sys.argv:
    from torch.nn.attention import SDPBackend, sdpa_kernel
    for name, be in (("cudnn", SDPBackend.CUDNN_ATTENTION), ("flash", SDPBackend.FLASH_ATTENTION)):
        try:
            qq, kk, vv = (x.clone().requires_grad_(True) for x in (q, k, v))
            g = torch.randn(B, H, S, HD, device=dev).bfloat16()
            with sdpa_kernel(be):
                am = None if kb is None else kb[:, None, None, :].bfloat16()
                f1 = lambda: F.scaled_dot_product_attention(qq, kk, vv, attn_mask=am, scale=0.125)  # noqa: E731
                o = f1()
                tf1 = t(lambda: f1())
                tb1 = t(lambda: torch.autograd.grad(o, (qq, kk, vv), g, retain_graph=True))
            print("sdpa/%s fwd %7.1f us   bwd %7.1f us" % (name, tf1, tb1), flush=True)
        except Exception as e:  # noqa: BLE001
            print("sdpa/%s unavailable: %r" % (name, e), flush=True)
