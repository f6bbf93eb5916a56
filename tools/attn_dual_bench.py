"""Two-context attention (Wan-2.1 image-to-video cross attention) against the composed route on the same inputs:
  forward:  one b2d_attn_dual_fwd_hd (also with both branch outputs written, as a backward's recompute runs it)
            vs  attn_fwd(text) + attn_fwd(image) + a bf16 add
  backward: one b2d_attn_dual_bwd_hd  vs  attn_bwd(text) + attn_bwd(image) + a bf16 dQ add (the composed route also
            runs the image dK/dV pass, which the dual backward leaves out for frozen image projections)
Device time from CUDA events over --iters launches after --warmup, with the card's name, power limit and SM clocks read
in the same run.  Default shape: one block of the Wan I2V-14B 480P example, B 1, H 40, Sq 20 280 latent tokens,
512 text + 257 image keys, head_dim 128.
  python tools/attn_dual_bench.py [--heads H] [--seq Sq] [--text Sk1] [--image Sk2] [--head-dim 64|128]
                                  [--iters N] [--warmup W]"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from finetrainers_b200 import ops  # noqa: E402


def _arg(name, default):
    return int(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def _card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    B, H, Sq, Sk1, Sk2, d = 1, _arg("--heads", 40), _arg("--seq", 20280), _arg("--text", 512), _arg("--image", 257), \
        _arg("--head-dim", 128)
    iters, warmup = _arg("--iters", 20), _arg("--warmup", 5)
    torch.manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda").bfloat16()  # noqa: E731
    q, k1, v1, k2, v2 = rnd(B, H, Sq, d), rnd(B, H, Sk1, d), rnd(B, H, Sk1, d), rnd(B, H, Sk2, d), rnd(B, H, Sk2, d)
    dout = rnd(B, Sq, H * d)
    scale = d ** -0.5
    out, o1, o2 = (torch.empty(B, Sq, H * d, dtype=torch.bfloat16, device="cuda") for _ in range(3))
    l1, l2 = torch.empty(B, H, Sq, device="cuda"), torch.empty(B, H, Sq, device="cuda")
    dq, dq2, dk1, dv1 = torch.empty_like(q), torch.empty_like(q), torch.empty_like(k1), torch.empty_like(v1)
    dk2, dv2 = torch.empty_like(k2), torch.empty_like(v2)
    ws = torch.empty(ops.attn_dual_bwd_ws_floats(B, H, Sq, Sk1, head_dim=d), device="cuda")
    ws2 = torch.empty(ops.attn_bwd_ws_floats(B, H, Sq, Sk2, head_dim=d), device="cuda")

    def dual_fwd():
        ops.attn_dual_fwd(q, k1, v1, Sk1, k2, v2, Sk2, out, l1, l2, B, H, Sq, scale, head_dim=d)

    def dual_fwd_branches():  # as the block backward recomputes it: both branch outputs written too
        ops.attn_dual_fwd(q, k1, v1, Sk1, k2, v2, Sk2, out, l1, l2, B, H, Sq, scale, out1=o1, out2=o2, head_dim=d)

    def composed_fwd():
        ops.attn_fwd(q, k1, v1, None, o1, l1, B, H, Sq, Sk1, scale, head_dim=d)
        ops.attn_fwd(q, k2, v2, None, o2, l2, B, H, Sq, Sk2, scale, head_dim=d)
        torch.add(o1, o2, out=out)

    def dual_bwd():
        ops.attn_dual_bwd(q, k1, v1, Sk1, k2, v2, Sk2, o1, o2, dout, l1, l2, ws, dq, dk1, dv1, B, H, Sq, scale,
                          head_dim=d)

    def composed_bwd():
        ops.attn_bwd(q, k1, v1, None, o1, dout, l1, ws, dq, dk1, dv1, B, H, Sq, Sk1, scale, head_dim=d)
        ops.attn_bwd(q, k2, v2, None, o2, dout, l2, ws2, dq2, dk2, dv2, B, H, Sq, Sk2, scale, head_dim=d)
        dq.add_(dq2)

    ops.attn_dual_fwd(q, k1, v1, Sk1, k2, v2, Sk2, out, l1, l2, B, H, Sq, scale, out1=o1, out2=o2, head_dim=d)
    res = {"card": _card(), "shape": dict(B=B, H=H, Sq=Sq, Sk1=Sk1, Sk2=Sk2, head_dim=d), "iters": iters}
    for name, fn in (("dual_fwd", dual_fwd), ("dual_fwd_branch_outputs", dual_fwd_branches),
                     ("composed_fwd", composed_fwd), ("dual_bwd", dual_bwd),
                     ("composed_bwd", composed_bwd), ("dual_fwd_again", dual_fwd), ("composed_fwd_again", composed_fwd)):
        res[name + "_ms"] = round(_time(fn, iters, warmup), 4)
    res["card_after"] = _card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
