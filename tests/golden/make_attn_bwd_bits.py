"""Writes tests/golden/attn_bwd_bits.json: the sha256 of out, lse, dq, dk and dv after one attention forward + backward
per shape, on inputs generated on the CPU from fixed seeds.  The hashes pin the attention kernels' results bit for bit:
a change that keeps every per-element sum in the same order reproduces them (tests/test_gpu_attention_bwd_tiles.py).
  python tests/golden/make_attn_bwd_bits.py [--lib PATH]
--lib PATH runs another build of the library."""
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "attn_bwd_bits.json")

# name -> (B, H, Sq, Sk, head_dim, key bias)
CASES = {
    "ltx_self": (1, 32, 2688, 2688, 64, False),
    "ltx_cross": (1, 32, 2688, 128, 64, True),
    "ltx13b_self": (1, 32, 2688, 2688, 128, False),
    "ragged_d64_bias": (1, 4, 1000, 640, 64, True),
    "ragged_d64_b2": (2, 3, 193, 1000, 64, False),
    "ragged_d64_small": (1, 5, 65, 129, 64, True),
    "split_d64": (1, 4, 1000, 300, 64, True),
    "split_d128": (1, 2, 1000, 300, 128, True),
    "ragged_d128": (2, 2, 129, 191, 128, True),
    "one_by_one": (1, 3, 1, 1, 64, False),
}


def inputs(B, H, Sq, Sk, d, bias, seed=0):
    """bf16 q, k, v [B,H,S,d], token-major dout [B,Sq,H*d] and the fp32 key bias [B,Sk] (uniform in [-4, 4) on the
    kept keys, -10000 on the last fifth), all drawn on the CPU"""
    gen = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, H, S, d, generator=gen).bfloat16() for S in (Sq, Sk, Sk))
    dout = torch.randn(B, Sq, H * d, generator=gen).bfloat16()
    kb = None
    if bias:
        kb = torch.rand(B, Sk, generator=gen) * 8 - 4
        kb[:, Sk - Sk // 5:] = -10000.0
    return q, k, v, dout, kb


def run(B, H, Sq, Sk, d, bias):
    """fwd + bwd through ops on cuda:0; returns {name: tensor} for out, lse, dq, dk, dv"""
    from finetrainers_b200 import ops
    q, k, v, dout, kb = (None if t is None else t.cuda() for t in inputs(B, H, Sq, Sk, d, bias))
    out = torch.zeros(B, Sq, H * d, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(B, H, Sq, device="cuda")
    scale = d ** -0.5
    ops.attn_fwd(q, k, v, kb, out, lse, B, H, Sq, Sk, scale, head_dim=d)
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    ws = torch.zeros(ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=d), device="cuda")
    ops.attn_bwd(q, k, v, kb, out, dout, lse, ws, dq, dk, dv, B, H, Sq, Sk, scale, head_dim=d)
    torch.cuda.synchronize()
    return {"out": out, "lse": lse, "dq": dq, "dk": dk, "dv": dv}


def sha256(t):
    t = t.detach().cpu().contiguous()
    bits = t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)
    return hashlib.sha256(bits.numpy().tobytes()).hexdigest()


def hashes(case):
    return {name: sha256(t) for name, t in run(*CASES[case]).items()}


def main():
    if "--lib" in sys.argv:
        from finetrainers_b200 import lib
        lib.LIB_PATH = os.path.abspath(sys.argv[sys.argv.index("--lib") + 1])
    bits = {case: hashes(case) for case in CASES}
    with open(OUT, "w") as f:
        json.dump(bits, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {OUT}: {len(bits)} shapes")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
