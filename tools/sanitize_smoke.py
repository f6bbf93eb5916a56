"""Small-shape pass over every libb2d kernel for `compute-sanitizer --tool memcheck` (ragged shapes on purpose: partial
tiles, odd batch, key masks).  Usage: compute-sanitizer --tool memcheck python tools/sanitize_smoke.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from finetrainers_b200 import ops  # noqa: E402
from _util import SMALL, build_pair, rnd, run_b200_micro  # noqa: E402

torch.manual_seed(0)
dev = "cuda"
# GEMM: majors, epilogues, extension, batch, split-K
for (M, N, K, a_mn, b_mn) in [(200, 192, 136, False, False), (300, 64, 256, False, True), (304, 128, 200, True, True)]:
    A = rnd(K, M) if a_mn else rnd(M, K)
    B = rnd(K, N, scale=0.05) if b_mn else rnd(N, K, scale=0.05)
    if a_mn:
        out = torch.zeros(M, N, device=dev)
        ops.gemm(A, B, out, M=M, N=N, K=K, a_mn=True, b_mn=b_mn, epi=ops.EPI_F32_ATOMIC, splits=2, block_n=64)
        outT = torch.zeros(N, M, device=dev)
        ops.gemm(A, B, outT, M=M, N=N, K=K, a_mn=True, b_mn=b_mn, epi=ops.EPI_F32_ATOMIC_T, block_n=64)
    else:
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        out2 = torch.zeros_like(out)
        bias, res = rnd(N), rnd(M, N)
        ops.gemm(A, B, out, M=M, N=N, K=K, b_mn=b_mn, bias=bias, epi=ops.EPI_GELU, out2=out2)
        ops.gemm(A, B, out, M=M, N=N, K=K, b_mn=b_mn, bias=bias, epi=ops.EPI_GATE_RES, res=res)
        ops.gemm(A, B, out, M=M, N=N, K=K, b_mn=b_mn, epi=ops.EPI_MUL_DGELU, aux=res)
# every tile width, both B layouts, ragged M / N / K, LoRA extension
for (M, N, K, bn, b_mn) in [(300, 520, 200, 256, False), (700, 320, 136, 160, True), (260, 384, 64, 192, False), (129, 128, 64, 128, True)]:
    A = rnd(M, K)
    B = rnd(K, N, scale=0.05) if b_mn else rnd(N, K, scale=0.05)
    u = rnd(M, 64, scale=0.3)
    Bl = rnd(64, N, scale=0.05) if b_mn else rnd(N, 64, scale=0.05)
    out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    ops.gemm(A, B, out, M=M, N=N, K=K, b_mn=b_mn, bias=rnd(N), A2=u, B2=Bl, K2=64, block_n=bn)
# attention: ragged query / key lengths, short keys (split dK/dV pass)
for (B_, H, Sq, Sk, use_bias) in [(1, 2, 200, 72, True), (2, 2, 130, 257, True), (1, 3, 1, 1, False), (3, 2, 300, 128, False),
                                  (1, 2, 640, 300, True), (1, 1, 384, 384, False)]:
    q, k, v = rnd(B_, H, Sq, 64), rnd(B_, H, Sk, 64), rnd(B_, H, Sk, 64)
    kb = None
    if use_bias:
        kb = torch.zeros(B_, Sk, device=dev)
        kb[:, Sk // 2:] = -10000.0
    out = torch.zeros(B_, Sq, H * 64, device=dev, dtype=torch.bfloat16)
    lse = torch.zeros(B_, H, Sq, device=dev)
    ops.attn_fwd(q, k, v, kb, out, lse, B_, H, Sq, Sk, 0.125)
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    ws = torch.zeros(ops.attn_bwd_ws_floats(B_, H, Sq, Sk), device=dev)
    ops.attn_bwd(q, k, v, kb, out, rnd(B_, Sq, H * 64), lse, ws, dq, dk, dv, B_, H, Sq, Sk, 0.125)
# whole small-model step (row kernels, fused q|k|v, batched text K/V, deferred adapter gradients, optimiser)
O, om, bm = build_pair(SMALL, 16)
batch = O.make_synthetic_batch(om.cfg, 2, 2, 3, 5, text_len=20, seed=3)
st, loss, _ = run_b200_micro(bm, batch)
st.optimizer_step()
torch.cuda.synchronize()
print("sanitize smoke done, loss", loss)
