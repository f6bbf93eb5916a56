"""Two-context attention (b2d_attn_dual_fwd_hd / b2d_attn_dual_bwd_hd, Wan image-to-video cross attention) against the
single-context kernels and the fp64 reference of test_gpu_attention_conformance.py.

  forward:  lse1, lse2, bf16(O1), bf16(O2) bit-identical to b2d_attn_fwd_hd on (q, k1, v1) and (q, k2, v2);
            out == bf16(float(bf16(O1)) + float(bf16(O2))) bit for bit.
  backward: dk1, dv1 bit-identical to b2d_attn_bwd_hd(q, k1, v1, NULL, out1, dout, lse1) and inside its fp64 bounds;
            dq within the sum of the two contexts' fp64 dQ bounds (each without its final rounding) plus one bf16 ulp of
            the summed reference: the kernel accumulates both contexts in fp32 and rounds once.
Every output sits inside a sentinel buffer and the workspace starts NaN-filled; each (sample, head) is scaled by its own
power of two, so a row term read for the wrong context, sample or head fails element-wise.  The shapes cover every
dispatch branch: Sk1 on both sides of each key tile and of 512 (the split dK/dV path and its workspace tail), Sk2 from
one key to several tiles, one ragged or full query tile, the unsplit dK/dV path at 40 heads, and the real I2V-14B cross
attention; a forward given only one of out1 / out2 writes the same bits and leaves the other buffer alone."""
import math

import pytest
import torch

from _util import bf16_ulp, check_bound, check_sentinel, sentinel_buffer, window
from test_gpu_attention_conformance import mags, reference

pytestmark = pytest.mark.gpu

PAD = 512


def _bits(t):
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _same(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), f"{what}: not bit-identical ({(_bits(a) != _bits(b)).sum().item()} differ)"


def _guarded(shape, dtype):
    n = math.prod(shape)
    buf = sentinel_buffer(n + 2 * PAD, dtype)
    return buf, buf[PAD:PAD + n].view(shape)


def _inputs(B, H, Sq, Sk1, Sk2, d, seed):
    gen = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    out = []
    for S in (Sq, Sk1, Sk1, Sk2, Sk2, Sq):
        out.append((torch.randn(B, H, S, d, device="cuda") * mags(B, H, gen=gen)).bfloat16())
    q, k1, v1, k2, v2, g = out
    return q, k1, v1, k2, v2, g, g.transpose(1, 2).reshape(B, Sq, H * d).contiguous()


CASES = [(2, 3, 1000, 512, 257), (2, 3, 1000, 383, 1), (1, 5, 300, 512, 1), (1, 5, 300, 200, 257)]

# Every dispatch branch of the two-context kernels.  Sk1 (text keys) on both sides of the 64- and 128-row tiles and of
# Sk1 = 512, above which the single-context workspace has no partial-sum tail, so context 2's row terms sit at another
# offset; Sk2 (image keys) from one key to several streamed tiles, so the forward's ring and the dQ pass switch contexts
# at many tile phases.  Sq = 1000 with B H = 6 takes the split dK/dV path whenever Sk1 <= 512; Sq = 1, 127 and 128 (one
# ragged or full query tile, never split) run on a subset that still covers every Sk1 and every Sk2.
GRID_SK1 = (1, 64, 128, 129, 383, 512, 513, 1023)
GRID_SK2 = (1, 128, 257, 700)
GRID = [(2, 3, 1000, s1, s2) for s1 in GRID_SK1 for s2 in GRID_SK2]
GRID += [(2, 3, sq, s1, GRID_SK2[(i + j) % len(GRID_SK2)]) for j, sq in enumerate((1, 127, 128))
         for i, s1 in enumerate(GRID_SK1)]
# B H = 160 (key) CTAs fill the GPU: the unsplit dK/dV path, as Wan I2V-14B's cross attention (40 heads) takes it
UNSPLIT = [(4, 40, 1000, 383, 257), (4, 40, 1000, 512, 257)]


def _ids(cases):
    return [f"B{c[0]}H{c[1]}Sq{c[2]}Sk{c[3]}+{c[4]}" for c in cases]


def _run_case(B, H, Sq, Sk1, Sk2, d, heads=None):
    """Both kernels on one shape, every output in a sentinel buffer and a NaN-filled workspace: bit identity with the
    single-context kernels (all heads), and dk1 / dv1 / dq against fp64 on the first ``heads`` heads (all by default).
    Returns the worst error / bound of dq, dk1 and dv1."""
    from finetrainers_b200 import ops
    scale = d ** -0.5
    q, k1, v1, k2, v2, g, g_tok = _inputs(B, H, Sq, Sk1, Sk2, d, seed=Sq + Sk1 + Sk2 + d)
    bufs, t = {}, {}
    for name, shape, dt in (("out", (B, Sq, H * d), torch.bfloat16), ("out1", (B, Sq, H * d), torch.bfloat16),
                            ("out2", (B, Sq, H * d), torch.bfloat16), ("lse1", (B, H, Sq), torch.float32),
                            ("lse2", (B, H, Sq), torch.float32), ("dq", (B, H, Sq, d), torch.bfloat16),
                            ("dk1", (B, H, Sk1, d), torch.bfloat16), ("dv1", (B, H, Sk1, d), torch.bfloat16)):
        bufs[name], t[name] = _guarded(shape, dt)
    ops.attn_dual_fwd(q, k1, v1, Sk1, k2, v2, Sk2, t["out"], t["lse1"], t["lse2"], B, H, Sq, scale, out1=t["out1"],
                      out2=t["out2"], head_dim=d)
    ws = torch.full((ops.attn_dual_bwd_ws_floats(B, H, Sq, Sk1, head_dim=d),), float("nan"), device="cuda")
    ops.attn_dual_bwd(q, k1, v1, Sk1, k2, v2, Sk2, t["out1"], t["out2"], g_tok, t["lse1"], t["lse2"], ws, t["dq"],
                      t["dk1"], t["dv1"], B, H, Sq, scale, head_dim=d)
    torch.cuda.synchronize()
    for name, buf in bufs.items():
        n = t[name].numel()
        check_sentinel(buf, [window(buf, PAD, 1, n, n)], name)

    # the forward without the branch outputs writes the same out and lse
    out_b, l1_b, l2_b = torch.empty_like(t["out"]), torch.empty_like(t["lse1"]), torch.empty_like(t["lse2"])
    ops.attn_dual_fwd(q, k1, v1, Sk1, k2, v2, Sk2, out_b, l1_b, l2_b, B, H, Sq, scale, head_dim=d)
    for a, b, what in ((out_b, t["out"], "out"), (l1_b, t["lse1"], "lse1"), (l2_b, t["lse2"], "lse2")):
        _same(a, b, f"{what} without out1 / out2")

    # each context against the single-context kernels
    for i, (k, v, Sk) in enumerate(((k1, v1, Sk1), (k2, v2, Sk2)), 1):
        o, l = torch.empty_like(t["out"]), torch.empty(B, H, Sq, device="cuda")
        ops.attn_fwd(q, k, v, None, o, l, B, H, Sq, Sk, scale, head_dim=d)
        _same(t[f"out{i}"], o, f"out{i}")
        _same(t[f"lse{i}"], l, f"lse{i}")
    _same(t["out"], (t["out1"].float() + t["out2"].float()).bfloat16(), "out = bf16(out1 + out2)")
    dq_s, dk_s, dv_s = torch.empty_like(q), torch.empty_like(k1), torch.empty_like(v1)
    ws1 = torch.full((ops.attn_bwd_ws_floats(B, H, Sq, Sk1, head_dim=d),), float("nan"), device="cuda")
    ops.attn_bwd(q, k1, v1, None, t["out1"], g_tok, t["lse1"], ws1, dq_s, dk_s, dv_s, B, H, Sq, Sk1, scale, head_dim=d)
    _same(t["dk1"], dk_s, "dk1")
    _same(t["dv1"], dv_s, "dv1")

    n = H if heads is None else heads
    q, k1, v1, k2, v2, g = (x[:, :n] for x in (q, k1, v1, k2, v2, g))
    r1, r2 = reference(q, k1, v1, None, scale, g), reference(q, k2, v2, None, scale, g)
    rk = check_bound(t["dk1"][:, :n], *r1["dk"], "dk1")
    rv = check_bound(t["dv1"][:, :n], *r1["dv"], "dv1")
    dq1, bdq1 = r1["dq"]
    dq2, bdq2 = r2["dq"]
    dq = dq1 + dq2
    bound = (bdq1 - bf16_ulp(dq1)) + (bdq2 - bf16_ulp(dq2)) + bf16_ulp(dq)
    ratio = check_bound(t["dq"][:, :n], dq, bound, f"dq B{B} H{H} Sq{Sq} Sk{Sk1}+{Sk2} d{d}")
    if Sk2 > 1:  # a single key has dS = P (dP - delta) = 0; otherwise dq without context 2 must miss its bound
        assert ((dq1 - dq).abs() > bound).any(), "context 2 contributes nothing to dq in this case"
    print(f"dual d{d} B{B} H{H} Sq{Sq} Sk{Sk1}+{Sk2}: error/bound dq {ratio:.3f}, dk1 {rk:.3f}, dv1 {rv:.3f}")
    return ratio, rk, rv


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("B,H,Sq,Sk1,Sk2", CASES, ids=_ids(CASES))
def test_dual_attention(B, H, Sq, Sk1, Sk2, d):
    _run_case(B, H, Sq, Sk1, Sk2, d)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("B,H,Sq,Sk1,Sk2", GRID, ids=_ids(GRID))
def test_dual_attention_dispatch_grid(B, H, Sq, Sk1, Sk2, d):
    _run_case(B, H, Sq, Sk1, Sk2, d)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("B,H,Sq,Sk1,Sk2", UNSPLIT, ids=_ids(UNSPLIT))
def test_dual_attention_unsplit_dkv(B, H, Sq, Sk1, Sk2, d):
    _run_case(B, H, Sq, Sk1, Sk2, d)


@pytest.mark.timeout(600)
def test_dual_attention_wan_i2v_14b_cross_attention():
    """The real I2V-14B cross attention of one 81 x 480 x 832 clip: 40 heads x 128, 32760 queries (a ragged last query
    tile), 512 text and 257 image keys.  Every head bit-identical to the single-context kernels; two heads against fp64
    with the element-wise bounds."""
    _run_case(1, 40, 32760, 512, 257, 128, heads=2)


OPTIONAL = [(2, 3, 1000, 513, 257), (1, 5, 127, 64, 700)]


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("B,H,Sq,Sk1,Sk2", OPTIONAL, ids=_ids(OPTIONAL))
@pytest.mark.parametrize("given", ["out1", "out2"])
def test_dual_attention_one_branch_output(B, H, Sq, Sk1, Sk2, d, given):
    """Only one of out1 / out2: out, lse1, lse2 and the given branch output bit-identical to the call that writes
    both; the omitted branch's buffer and everything around the written ones keep their sentinels."""
    from finetrainers_b200 import ops
    scale = d ** -0.5
    q, k1, v1, k2, v2, _, _ = _inputs(B, H, Sq, Sk1, Sk2, d, seed=7 + Sq + Sk1 + Sk2 + d)
    shapes = {"out": (B, Sq, H * d), "out1": (B, Sq, H * d), "out2": (B, Sq, H * d), "lse1": (B, H, Sq),
              "lse2": (B, H, Sq)}
    full = {n: torch.empty(s, dtype=torch.float32 if n.startswith("lse") else torch.bfloat16, device="cuda")
            for n, s in shapes.items()}
    ops.attn_dual_fwd(q, k1, v1, Sk1, k2, v2, Sk2, full["out"], full["lse1"], full["lse2"], B, H, Sq, scale,
                      out1=full["out1"], out2=full["out2"], head_dim=d)
    bufs, t = {}, {}
    for n, s in shapes.items():
        bufs[n], t[n] = _guarded(s, full[n].dtype)
    ops.attn_dual_fwd(q, k1, v1, Sk1, k2, v2, Sk2, t["out"], t["lse1"], t["lse2"], B, H, Sq, scale,
                      **{given: t[given]}, head_dim=d)
    torch.cuda.synchronize()
    omitted = "out2" if given == "out1" else "out1"
    for n, buf in bufs.items():
        if n == omitted:
            check_sentinel(buf, [], f"{n} (not passed)")
            continue
        check_sentinel(buf, [window(buf, PAD, 1, t[n].numel(), t[n].numel())], n)
        _same(t[n], full[n], f"{n} with only {given}")


def test_dual_refusals():
    from finetrainers_b200 import ops
    from finetrainers_b200.lib import B2DError
    q, k1, v1, k2, v2, g, g_tok = _inputs(1, 2, 130, 64, 3, 128, 0)
    out, l1, l2 = torch.empty(1, 130, 256, dtype=torch.bfloat16, device="cuda"), torch.empty(1, 2, 130, device="cuda"), \
        torch.empty(1, 2, 130, device="cuda")
    with pytest.raises(B2DError, match=r"\(code -1\)"):
        ops.attn_dual_fwd(q, k1, v1, 64, k2, v2, 3, out, l1, l2, 1, 2, 130, 0.1, head_dim=96)
    with pytest.raises(B2DError, match=r"\(code -1\)"):
        ops.attn_dual_fwd(q, k1, v1, 64, k2, v2, 0, out, l1, l2, 1, 2, 130, 0.1)
    with pytest.raises(B2DError, match=r"\(code -5\)"):
        ops.attn_dual_fwd(q, k1, v1, 64, k2, v2, 3, out, None, l2, 1, 2, 130, 0.1)
    with pytest.raises(B2DError, match=r"\(code -2\)"):
        ops.attn_dual_fwd(q, k1, v1, 64, k2, v2, 3, out.view(-1)[8:], l1, l2, 1, 2, 129, 0.1)
    ws = torch.empty(ops.attn_dual_bwd_ws_floats(1, 2, 130, 64) - 1, device="cuda")
    with pytest.raises(B2DError, match="workspace too small"):
        ops.attn_dual_bwd(q, k1, v1, 64, k2, v2, 3, out, out, g_tok, l1, l2, ws, q, k1, v1, 1, 2, 130, 0.1)
