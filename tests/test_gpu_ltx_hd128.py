"""GPU: the head_dim-128 LTX-Video geometry.  The q/k-norm + RoPE + head-split row kernels at head_dim 128 against an
element-wise fp64 reference (bounds as in test_gpu_elem.py part B: forward ulp16(ref) + 2^-16 * 2 rowmax|n|, backward
ulp16(ref) + 2^-16 * rstd * rowmax|g| * (1 + rowmax|xhat|)^2, or 2 rowmax|dy| without a norm), outputs inside sentinel
buffers and unread inputs NaN; bit identity of the head_dim-taking entry points with the head_dim-64 ones; their argument
checks; then the training step at head_dim 128 against the CPU oracle (small models, the 13B width with two blocks),
under CUDA graphs, with layerwise fp8 storage, and the whole 13B geometry run twice."""
import copy
import ctypes as C

import pytest
import torch

from _util import (bf16_ulp, build_pair, check_bound, check_sentinel, rel_err, run_b200_micro, sentinel_buffer, window)

pytestmark = pytest.mark.gpu

NAN = float("nan")
PAD = 64
ALIGN, SHAPE, ARG = -2, -1, -5
SMALL128 = dict(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=128, cross_attention_dim=256,
                num_layers=2, caption_channels=128)
CLI_SKIP = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def _rowmax(t):
    return t.abs().amax(-1, keepdim=True)


def _bits(t):
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


class Guarded:
    """`n` output elements with PAD sentinel elements on each side."""

    def __init__(self, n):
        self.n = n
        self.buf = sentinel_buffer(n + 2 * PAD, torch.bfloat16)
        self.t = self.buf[PAD:PAD + n]

    def check(self, what, wins=None):
        check_sentinel(self.buf, wins if wins is not None else [window(self.buf, PAD, 1, self.n, self.n)], what)


class Problem:
    """nseg D-wide segments (D = H * hd) at col_off of rows [B*S, ld]; every other source column, the table row past S
    and the weight elements past D are NaN.  Weights are stacked per block of rows_per_w rows when rows_per_w > 0."""

    def __init__(self, B, S, H, hd, nseg, wmask, rope, col_off=24, ld_extra=40, dx_col_off=16, ld_dx_extra=88,
                 rows_per_w=0, w_stride=0, eps=1e-5, seed=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.B, self.S, self.H, self.hd, self.nseg, self.wmask, self.rope, self.eps = B, S, H, hd, nseg, wmask, rope, eps
        self.D = D = H * hd
        self.rows = rows = B * S
        self.col_off, self.ld = col_off, col_off + nseg * D + ld_extra
        self.dx_col_off, self.ld_dx = dx_col_off, dx_col_off + nseg * D + ld_dx_extra
        self.rows_per_w, self.w_stride = rows_per_w, w_stride
        self.src = torch.full((rows, self.ld), NAN, device="cuda", dtype=torch.bfloat16)
        self.src[:, col_off:col_off + nseg * D] = _rnd(g, rows, nseg * D)
        self.src[1 % rows, col_off:col_off + D] *= 1e-4          # a row small enough that eps decides its RMS
        ang = torch.randn(S + 1, D // 2, device="cuda", generator=g) * 3
        self.cos, self.sin = ang.cos(), ang.sin()
        self.cos[S], self.sin[S] = NAN, NAN
        nblk = rows // rows_per_w if rows_per_w else 1
        self.w = []
        for i in range(nseg):
            if not (wmask >> i) & 1:
                self.w.append(None)
                continue
            stride = w_stride if rows_per_w else 0
            w = torch.full((nblk * stride + 2 * D,), NAN, device="cuda", dtype=torch.bfloat16)
            for k in range(nblk):
                w[k * stride:k * stride + D] = (1 + 0.2 * torch.randn(D, device="cuda", generator=g)).bfloat16()
            self.w.append(w)
        self.dy = [_rnd(g, B, H, S, hd) for _ in range(nseg)]

    def seg(self, i):
        return self.src[:, self.col_off + i * self.D:self.col_off + (i + 1) * self.D]

    def weight_rows(self, i):
        w, D = self.w[i], self.D
        if not self.rows_per_w:
            return w[:D].double()[None].expand(self.rows, D)
        blk = torch.arange(self.rows, device="cuda") // self.rows_per_w
        return torch.stack([w[k * self.w_stride:k * self.w_stride + D] for k in range(int(blk.max()) + 1)]).double()[blk]

    def heads(self, t):      # [rows, D] -> [B, H, S, hd]: channel c of a row is lane c % hd of head c // hd
        return t.reshape(self.B, self.S, self.H, self.hd).transpose(1, 2)

    def rows_of(self, t):
        return t.transpose(1, 2).reshape(self.rows, self.D)

    def tables(self):
        return (self.cos, self.sin) if self.rope else (None, None)

    def reference(self, i):
        x = self.seg(i).double().requires_grad_(True)
        n = x
        s_idx = torch.arange(self.rows, device="cuda") % self.S
        norm, rot = self.w[i] is not None, (self.rope >> i) & 1
        if norm:
            rstd = torch.rsqrt((x * x).mean(-1, keepdim=True) + self.eps)     # over all D channels: across heads
            n = x * rstd * self.weight_rows(i)
        o = n
        if rot:
            c, s = self.cos[:self.S].double()[s_idx], self.sin[:self.S].double()[s_idx]
            a, b = n.unflatten(-1, (-1, 2)).unbind(-1)
            o = torch.stack([a * c - b * s, b * c + a * s], -1).flatten(-2)
        fwd = self.heads(o)
        fwd.backward(self.dy[i].double())
        f = fwd.detach()
        fb = bf16_ulp(f) + 2.0 ** -16 * 2 * self.heads(_rowmax(n.detach()).expand(-1, self.D))
        dyr = self.rows_of(self.dy[i].double())
        if norm:
            if rot:
                a, b = dyr.unflatten(-1, (-1, 2)).unbind(-1)
                dyr = torch.stack([a * c + b * s, b * c - a * s], -1).flatten(-2)
            gw = dyr * self.weight_rows(i)
            scl = rstd.detach() * _rowmax(gw) * (1 + _rowmax(x.detach() * rstd.detach())) ** 2
        else:
            scl = 2 * _rowmax(dyr)
        return f, x.grad, fb, bf16_ulp(x.grad) + 2.0 ** -16 * scl

    def run_fwd(self, ops, fn=None):
        dsts = [Guarded(self.B * self.H * self.S * self.hd) for _ in range(self.nseg)]
        c, s = self.tables()
        (fn or ops.qkv_norm_rope_fwd)(self.src, self.ld, self.col_off, self.w, self.rope, c, s,
                                      [d.t.view(self.B, self.H, self.S, self.hd) for d in dsts], self.B, self.S, self.H,
                                      self.eps, rows_per_w=self.rows_per_w, w_stride=self.w_stride, head_dim=self.hd)
        return dsts

    def run_bwd(self, ops, fn=None):
        dx = Guarded(self.rows * self.ld_dx)
        c, s = self.tables()
        (fn or ops.qkv_norm_rope_bwd)(self.dy, self.src, self.ld, self.col_off, self.w, self.rope, c, s,
                                      dx.t.view(self.rows, self.ld_dx), self.ld_dx, self.dx_col_off, self.B, self.S,
                                      self.H, self.eps, rows_per_w=self.rows_per_w, w_stride=self.w_stride,
                                      head_dim=self.hd)
        return dx

    def check(self, ops, what):
        dsts, dx = self.run_fwd(ops), self.run_bwd(ops)
        dxw = window(dx.buf, PAD + self.dx_col_off, self.rows, self.nseg * self.D, self.ld_dx)
        worst = 0.0
        for i in range(self.nseg):
            f, gx, fb, gb = self.reference(i)
            out = dsts[i].t.view(self.B, self.H, self.S, self.hd)
            dxi = dxw[:, i * self.D:(i + 1) * self.D]
            tag = f"{what} seg {i} (w {self.wmask:03b}, rope {self.rope:03b})"
            worst = max(worst, check_bound(out, f, fb, tag + " fwd"), check_bound(dxi, gx, gb, tag + " bwd"))
            if self.w[i] is None and not (self.rope >> i) & 1:       # neither norm nor rope: a copy both ways
                assert torch.equal(_bits(out), _bits(self.heads(self.seg(i)))), tag
                assert torch.equal(_bits(dxi), _bits(self.rows_of(self.dy[i]))), tag
            dsts[i].check(tag + " dst")
        dx.check(what + " dx", [dxw])
        return worst


# ---------------------------------------------------------------------------------------------------------------------
# row kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nseg", [1, 2, 3])
def test_hd128_every_weight_and_rope_combination(ops, nseg):
    """D = 256 (2 heads x 128): every weight present / absent x every rope_mask, B = 2, S = 7."""
    for wmask in range(1 << nseg):
        for rope in range(1 << nseg):
            Problem(2, 7, 2, 128, nseg, wmask, rope, seed=wmask * 8 + rope).check(ops, f"nseg={nseg}")


# every segment normed and not, rotated and not, the third segment's norm with and without the first two
SUBSET = [(3, 0b011, 0b011), (3, 0b100, 0b100), (3, 0b101, 0b010), (3, 0b111, 0b111), (3, 0b000, 0b000),
          (2, 0b10, 0b01), (2, 0b01, 0b00), (1, 0b1, 0b1), (1, 0b1, 0b0)]


@pytest.mark.parametrize("S", [7, 131])
@pytest.mark.parametrize("H", [6, 16, 17, 32, 64])
def test_hd128_widths(ops, H, S):
    """D = 768 and 2048 (one chunk), 2176 and 4096 (two chunks: the 13B row, three segments in the two-chunk kernel),
    8192 (four chunks); col_off = 24 and ld = 3 D + 64 > 3 D; S is a multiple of nothing."""
    worst = 0.0
    for nseg, wmask, rope in SUBSET:
        worst = max(worst, Problem(2, S, H, 128, nseg, wmask, rope, seed=H + S + wmask).check(ops, f"H={H} S={S}"))
    print(f"\nhead_dim 128, D = {H * 128}, S = {S}: worst error / bound {worst:.3f}")


def test_hd128_block_stacked_weights(ops):
    """rows_per_w > 0 as the text-side k|v launch uses it: three blocks of 2 x 5 rows at D = 4096, weights w_stride apart,
    the k segment normed and the v segment copied; plus a rotated form; rows_per_w = rows equals rows_per_w = 0."""
    Problem(6, 5, 32, 128, 2, 0b01, 0b00, rows_per_w=10, w_stride=4096, seed=3).check(ops, "kv2 layout")
    Problem(4, 7, 2, 128, 3, 0b011, 0b101, rows_per_w=14, w_stride=2 * 128 + 24, seed=11).check(ops, "stacked")
    q = Problem(2, 7, 2, 128, 3, 0b111, 0b011, seed=12)
    d0, x0 = q.run_fwd(ops), q.run_bwd(ops)
    q.rows_per_w, q.w_stride = q.rows, 8
    d1, x1 = q.run_fwd(ops), q.run_bwd(ops)
    for a, b in zip(d0, d1):
        assert torch.equal(_bits(a.buf), _bits(b.buf))
    assert torch.equal(_bits(x0.buf), _bits(x1.buf))


def test_hd128_single_segment_wrappers(ops):
    """ops.qknorm_rope_fwd / bwd with head_dim = 128 are the one-segment form."""
    for norm, rope in ((True, True), (True, False), (False, True)):
        p = Problem(3, 7, 6, 128, 1, int(norm), int(rope), seed=5)
        c, s = p.tables()
        d0, x0 = p.run_fwd(ops), p.run_bwd(ops)
        dst, dx = Guarded(d0[0].n), Guarded(x0.n)
        ops.qknorm_rope_fwd(p.src, p.ld, p.col_off, p.w[0], c, s, dst.t.view(p.B, p.H, p.S, 128), p.B, p.S, p.H, norm,
                            p.eps, head_dim=128)
        ops.qknorm_rope_bwd(p.dy[0], p.src, p.ld, p.col_off, p.w[0], c, s, dx.t.view(p.rows, p.ld_dx), p.ld_dx,
                            p.dx_col_off, p.B, p.S, p.H, norm, p.eps, head_dim=128)
        assert torch.equal(_bits(dst.buf), _bits(d0[0].buf)) and torch.equal(_bits(dx.buf), _bits(x0.buf))


def _hd_entry(ops, direction):
    """The head_dim-taking entry point called directly (ops routes head_dim 64 to the entry points without it)."""
    from finetrainers_b200 import lib
    so, P = lib.load(), ops._ptr

    def fwd(src, ld, col_off, weights, rope_mask, cos, sin, dsts, B, S, H, eps, rows_per_w=0, w_stride=0, *, head_dim):
        n = len(dsts)
        w, d = list(weights) + [None] * (3 - n), list(dsts) + [None] * (3 - n)
        lib.check(so.b2d_qkv_norm_rope_hd_fwd(P(src), C.c_int64(ld), C.c_int64(col_off), n, P(w[0]), P(w[1]), P(w[2]),
                                              int(rope_mask), P(cos), P(sin), P(d[0]), P(d[1]), P(d[2]), B, S, H,
                                              int(head_dim), C.c_float(eps), int(rows_per_w), C.c_int64(w_stride),
                                              ops._stream()), "hd_fwd")

    def bwd(dys, x, ld, col_off, weights, rope_mask, cos, sin, dx, ld_dx, dx_col_off, B, S, H, eps, rows_per_w=0,
            w_stride=0, *, head_dim):
        n = len(dys)
        w, d = list(weights) + [None] * (3 - n), list(dys) + [None] * (3 - n)
        lib.check(so.b2d_qkv_norm_rope_hd_bwd(P(d[0]), P(d[1]), P(d[2]), P(x), C.c_int64(ld), C.c_int64(col_off), n,
                                              P(w[0]), P(w[1]), P(w[2]), int(rope_mask), P(cos), P(sin), P(dx),
                                              C.c_int64(ld_dx), C.c_int64(dx_col_off), B, S, H, int(head_dim),
                                              C.c_float(eps), int(rows_per_w), C.c_int64(w_stride), ops._stream()),
                  "hd_bwd")

    return fwd if direction == "fwd" else bwd


@pytest.mark.parametrize("H", [2, 32, 33, 128])
def test_hd_entry_points_at_64_are_bit_identical_to_the_old_ones(ops, H):
    for nseg, wmask, rope in SUBSET[:4] + SUBSET[5:6] + SUBSET[7:8]:
        p = Problem(2, 9, H, 64, nseg, wmask, rope, seed=H + nseg)
        d_old, x_old = p.run_fwd(ops), p.run_bwd(ops)
        d_new, x_new = p.run_fwd(ops, _hd_entry(ops, "fwd")), p.run_bwd(ops, _hd_entry(ops, "bwd"))
        for a, b in zip(d_old, d_new):
            assert torch.equal(_bits(a.buf), _bits(b.buf)), (H, nseg, wmask, rope)
        assert torch.equal(_bits(x_old.buf), _bits(x_new.buf)), (H, nseg, wmask, rope)
    p = Problem(4, 7, H, 64, 2, 0b01, 0b00, rows_per_w=14, w_stride=H * 64 + 8, seed=H)
    a, b = p.run_fwd(ops), p.run_fwd(ops, _hd_entry(ops, "fwd"))
    assert all(torch.equal(_bits(x.buf), _bits(y.buf)) for x, y in zip(a, b))
    assert torch.equal(_bits(p.run_bwd(ops).buf), _bits(p.run_bwd(ops, _hd_entry(ops, "bwd")).buf))


def test_hd_entry_points_refuse_bad_arguments(ops):
    """Argument checks that return before any launch: head_dim, alignment, rope_mask / segments."""
    from finetrainers_b200.lib import B2DError
    p = Problem(2, 7, 2, 128, 3, 0b011, 0b011, seed=1)
    B, S, H = p.B, p.S, p.H
    dv = [torch.zeros(B, H, S, 128, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
    dx = torch.zeros(p.rows, p.ld_dx, dtype=torch.bfloat16, device="cuda")

    def code(c, fn):
        with pytest.raises(B2DError, match=rf"\(code {c}\)"):
            fn()

    def fwd(src=p.src, ld=p.ld, co=p.col_off, w=p.w, rope=p.rope, d=dv, hd=128, H=H, fn=ops.qkv_norm_rope_fwd):
        fn(src, ld, co, w, rope, p.cos, p.sin, d, B, S, H, p.eps, head_dim=hd)

    def bwd(dy=p.dy, x=p.src, w=p.w, rope=p.rope, dxt=dx, ld_dx=p.ld_dx, hd=128, fn=ops.qkv_norm_rope_bwd):
        fn(dy, x, p.ld, p.col_off, w, rope, p.cos, p.sin, dxt, ld_dx, p.dx_col_off, B, S, H, p.eps, head_dim=hd)

    for hd in (96, 32, 256, 0):
        code(SHAPE, lambda: fwd(hd=hd))
        code(SHAPE, lambda: bwd(hd=hd))
    code(SHAPE, lambda: fwd(hd=64, fn=_hd_entry(ops, "fwd"), H=129))       # 129 x 64 > 8192 columns
    code(SHAPE, lambda: fwd(H=65))                                         # 65 x 128 > 8192 columns
    mis = lambda t: t.reshape(-1)[1:]                                      # noqa: E731  2 bytes off alignment
    code(ALIGN, lambda: fwd(src=mis(p.src)))
    code(ALIGN, lambda: fwd(w=[mis(p.w[0]), p.w[1], None]))
    code(ALIGN, lambda: fwd(d=[mis(dv[0]), dv[1], dv[2]]))
    code(ALIGN, lambda: fwd(ld=p.ld + 4))
    code(ALIGN, lambda: fwd(co=p.col_off + 4))
    code(ALIGN, lambda: bwd(dxt=mis(dx)))
    code(ALIGN, lambda: bwd(dy=[mis(p.dy[0]), p.dy[1], p.dy[2]]))
    code(ALIGN, lambda: bwd(ld_dx=p.ld_dx + 2))
    code(ARG, lambda: fwd(w=p.w[:2], rope=0b100, d=dv[:2]))                # rope_mask names a missing third segment
    code(ARG, lambda: bwd(dy=p.dy[:1], w=p.w[:1], rope=0b10))
    code(ARG, lambda: fwd(d=[dv[0], None, dv[2]]))
    torch.cuda.synchronize()
    assert all(not t.any() for t in dv) and not dx.any()                   # nothing was launched


# ---------------------------------------------------------------------------------------------------------------------
# the training step at head_dim 128
# ---------------------------------------------------------------------------------------------------------------------
def _lora_grad_errors(bm, om):
    og = dict(om.named_parameters())
    errs = {}
    for n, p in bm.named_parameters():
        if "lora_" in n:
            go = og[n].grad
            assert go is not None and go.abs().max().item() > 0, n
            errs[n] = (p.grad.float().cpu() - go).abs().max().item() / go.abs().max().item()
    return errs


def _build_pair(cfg_kwargs, rank, alpha, ffn, seed=0):
    """_util.build_pair, or its feed-forward-adapter form (oracle adapters on every target, same init)."""
    if not ffn:
        return build_pair(cfg_kwargs, rank, seed=seed, alpha=alpha)
    from oracle import ltx_oracle as O
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, LORA_FFN_TARGETS
    om = O.LTXTransformerOracle(O.LTXConfig(**cfg_kwargs))
    O.add_lora(om, rank, alpha)
    for blk in om.transformer_blocks:
        blk.ff.net[0].proj = O.LoraLinear(blk.ff.net[0].proj, rank, alpha)
        blk.ff.net[2] = O.LoraLinear(blk.ff.net[2], rank, alpha)
    O.synthetic_init_(om, seed=seed, lora_b_std=0.02)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    bm = B200LTXTransformer(LTXConfig(**cfg_kwargs), torch.bfloat16, "cuda")
    bm.add_adapter(rank, alpha, target_modules=list(LORA_FFN_TARGETS))
    bm.load_state_dict(om.state_dict(), strict=True)
    bm.prepare()
    return O, om, bm


@pytest.mark.parametrize("ffn", [False, True], ids=["attn", "attn+ffn"])
@pytest.mark.parametrize("heads,rank,alpha,shape", [(2, 8, 16, (2, 2, 4, 9, 24)), (2, 64, 64, (2, 2, 4, 8, 32)),
                                                    (4, 128, 128, (2, 2, 4, 9, 24)), (3, 64, 32, (1, 3, 5, 5, 17))])
def test_small_model_step_matches_oracle_hd128(heads, rank, alpha, shape, ffn):
    """2 / 3 / 4 heads x 128, 2 blocks, ragged and 64-aligned token counts, ranks 8 / 64 / 128; the tolerances of
    test_gpu_model.py::test_small_model_step_matches_oracle."""
    cfgk = dict(SMALL128, num_attention_heads=heads, cross_attention_dim=heads * 128)
    O, om, bm = _build_pair(cfgk, rank, alpha, ffn)
    B, F, H, W, L = shape
    batch = O.make_synthetic_batch(om.cfg, B, F, H, W, text_len=L, seed=7, text_scale=1.0)
    loss_o, pred_o = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
    st, loss_b, pred_b = run_b200_micro(bm, batch)
    loss_err = abs(loss_b - loss_o.item()) / abs(loss_o.item())
    assert loss_err < 1e-3
    assert rel_err(pred_b, pred_o) < 3e-2
    og = dict(om.named_parameters())
    errs = _lora_grad_errors(bm, om)
    assert len(errs) == 2 * (10 if ffn else 8) * 2
    gmax = max(p.grad.abs().max().item() for n, p in om.named_parameters() if "lora_" in n)
    for n, e in errs.items():
        assert og[n].grad.abs().max().item() > gmax / 300, (n, og[n].grad.abs().max().item(), gmax)
        assert e < 5e-2, (n, e)
    params = [p for n, p in om.named_parameters() if "lora_" in n]
    O.clip_grad_norm_(params, 1.0)
    torch.optim.AdamW(params, lr=5e-5, betas=(0.9, 0.99), weight_decay=1e-4, eps=1e-8).step()
    st.optimizer_step()
    torch.cuda.synchronize()
    for n, p in bm.named_parameters():
        if "lora_" in n:
            assert (p.detach().float().cpu() - og[n].detach()).abs().max().item() < 2e-4, n
    print(f"\n{heads} x 128 rank {rank} alpha {alpha} ffn {ffn}: loss err {loss_err:.2e}, worst grad err "
          f"{max(errs.values()):.2e} ({max(errs, key=errs.get)})")


@pytest.mark.timeout(2400)
def test_13b_width_two_block_forward_backward_matches_oracle():
    """The 13B width (D = 4096, 32 heads x 128, S = 2688 tokens, L = 128 text keys with a ragged mask, r = 64), 2 blocks,
    B = 1: loss and every LoRA gradient against the fp32 oracle, at the shapes the 13B step's kernels run at (the
    two-chunk row kernels with three segments, head_dim-128 attention over 21 query tiles, N = 4096 / 12288 / 16384
    GEMMs).  The CPU oracle does about four times the work of the 2048-wide case."""
    from finetrainers_b200.model import LTXConfig
    cfgk = dict(LTXConfig.ltx_13b().to_dict(), num_layers=2)
    O, om, bm = build_pair(cfgk, 64, alpha=64)
    batch = O.make_synthetic_batch(om.cfg, 1, 7, 16, 24, seed=1234, text_scale=1.0)
    assert 0 < int(batch["encoder_attention_mask"].sum()) < 128
    loss_o, pred_o = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
    st, loss_b, pred_b = run_b200_micro(bm, batch)
    loss_err = abs(loss_b - loss_o.item()) / abs(loss_o.item())
    errs = _lora_grad_errors(bm, om)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    print(f"\n13B width, two blocks: loss b200 {loss_b:.6f} oracle {loss_o.item():.6f} rel {loss_err:.2e}; "
          f"pred err {rel_err(pred_b, pred_o):.2e}; grad errors (worst 4): {worst}")
    assert loss_err < 1e-3
    assert rel_err(pred_b, pred_o) < 3e-2
    assert len(errs) == 2 * 16
    for n, e in errs.items():
        assert e < 5e-2, (n, e, worst)
    og = dict(om.named_parameters())
    gb = torch.cat([p.grad.float().cpu().flatten() for n, p in bm.named_parameters() if "lora_" in n])
    go = torch.cat([og[n].grad.flatten() for n, p in bm.named_parameters() if "lora_" in n])
    assert torch.dot(gb, go) / (gb.norm() * go.norm()) > 0.999
    assert abs(gb.norm() / go.norm() - 1) < 1e-2


def _gpu_batch(cfgk, i, B=2, shape=(2, 4, 9), L=24):
    from oracle import ltx_oracle as O
    batch = O.make_synthetic_batch(O.LTXConfig(**cfgk), B, *shape, text_len=L, seed=100 + i, text_scale=1.0)
    cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(),
            "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
    lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(),
           "latents_std": batch["latents_std"].cuda()}
    return cond, lat, batch["sigmas"].view(-1).cuda(), batch["noise"].cuda()


def test_cuda_graph_step_is_bit_identical_to_eager_hd128():
    """Gradient accumulation 2, six micro-steps (three optimizer steps; the graph arm captures on its third call and
    replays after): the same loss, gradient and parameter bits as the eager arm."""
    from finetrainers_b200.trainer import SFTTrainStep
    runs = {}
    for mode in ("eager", "graph"):
        _, om, bm = build_pair(SMALL128, 64, seed=1)
        st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, use_cuda_graph=(mode == "graph"), seed=5,
                          gradient_accumulation_steps=2)
        st.spec.first_frame_conditioning_p = 0.0
        trace = []
        for i in range(6):
            cond, lat, sig, noise = _gpu_batch(SMALL128, i)
            st.train_step(cond, lat, sigmas=sig, noise=noise)
            torch.cuda.synchronize()
            trace.append((st.loss_buf.clone(), bm.lora_grad_flat.clone(), bm.lora_flat.clone()))
        assert st.opt_step == 3
        if mode == "graph":
            assert len(st._graphs) >= 1
        runs[mode] = trace
    for i, (a, b) in enumerate(zip(runs["eager"], runs["graph"])):
        for x, y, what in zip(a, b, ("loss", "grad", "param")):
            assert torch.equal(x, y), (i, what)
    assert runs["eager"][4][1].abs().max().item() > 0      # mid-accumulation (the optimizer step clears the gradient)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_layerwise_fp8_is_bit_identical_to_prerounded_bf16_hd128(graph):
    """e4m3fn storage with the CLI skip list, five blocks of 2 heads x 128 (both block slots refilled in each direction):
    the same bits as a bf16 model whose cast linears were rounded through fp8, as test_gpu_layerwise.py has at 64."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, apply_layerwise_casting
    from finetrainers_b200.trainer import SFTTrainStep
    cfgk = dict(SMALL128, num_layers=5)
    torch.manual_seed(0)
    a = B200LTXTransformer(LTXConfig(**cfgk), torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in a.named_parameters():
            p.normal_(0, 0.05) if "norm_" not in n else p.normal_(1.0, 0.1)
    b = copy.deepcopy(a)
    apply_layerwise_casting(a, torch.float8_e4m3fn, torch.bfloat16, CLI_SKIP)
    mods = dict(b.named_modules())
    with torch.no_grad():
        for n in a._lw_cfg["cast"]:
            for p in (mods[n].weight, mods[n].bias):
                p.copy_(p.to(torch.float8_e4m3fn).to(torch.bfloat16))
    for m in (a, b):
        m.add_adapter(64, 64)
        m.prepare()
    with torch.no_grad():
        a.lora_flat.normal_(0, 0.05)
        b.lora_flat.copy_(a.lora_flat)
    assert a._lw is not None and b._lw is None
    sa, sb = (SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=graph) for m in (a, b))
    for s in (sa, sb):
        s.spec.first_frame_conditioning_p = 0.0
    for i in range(4):
        cond, lat, sig, noise = _gpu_batch(cfgk, i)
        for s in (sa, sb):
            s.micro_step(dict(cond), dict(lat), sigmas=sig, noise=noise)
        torch.cuda.synchronize()
        assert torch.equal(sa.loss_buf, sb.loss_buf), i
        assert a.lora_grad_flat.abs().max().item() > 0
        assert torch.equal(a.lora_grad_flat, b.lora_grad_flat), i
        sa.optimizer_step()
        sb.optimizer_step()
        torch.cuda.synchronize()
        assert torch.equal(a.lora_flat, b.lora_flat), i
    assert a.transformer_blocks[3].attn1.to_q.base_layer.weight.dtype == torch.float8_e4m3fn


@pytest.mark.timeout(1800)
def test_13b_geometry_runs_and_repeats():
    """The whole 13B geometry (48 blocks, B = 1, 2688 tokens, r = 64), two seeded runs of 3 optimizer steps each: finite
    loss and gradient norm, the two runs bit-identical, peak memory below 70 GB.  There is no oracle at this size (its
    fp32 weights alone are 52 GB): this checks that the step runs, fits and repeats, not what it computes - the
    two-block test above does that at the same width."""
    import gc
    import random
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    from finetrainers_b200.trainer import SFTTrainStep
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 70e9:
        pytest.skip(f"needs 70 GB of free device memory, {free / 1e9:.1f} GB are free")
    cfg = LTXConfig.ltx_13b()

    def run():
        torch.manual_seed(0)
        random.seed(0)          # the step draws its first-frame-conditioning coin from Python's generator
        m = B200LTXTransformer(cfg, torch.bfloat16, "cuda")
        with torch.no_grad():
            for n, p in m.named_parameters():
                if "scale_shift_table" in n:
                    p.normal_(0, 1.0 / p.shape[-1] ** 0.5)
                elif "norm_q" in n or "norm_k" in n:
                    p.fill_(1.0)
                else:
                    p.normal_(0, 0.02)
        m.add_adapter(64, 64)
        m.prepare()
        with torch.no_grad():
            m.lora_flat.normal_(0, 0.01)       # non-zero B: every adapter gradient is non-trivial
        st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)
        g = torch.Generator().manual_seed(1234)
        lat = torch.randn(1, 128, 7, 16, 24, generator=g).bfloat16().cuda()
        ehs = (torch.randn(1, 128, 4096, generator=g) * 0.1).bfloat16().cuda()
        mask = (torch.arange(128)[None] < 100).cuda()
        mean, std = torch.zeros(1, 128, device="cuda"), torch.ones(1, 128, device="cuda")
        out = []
        for _ in range(3):
            st.train_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                          {"latents": lat, "latents_mean": mean, "latents_std": std})
            torch.cuda.synchronize()
            out.append((st.metrics[1].item(), st.metrics[0].item()))
        return out, m.lora_flat.clone()

    torch.cuda.reset_peak_memory_stats()
    m0, p0 = run()
    peak = torch.cuda.max_memory_allocated()
    gc.collect()
    torch.cuda.empty_cache()
    m1, p1 = run()
    print(f"\n13B geometry: (loss, grad norm) per step {m0}; max_memory_allocated {peak / 1e9:.2f} GB")
    for loss, gn in m0:
        assert loss == loss and abs(loss) < float("inf") and loss > 0
        assert gn == gn and 0 < gn < float("inf")
    assert m0 == m1
    assert torch.equal(p0, p1)
    assert peak < 70e9
