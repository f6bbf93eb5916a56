"""Elementwise kernel conformance: every entry point of b2d_elem.cu against an fp64 reference computed on the GPU from
the same bf16 / fp32 inputs, with the outputs inside sentinel buffers and the inputs a kernel must not read poisoned.

Every check has three parts: each element against the fp64 reference under the bound below; every element of an
output buffer outside the output window keeps the sentinel bit pattern (_util.sentinel_buffer); and every input element
the kernel must not read (unused temb chunks and table rows, source columns outside the segment window, table rows past
S, weight elements past D) holds NaN, so that reading one turns an output into NaN, which check_bound rejects.

Bounds (ulp16 / ulp32 = bf16 / fp32 spacing at the reference value; "rowmax" = the largest magnitude in the row):
  A  norm_modulate fwd:  ulp16(ref) + 2^-16 * rowmax(|xhat (1 + scale)| + |shift|)
     norm_modulate bwd:  ulp16(ref) + 2^-16 * (|dx_in| + rstd * rowmax|g| * (1 + rowmax|xhat|)^2),  g = dy (1 + scale)
     out2, colscale:     ulp16(ref) + 2^-22 |ref|  (two fp32 roundings of a product of bf16 values)
     The fp32 row statistics (a per-thread serial sum, then a warp and a block tree) carry a relative error below
     2^-18 for D <= 8192; the final mean / variance / g - xhat * mean(g xhat) steps scale it by at most the terms named.
  B  q/k fwd:  ulp16(ref) + 2^-16 * 2 rowmax|n|                 (n = the normalized, unrotated segment row)
     q/k bwd:  ulp16(ref) + 2^-16 * rstd * rowmax|g| * (1 + rowmax|xhat|)^2,  g = rope^T(dy) * w  (2 rowmax|dy| unnormed)
  C  rope_table: |cos - cos64|, |sin - sin64| <= 32 * (ulp32(fr) |2g - 1| + fr ulp32(g)) + ulp32(1), where fr is the
     frequency * pi/2 and g the grid coordinate.  Derivation: lin = fi / (nf - 1) is evaluated in fp32 with two
     roundings (|d lin| <= 2^-23), and powf adds 2 ulp, so fr carries a relative error <= ln(1e4) 2^-23 + 3 * 2^-24 <=
     24 ulp32(fr) / fr; g = f * sf is one rounding (ulp32(g) / 2), 2g - 1 is exact (Sterbenz) or rounds by at most
     2^-25 <= ulp32(fr) |2g - 1| / fr when |2g - 1| >= 1/2; the product fr * (2g - 1) rounds by ulp32(ang) / 2; sinf /
     cosf (full range reduction, no fast math) add <= 2 ulp32(1).  32 covers the sum.
  D  loss:      L * 2^-24 * loss64 with L = 8 * ceil(B * per_sample / (8 * 296 * 256)) + 40: the additions along the
                longest path of the reduction tree (8 terms per grid-stride step per thread, a warp tree of 5, a block
                tree of 5 + 3, the 296 partials: 2 serial + 5 + 3), plus the roundings of each term and of 1 / (n B).
                All terms are non-negative, so each rounding is relative to the total.
     dpred:     ulp16(ref) + 2^-20 |ref|
     sumsq:     L * 2^-24 * (out0 + sum x^2) with L = 4 * ceil(n / (4 * 296 * 256)) + 40, the same tree with 4 terms
                per step, plus the += of the previous value.
     sinusoid:  ulp16(ref) + 12 * 2^-23 * |t * freq| + 2^-23: the fp32 freq = expf(c * i / 128) is off by at most
                (9.21 + 2) 2^-23 relative, and t * freq rounds once; one bf16 ulp covers the final rounding.
     adamw:     m, v: 2 ulp32 + 2^-18 * (|b m| + |(1 - b) g'|), the magnitudes of their two terms (m may cancel);
                p: 2 ulp32(p) + 2^-18 * lr / bc1 * (|b1 m| + |(1 - b1) g'|) / denom, the update at that scale.
     cast, prep_noise_pack: bit-exact (NaN inputs: NaN outputs).

The worst error / bound ratio of each part is printed at the end of the module (pytest -s).  Measured on an H100 80GB
HBM3 at a 400 W power limit: every bf16 output 0.50 or just below (its own rounding: the fp32 arithmetic is far inside
the 2^-16 terms), rope_table 0.19 (oracle 0.19), adamw 0.72, loss 0.025, sumsq 0.024.
"""
import math

import pytest
import torch

from _util import bf16_ulp, check_bound, check_sentinel, f32_ulp, sentinel_buffer, window

pytestmark = pytest.mark.gpu

NAN = float("nan")
PAD = 64            # sentinel elements on each side of an output window
REDUCE = 296        # B2D_REDUCE_PARTIALS


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


WORST = {}   # part -> worst error / bound ratio seen in this run (printed at the end of the module)


def _bound(part, got, ref, bound, what):
    r = check_bound(got, ref, bound, what)
    WORST[part] = max(WORST.get(part, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst error/bound ratio per part:", {k: round(v, 4) for k, v in sorted(WORST.items())})


def _raises_code(code, fn):
    from finetrainers_b200.lib import B2DError
    with pytest.raises(B2DError, match=rf"\(code {code}\)"):
        fn()


def _bits(t):
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _same_bits(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), what


class Guarded:
    """An output of `n` elements inside a sentinel-filled buffer with PAD elements of margin on each side; `shift`
    elements move the window off the buffer's 16-byte alignment."""

    def __init__(self, n, dtype=torch.bfloat16, shift=0):
        self.n, self.off = n, PAD + shift
        self.buf = sentinel_buffer(n + 2 * PAD + shift, dtype)
        self.t = self.buf[self.off:self.off + n]

    def view(self, *shape):
        return self.t.view(*shape)

    def check(self, what, wins=None):
        """Only `wins` (default: the whole window) may have changed."""
        if wins is None:
            wins = [window(self.buf, self.off, 1, self.n, self.n)] if self.n else []
        check_sentinel(self.buf, wins, what)


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


# ---------------------------------------------------------------------------------------------------------------------
# A. norm_modulate_fwd / bwd, colscale
# ---------------------------------------------------------------------------------------------------------------------
def _rows_with_edges(g, R, D):
    """Random rows, with the statistics edges in rows 1-3: a large common offset next to the spread (mean 32, std 1), a
    constant row (LN variance 0: eps decides), and rows small enough that eps matters for RMS (|x| ~ 1e-4)."""
    x = torch.randn(R, D, device="cuda", generator=g)
    x[1] = 32 + torch.randn(D, device="cuda", generator=g)
    x[2] = 0.75
    x[3] = 1e-4 * torch.randn(D, device="cuda", generator=g)
    return x.bfloat16()


def _temb(g, nb, D, chunks, stride=None):
    """[nb, stride] with stride = 6 D by default: only the listed D-wide chunks hold values, the rest NaN."""
    t = torch.full((nb, stride or 6 * D), NAN, device="cuda", dtype=torch.bfloat16)
    for c in chunks:
        t[:, c * D:(c + 1) * D] = _rnd(g, nb, D, scale=0.3)
    return t


def _table(g, D, rows):
    tab = torch.full((6, D), NAN, device="cuda", dtype=torch.bfloat16)
    for r in rows:
        tab[r] = _rnd(g, D, scale=0.3)
    return tab


def _norm64(x, ln, eps):
    xc = x - x.mean(-1, keepdim=True) if ln else x
    return xc * torch.rsqrt((xc * xc).mean(-1, keepdim=True) + eps)


def _rowmax(t):
    return t.abs().amax(-1, keepdim=True)


def _norm_modulate_case(ops, R, D, rps, ln, eps=1e-6, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    nb = R // rps
    b = torch.arange(R, device="cuda") // rps
    x = _rows_with_edges(g, R, D)
    # forward: shift / scale from table rows 3 / 4 and temb chunks 3 / 4 (the FFN norm); everything else is NaN
    tab, temb = _table(g, D, (3, 4)), _temb(g, nb, D, (3, 4))
    row = lambda i, tb, te: tb[i].double()[None] + te[:, i * D:(i + 1) * D].double()[b]
    y = Guarded(R * D)
    ops.norm_modulate_fwd(x, y.view(R, D), tab[3], temb[:, 3 * D:], tab[4], temb[:, 4 * D:], 6 * D, R, D, rps, eps, ln)
    xd = x.double().requires_grad_(True)
    xhat = _norm64(xd, ln, eps)
    shift, scale = row(3, tab, temb), row(4, tab, temb)
    ref = xhat * (1 + scale) + shift
    r = ref.detach()
    _bound("A norm_modulate_fwd", y.view(R, D), r,
           bf16_ulp(r) + 2.0 ** -16 * _rowmax(xhat.detach().abs() * (1 + scale).abs() + shift.abs()), f"fwd D={D} ln={ln}")
    y.check("norm_modulate_fwd y")

    # backward: scale from row / chunk 1, gate2 from row / chunk 5 (the attention norm); everything else NaN
    tab, temb = _table(g, D, (1, 5)), _temb(g, nb, D, (1, 5))
    xd = x.double().requires_grad_(True)
    xhat = _norm64(xd, ln, eps)
    scale, gate2 = row(1, tab, temb), row(5, tab, temb)
    dy, dxin = _rnd(g, R, D), _rnd(g, R, D)
    (xhat * (1 + scale)).backward(dy.double())
    gd = dy.double() * (1 + scale)
    xc = xd.detach() - xd.detach().mean(-1, keepdim=True) if ln else xd.detach()
    rstd = torch.rsqrt((xc * xc).mean(-1, keepdim=True) + eps)
    scl = rstd * _rowmax(gd) * (1 + _rowmax(xhat.detach())) ** 2
    grad = xd.grad
    dx, o2 = Guarded(R * D), Guarded(R * D)
    ops.norm_modulate_bwd(dy, x, dxin, dx.view(R, D), tab[1], temb[:, D:], 6 * D, R, D, rps, eps, ln, gate2_tab=tab[5],
                          gate2_emb=temb[:, 5 * D:], out2=o2.view(R, D))
    refdx = dxin.double() + grad
    _bound("A norm_modulate_bwd", dx.view(R, D), refdx, bf16_ulp(refdx) + 2.0 ** -16 * (dxin.double().abs() + scl),
           f"bwd D={D} ln={ln}")
    ref2 = dx.view(R, D).double() * gate2
    _bound("A norm_modulate_bwd out2", o2.view(R, D), ref2, bf16_ulp(ref2) + 2.0 ** -22 * ref2.abs(), f"out2 D={D}")
    dx.check("norm_modulate_bwd dx")
    o2.check("norm_modulate_bwd out2")
    # in place (dx_in == dx_out, as the attention-norm backward runs): the same bits as out of place
    inpl = dxin.clone()
    ops.norm_modulate_bwd(dy, x, inpl, inpl, tab[1], temb[:, D:], 6 * D, R, D, rps, eps, ln, gate2_tab=tab[5],
                          gate2_emb=temb[:, 5 * D:], out2=o2.view(R, D))
    _same_bits(inpl, dx.view(R, D), f"in-place bwd D={D}")
    # dx_in = NULL, no out2
    dx0 = Guarded(R * D)
    ops.norm_modulate_bwd(dy, x, None, dx0.view(R, D), tab[1], temb[:, D:], 6 * D, R, D, rps, eps, ln)
    _bound("A norm_modulate_bwd", dx0.view(R, D), grad, bf16_ulp(grad) + 2.0 ** -16 * scl, f"bwd dx_in=NULL D={D}")
    dx0.check("norm_modulate_bwd dx (dx_in = NULL)")


@pytest.mark.parametrize("rps", [5, 1])
@pytest.mark.parametrize("ln", [0, 1])
@pytest.mark.parametrize("D", [8, 72, 2048, 2056, 4104, 6144, 8192])
def test_norm_modulate(ops, D, ln, rps):
    """Every ROW_DISPATCH instantiation: 1 chunk (D = 8, 72, 2048), 2 chunks (2056, 4104), the 3-chunk width that runs
    the 4-chunk kernel (6144) and 4 chunks (8192); four samples of 5 rows, or one row per sample."""
    _norm_modulate_case(ops, 4 * rps, D, rps, ln, seed=D + ln)


@pytest.mark.parametrize("R", [2688, 5376])
def test_norm_modulate_step_shapes(ops, R):
    _norm_modulate_case(ops, R, 2048, 2688, 0, seed=R)


@pytest.mark.parametrize("D", [72, 2048])
def test_norm_modulate_final_layer_form(ops, D):
    """The output head's call form: shift and scale both come from the same [B, D] embedding (shift_emb == scale_emb,
    emb_stride = D), table rows 0 and 1, LayerNorm with eps 1e-6; forward and backward (dx_in = NULL)."""
    g = torch.Generator(device="cuda").manual_seed(D)
    nb, rps, eps = 3, 7, 1e-6
    R = nb * rps
    b = torch.arange(R, device="cuda") // rps
    x = _rows_with_edges(g, R, D)
    tab = _table(g, D, (0, 1))
    emb = _rnd(g, nb, D, scale=0.3)
    y = Guarded(R * D)
    ops.norm_modulate_fwd(x, y.view(R, D), tab[0], emb, tab[1], emb, D, R, D, rps, eps, True)
    xd = x.double().requires_grad_(True)
    xhat = _norm64(xd, True, eps)
    shift, scale = tab[0].double()[None] + emb.double()[b], tab[1].double()[None] + emb.double()[b]
    r = (xhat * (1 + scale) + shift).detach()
    _bound("A norm_modulate_fwd", y.view(R, D), r,
           bf16_ulp(r) + 2.0 ** -16 * _rowmax(xhat.detach().abs() * (1 + scale).abs() + shift.abs()), "final fwd")
    y.check("final-layer fwd")
    dy = _rnd(g, R, D)
    (xhat * (1 + scale)).backward(dy.double())
    xc = xd.detach() - xd.detach().mean(-1, keepdim=True)
    rstd = torch.rsqrt((xc * xc).mean(-1, keepdim=True) + eps)
    scl = rstd * _rowmax(dy.double() * (1 + scale)) * (1 + _rowmax(xhat.detach())) ** 2
    dx = Guarded(R * D)
    ops.norm_modulate_bwd(dy, x, None, dx.view(R, D), tab[1], emb, D, R, D, rps, eps, True)
    _bound("A norm_modulate_bwd", dx.view(R, D), xd.grad, bf16_ulp(xd.grad) + 2.0 ** -16 * scl, "final bwd")
    dx.check("final-layer bwd")


@pytest.mark.parametrize("D,rps", [(8, 5), (72, 1), (2056, 3), (2048, 2688)])
def test_colscale(ops, D, rps):
    """out = x * (tab[c] + emb[b, c]) with emb_stride != D and != 6 D; unused table rows and temb chunks are NaN."""
    g = torch.Generator(device="cuda").manual_seed(D)
    nb = 3 if rps < 100 else 2
    R = nb * rps
    x = _rnd(g, R, D)
    es = 6 * D + 8
    tab, temb = _table(g, D, (5,)), _temb(g, nb, D, (5,), stride=es)
    out = Guarded(R * D)
    ops.colscale(x, out.view(R, D), tab[5], temb[:, 5 * D:], es, R, D, rps)
    b = torch.arange(R, device="cuda") // rps
    ref = x.double() * (tab[5].double()[None] + temb[:, 5 * D:6 * D].double()[b])
    _bound("A colscale", out.view(R, D), ref, bf16_ulp(ref) + 2.0 ** -22 * ref.abs(), f"colscale D={D}")
    out.check("colscale out")


# ---------------------------------------------------------------------------------------------------------------------
# B. qkv_norm_rope_fwd / bwd and qknorm_rope_fwd / bwd
# ---------------------------------------------------------------------------------------------------------------------
class QkvProblem:
    """Packed rows [B*S, ld] whose nseg D-wide segments start at col_off; every other column is NaN.  Random angles give
    the (cos, sin) tables [S, D/2] (plus one NaN row past S); weights are [D] followed by D NaN elements, or stacked per
    block with stride w_stride when rows_per_w > 0."""

    def __init__(self, B, S, H, nseg, wmask, rope, col_off=24, ld_extra=40, dx_col_off=16, ld_dx_extra=88,
                 rows_per_w=0, w_stride=0, eps=1e-5, seed=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.B, self.S, self.H, self.nseg, self.wmask, self.rope, self.eps = B, S, H, nseg, wmask, rope, eps
        self.D = D = H * 64
        self.rows = rows = B * S
        self.col_off, self.ld = col_off, col_off + nseg * D + ld_extra
        self.dx_col_off, self.ld_dx = dx_col_off, dx_col_off + nseg * D + ld_dx_extra
        self.rows_per_w, self.w_stride = rows_per_w, w_stride
        self.src = torch.full((rows, self.ld), NAN, device="cuda", dtype=torch.bfloat16)
        self.src[:, col_off:col_off + nseg * D] = _rnd(g, rows, nseg * D)
        ang = torch.randn(S + 1, D // 2, device="cuda", generator=g) * 3
        self.cos, self.sin = ang.cos(), ang.sin()
        self.cos[S], self.sin[S] = NAN, NAN
        nblk = rows // rows_per_w if rows_per_w else 1
        self.w = []
        for i in range(nseg):
            if not (wmask >> i) & 1:
                self.w.append(None)
                continue
            if rows_per_w:
                w = torch.full((nblk * w_stride + D,), NAN, device="cuda", dtype=torch.bfloat16)
                for k in range(nblk):
                    w[k * w_stride:k * w_stride + D] = (1 + 0.2 * torch.randn(D, device="cuda", generator=g)).bfloat16()
            else:
                w = torch.full((2 * D,), NAN, device="cuda", dtype=torch.bfloat16)
                w[:D] = (1 + 0.2 * torch.randn(D, device="cuda", generator=g)).bfloat16()
            self.w.append(w)
        self.dy = [_rnd(g, B, H, S, 64) for _ in range(nseg)]

    def seg(self, i):
        return self.src[:, self.col_off + i * self.D:self.col_off + (i + 1) * self.D]

    def weight_rows(self, i):
        """[rows, D] fp64 weights of segment i (per-block when stacked)."""
        w, D = self.w[i], self.D
        if not self.rows_per_w:
            return w[:D].double()[None].expand(self.rows, D)
        blk = torch.arange(self.rows, device="cuda") // self.rows_per_w
        return torch.stack([w[k * self.w_stride:k * self.w_stride + D] for k in range(int(blk.max()) + 1)]).double()[blk]

    def heads(self, t):  # [rows, D] -> [B, H, S, 64]
        return t.reshape(self.B, self.S, self.H, 64).transpose(1, 2)

    def rows_of(self, t):  # [B, H, S, 64] -> [rows, D]
        return t.transpose(1, 2).reshape(self.rows, self.D)

    def tables(self):
        return (self.cos, self.sin) if self.rope else (None, None)

    def reference(self, i):
        """(fwd ref [B,H,S,64], dx ref [rows, D], fwd bound, dx bound) of segment i, fp64 with autograd."""
        x = self.seg(i).double().requires_grad_(True)
        n = x
        s_idx = torch.arange(self.rows, device="cuda") % self.S
        norm = self.w[i] is not None
        if norm:
            rstd = torch.rsqrt((x * x).mean(-1, keepdim=True) + self.eps)
            n = x * rstd * self.weight_rows(i)
        o = n
        if (self.rope >> i) & 1:
            c, s = self.cos[:self.S].double()[s_idx], self.sin[:self.S].double()[s_idx]
            a, b = n.unflatten(-1, (-1, 2)).unbind(-1)
            o = torch.stack([a * c - b * s, b * c + a * s], -1).flatten(-2)
        fwd = self.heads(o)
        fwd.backward(self.dy[i].double())
        f = fwd.detach()
        fb = bf16_ulp(f) + 2.0 ** -16 * 2 * self.heads(_rowmax(n.detach()).expand(-1, self.D))
        dx = x.grad
        if norm:
            dyr = self.rows_of(self.dy[i].double())
            if (self.rope >> i) & 1:
                a, b = dyr.unflatten(-1, (-1, 2)).unbind(-1)
                dyr = torch.stack([a * c + b * s, b * c - a * s], -1).flatten(-2)
            gw = dyr * self.weight_rows(i)
            xhat = x.detach() * rstd.detach()
            scl = rstd.detach() * _rowmax(gw) * (1 + _rowmax(xhat)) ** 2
        else:
            scl = 2 * _rowmax(self.rows_of(self.dy[i].double()))
        return f, dx, fb, bf16_ulp(dx) + 2.0 ** -16 * scl

    def run_fwd(self, ops):
        n = self.B * self.H * self.S * 64
        dsts = [Guarded(n) for _ in range(self.nseg)]
        c, s = self.tables()
        ops.qkv_norm_rope_fwd(self.src, self.ld, self.col_off, self.w, self.rope, c, s,
                              [d.view(self.B, self.H, self.S, 64) for d in dsts], self.B, self.S, self.H, self.eps,
                              rows_per_w=self.rows_per_w, w_stride=self.w_stride)
        return dsts

    def run_bwd(self, ops):
        dx = Guarded(self.rows * self.ld_dx)
        c, s = self.tables()
        ops.qkv_norm_rope_bwd(self.dy, self.src, self.ld, self.col_off, self.w, self.rope, c, s,
                              dx.view(self.rows, self.ld_dx), self.ld_dx, self.dx_col_off, self.B, self.S, self.H,
                              self.eps, rows_per_w=self.rows_per_w, w_stride=self.w_stride)
        return dx

    def dx_window(self, dx):
        return window(dx.buf, dx.off + self.dx_col_off, self.rows, self.nseg * self.D, self.ld_dx)

    def check(self, ops, what):
        dsts, dx = self.run_fwd(ops), self.run_bwd(ops)
        dxw = self.dx_window(dx)
        for i in range(self.nseg):
            f, gx, fb, gb = self.reference(i)
            out = dsts[i].view(self.B, self.H, self.S, 64)
            dxi = dxw[:, i * self.D:(i + 1) * self.D]
            tag = f"{what} seg {i} (w {self.wmask:03b}, rope {self.rope:03b})"
            _bound("B qk fwd", out, f, fb, tag + " fwd")
            _bound("B qk bwd", dxi, gx, gb, tag + " bwd")
            if self.w[i] is None and not (self.rope >> i) & 1:   # neither norm nor rope: a copy both ways
                _same_bits(out, self.heads(self.seg(i)), tag + " fwd copy")
                _same_bits(dxi, self.rows_of(self.dy[i]), tag + " bwd copy")
            dsts[i].check(tag + " dst")
        dx.check(what + " dx", [dxw])
        return dsts, dx


@pytest.mark.parametrize("nseg", [1, 2, 3])
@pytest.mark.parametrize("H", [1, 2])
def test_qkv_every_combination(ops, H, nseg):
    """Every weight present / absent per segment x every rope_mask in 0 .. 2^nseg - 1 (the third segment's own norm
    reduction, rotated-but-unnormalized segments, ...), B = 2, S = 7."""
    for wmask in range(1 << nseg):
        for rope in range(1 << nseg):
            QkvProblem(2, 7, H, nseg, wmask, rope, seed=wmask * 8 + rope).check(ops, f"H={H} nseg={nseg}")


# a subset that still has every segment normed and not, rotated and not, and the third segment's norm with and without
# the first two
SUBSET = [(3, 0b011, 0b011), (3, 0b100, 0b100), (3, 0b101, 0b010), (3, 0b111, 0b111), (3, 0b000, 0b000),
          (2, 0b10, 0b01), (1, 0b1, 0b1)]


@pytest.mark.parametrize("S", [7, 129])
@pytest.mark.parametrize("H", [32, 33, 65, 128])
def test_qkv_heads(ops, H, S):
    """Every head count class: 1 chunk (32), 2 chunks (33), the 3-chunk width that runs the 4-chunk kernel (65), 4 chunks
    (128)."""
    for nseg, wmask, rope in SUBSET:
        QkvProblem(2, S, H, nseg, wmask, rope, seed=H + S + wmask).check(ops, f"H={H} S={S} nseg={nseg}")


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("rope", [False, True])
@pytest.mark.parametrize("H", [2, 33])
def test_qknorm_single_segment_equals_qkv(ops, H, norm, rope):
    """ops.qknorm_rope_fwd / bwd (one segment, normed iff ``norm``, rotated iff tables are passed) give the same bits as
    the nseg = 1 call of ops.qkv_norm_rope_*."""
    p = QkvProblem(3, 7, H, 1, int(norm), int(rope), seed=H)
    dsts, dx = p.run_fwd(ops), p.run_bwd(ops)
    c, s = p.tables()
    w = p.w[0]
    dst = Guarded(p.B * p.H * p.S * 64)
    ops.qknorm_rope_fwd(p.src, p.ld, p.col_off, w, c, s, dst.view(p.B, p.H, p.S, 64), p.B, p.S, p.H, norm, p.eps)
    _same_bits(dst.t, dsts[0].t, "qknorm_rope_fwd")
    dst.check("qknorm_rope_fwd dst")
    dx1 = Guarded(p.rows * p.ld_dx)
    ops.qknorm_rope_bwd(p.dy[0], p.src, p.ld, p.col_off, w, c, s, dx1.view(p.rows, p.ld_dx), p.ld_dx, p.dx_col_off,
                        p.B, p.S, p.H, norm, p.eps)
    _same_bits(dx1.buf, dx.buf, "qknorm_rope_bwd")


def test_qkv_stacked_weights_with_rope(ops):
    """rows_per_w > 0 (two blocks of 2 x 7 rows, w_stride != D) with a rotated normed segment, a normed unrotated one and
    a rotated copy; rows_per_w = rows gives the same bits as rows_per_w = 0."""
    p = QkvProblem(4, 7, 2, 3, 0b011, 0b101, rows_per_w=14, w_stride=2 * 64 + 24, seed=11)
    p.check(ops, "stacked")
    q = QkvProblem(2, 7, 2, 3, 0b111, 0b011, seed=12)
    dsts0, dx0 = q.run_fwd(ops), q.run_bwd(ops)
    q.rows_per_w, q.w_stride = q.rows, 8
    dsts1, dx1 = q.run_fwd(ops), q.run_bwd(ops)
    for a, b in zip(dsts0, dsts1):
        _same_bits(a.buf, b.buf, "rows_per_w = rows fwd")
    _same_bits(dx0.buf, dx1.buf, "rows_per_w = rows bwd")


def test_qkv_step_shapes(ops):
    """The training step's three call forms at D = 2048: q|k|v of one sample with mask 0b011 at S = 2688; the text-side
    k|v of 28 stacked blocks x L = 128 (k normed with per-block weights, v copied); q2 alone, normed, no RoPE."""
    QkvProblem(1, 2688, 32, 3, 0b011, 0b011, col_off=0, ld_extra=0, dx_col_off=0, ld_dx_extra=0, seed=1).check(ops, "qkv")
    QkvProblem(28, 128, 32, 2, 0b01, 0, col_off=0, ld_extra=0, dx_col_off=0, ld_dx_extra=0, rows_per_w=128,
               w_stride=2048, seed=2).check(ops, "text k|v")
    QkvProblem(1, 2688, 32, 1, 0b1, 0, col_off=0, ld_extra=0, dx_col_off=0, ld_dx_extra=0, seed=3).check(ops, "q2")


# ---------------------------------------------------------------------------------------------------------------------
# C. rope_table
# ---------------------------------------------------------------------------------------------------------------------
def _rope64(F, H, W, D, sf, sh, sw):
    """diffusers LTXVideoRotaryPosEmbed in fp64 from the fp32 scales: (cos, sin [S, D/2], bound [S, D/2])."""
    nf, pad = D // 6, D % 6
    s32 = torch.tensor([sf, sh, sw], dtype=torch.float32).double()
    f, h, w = torch.meshgrid(torch.arange(F), torch.arange(H), torch.arange(W), indexing="ij")
    grid = torch.stack([f, h, w], -1).reshape(-1, 3).double().cuda() * s32.cuda()           # [S, 3]
    fr = 10000.0 ** (torch.arange(nf, dtype=torch.float64, device="cuda") / (nf - 1)) * (math.pi / 2)
    ang = (fr[None, None, :] * (2 * grid[:, :, None] - 1)).transpose(1, 2).reshape(-1, 3 * nf)   # freq-major, then f,h,w
    g32 = grid.float().double()
    bound = 32 * (f32_ulp(fr)[None, None, :] * (2 * g32[:, :, None] - 1).abs() + fr[None, None, :] * f32_ulp(g32)[:, :, None])
    bound = bound.transpose(1, 2).reshape(-1, 3 * nf) + 2.0 ** -23
    S = F * H * W
    cos = torch.cat([torch.ones(S, pad // 2, dtype=torch.float64, device="cuda"), ang.cos()], 1)
    sin = torch.cat([torch.zeros(S, pad // 2, dtype=torch.float64, device="cuda"), ang.sin()], 1)
    bound = torch.cat([torch.zeros(S, pad // 2, dtype=torch.float64, device="cuda"), bound], 1)
    return cos, sin, bound


@pytest.mark.parametrize("F,H,W", [(7, 16, 24), (1, 5, 9), (3, 1, 4), (2, 6, 1)])
@pytest.mark.parametrize("D", [1536, 2048, 256])
def test_rope_table(ops, F, H, W, D):
    """D with 0, 2 and 4 pad columns; F, H or W equal to 1; non-square grids.  Pad pairs are exactly (1, 0).  The oracle
    (fp32, the reference's op order) obeys the same bound against fp64, so kernel and oracle agree within the sum of
    the two."""
    from oracle.ltx_oracle import ltx_rope_table
    sf, sh, sw = (8 / 25) / 20, 32 / 2048, 32 / 2048
    S, P = F * H * W, D // 2
    cos, sin = Guarded(S * P, torch.float32), Guarded(S * P, torch.float32)
    ops.rope_table(cos.t, sin.t, F, H, W, D, sf, sh, sw)
    cos.check("rope cos")
    sin.check("rope sin")
    c, s = cos.view(S, P), sin.view(S, P)
    c64, s64, bnd = _rope64(F, H, W, D, sf, sh, sw)
    pad = (D % 6) // 2
    assert torch.equal(c[:, :pad], torch.ones_like(c[:, :pad])) and torch.equal(s[:, :pad], torch.zeros_like(s[:, :pad]))
    _bound("C rope_table", c[:, pad:], c64[:, pad:], bnd[:, pad:], f"cos D={D}")
    _bound("C rope_table", s[:, pad:], s64[:, pad:], bnd[:, pad:], f"sin D={D}")
    rc, rs = ltx_rope_table(F, H, W, D, [8 / 25, 32, 32], 1, "cpu")
    rc, rs = rc[0][:, 0::2].cuda(), rs[0][:, 0::2].cuda()
    _bound("C rope_table oracle", rc[:, pad:], c64[:, pad:], bnd[:, pad:], f"oracle cos D={D}")
    _bound("C rope_table oracle", rs[:, pad:], s64[:, pad:], bnd[:, pad:], f"oracle sin D={D}")
    check_bound(c[:, pad:], rc[:, pad:], 2 * bnd[:, pad:], "kernel vs oracle cos")
    check_bound(s[:, pad:], rs[:, pad:], 2 * bnd[:, pad:], "kernel vs oracle sin")
    assert torch.equal(rc[:, :pad], c[:, :pad]) and torch.equal(rs[:, :pad], s[:, :pad])


# ---------------------------------------------------------------------------------------------------------------------
# D. step satellites
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,C,F,HW", [(3, 3, 1, 1), (3, 3, 2, 5), (1, 16, 1, 7), (2, 128, 3, 33)])
@pytest.mark.parametrize("first_frame", [False, True])
def test_prep_noise_pack(ops, B, C, F, HW, first_frame):
    """Bit-exact against the oracle's normalize / flow-match / pack, with sigma 0 and 1 among the samples and sigma_ff
    NULL or set; x_t and target inside sentinel buffers."""
    from oracle.ltx_oracle import flow_match_target, flow_match_xt, normalize_latents, pack_latents
    g = torch.Generator().manual_seed(B * 1000 + C + F + HW)
    lat, noise = torch.randn(B, C, F, 1, HW, generator=g).bfloat16(), torch.randn(B, C, F, 1, HW, generator=g).bfloat16()
    mean, std = torch.randn(B, C, generator=g), torch.rand(B, C, generator=g) + 0.5
    sig = torch.tensor([0.0, 1.0, 0.37, 0.81, 0.05][:B]) if B > 1 else torch.tensor([1.0])
    sff = torch.rand(B, generator=g) * 0.25 if first_frame else None
    n = B * F * HW * C
    xt, tg = Guarded(n), Guarded(n)
    ops.prep_noise_pack(lat.cuda(), noise.cuda(), mean.cuda(), std.cuda(), sig.cuda(),
                        sff.cuda() if first_frame else None, xt.t, tg.t, B, C, F, HW)
    x0 = normalize_latents(lat, mean, std)
    v = lambda s: s.view(B, 1, 1, 1, 1)
    if first_frame:
        noisy = torch.cat([flow_match_xt(x0[:, :, :1], noise[:, :, :1], v(sff)),
                           flow_match_xt(x0[:, :, 1:], noise[:, :, 1:], v(sig))], dim=2)
    else:
        noisy = flow_match_xt(x0, noise, v(sig))
    _same_bits(xt.t.cpu(), pack_latents(noisy).bfloat16().reshape(-1), "x_t")
    _same_bits(tg.t.cpu(), pack_latents(flow_match_target(noise, x0)).bfloat16().reshape(-1), "target")
    xt.check("x_t")
    tg.check("target")


def _loss_run(ops, pred, tg, wgt, ls, with_dpred, B, per):
    loss, ws = Guarded(1, torch.float32), Guarded(1024, torch.float32)
    dp = Guarded(B * per) if with_dpred else None
    ops.loss_mse(pred, tg, wgt, ls, loss.t, dp.t if dp else None, ws.t, B, per)
    loss.check("loss_out")
    ws.check("partial_ws", [window(ws.buf, PAD, 1, REDUCE, REDUCE)])
    if dp:
        dp.check("dpred")
    return loss.t.clone(), dp.t.clone() if dp else None


@pytest.mark.parametrize("B,per", [(1, 8), (2, 40 * 128), (3, 1000), (4, 64), (5, 2688 * 128), (2, 2688 * 128)])
def test_loss_mse(ops, B, per):
    """B = 1 .. 5; per_sample from one 8-vector to one where the grid-stride loop wraps several times; weight NULL or
    per sample, dpred NULL or written; two launches give the same bits; partial_ws beyond its 296 floats untouched."""
    g = torch.Generator(device="cuda").manual_seed(B * per)
    pred, tg = _rnd(g, B * per), _rnd(g, B * per)
    wgt, ls = torch.rand(B, device="cuda", generator=g) * 3, 0.37
    d = pred.double().view(B, per) - tg.double().view(B, per)
    iters = -(-(B * per // 8) // (REDUCE * 256))
    L = 8 * iters + 40
    for w in (wgt, None):
        w64 = w.double()[:, None] if w is not None else 1.0
        ref = (w64 * d * d).mean(1).mean() * ls
        loss, dp = _loss_run(ops, pred, tg, w, ls, True, B, per)
        _bound("D loss", loss, ref.reshape(1), L * 2.0 ** -24 * ref.reshape(1), f"loss B={B} per={per}")
        refg = (2 * w64 * d / (per * B) * ls).reshape(-1)
        _bound("D dpred", dp, refg, bf16_ulp(refg) + 2.0 ** -20 * refg.abs(), f"dpred B={B} per={per}")
        loss2, dp2 = _loss_run(ops, pred, tg, w, ls, True, B, per)
        _same_bits(loss2, loss, "loss repeat")
        _same_bits(dp2, dp, "dpred repeat")
        loss3, _ = _loss_run(ops, pred, tg, w, ls, False, B, per)
        _same_bits(loss3, loss, "loss with dpred = NULL")
    ones = torch.ones(B, device="cuda")
    _same_bits(_loss_run(ops, pred, tg, ones, ls, False, B, per)[0], _loss_run(ops, pred, tg, None, ls, False, B, per)[0],
               "weight NULL == ones")


def test_timestep_sinusoid(ops):
    """Every integer timestep 0 .. 999 the step feeds, plus fractional ones, against fp64."""
    t = torch.cat([torch.arange(1000, dtype=torch.float32), torch.tensor([0.5, 1e-3, 123.25, 999.9, 7.77])]).cuda()
    n = t.numel()
    out = Guarded(n * 256)
    ops.timestep_sinusoid(t, out.t, n)
    out.check("sinusoid")
    freq = torch.exp(-math.log(10000.0) * torch.arange(128, dtype=torch.float64, device="cuda") / 128)
    a = t.double()[:, None] * freq[None]
    ref = torch.cat([a.cos(), a.sin()], 1)
    err = 12 * 2.0 ** -23 * a.abs() + 2.0 ** -23
    _bound("D sinusoid", out.view(n, 256), ref, bf16_ulp(ref) + torch.cat([err, err], 1), "sinusoid")


def _cast_source(n, g):
    """For scale 0.5 and 2 (exact, so ties stay ties): ties between bf16 neighbours (to even: down, up), subnormals,
    +-inf, values whose product overflows fp32 or rounds to bf16 inf (at scale 2), NaN, signed zeros; the last (up to)
    three elements, which the scalar tail converts, sit just above a tie, where rounding toward zero differs."""
    special = torch.tensor([4 * (1 + 2.0 ** -8), -4 * (1 + 3 * 2.0 ** -8), 1e-40, -3e-39, 2.0 ** -130, float("inf"),
                            -float("inf"), 1.7e38, -3.39e38, 1.6947e38, NAN, 0.0, -0.0], dtype=torch.float32)
    src = torch.randn(n, generator=g) * 10
    k = min(n, special.numel())
    src[:k] = special[:k]
    t = min(n, 3)
    src[n - t:] = torch.tensor([4 * (1 + 2.0 ** -8 + 2.0 ** -20), -8 * (1 + 2.0 ** -8 + 2.0 ** -19), 3 * (1 + 2.0 ** -8)])[:t]
    return src.cuda()


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 1000003])
@pytest.mark.parametrize("scale", [0.5, 2.0])
def test_cast_f32_bf16(ops, n, scale):
    """Bit-exact against torch's round-to-nearest-even of src * scale (ties, subnormals, infinities, overflow; NaN in,
    NaN out); dst 8-byte but not 16-byte aligned, with a sentinel right after dst[n - 1]."""
    src = _cast_source(n, torch.Generator().manual_seed(n))
    dst = Guarded(n, shift=4)
    ops.cast_f32_bf16(src, dst.t, n, scale)
    dst.check("cast dst")
    ref = (src * scale).bfloat16()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(dst.t), nan)
    _same_bits(dst.t[~nan], ref[~nan], f"cast n={n}")


def _sumsq_run(ops, x, n, out0):
    out, ws = Guarded(1, torch.float32), Guarded(1024, torch.float32)
    out.t.fill_(out0)
    ops.sumsq(x, n, out.t, ws.t)
    out.check("sumsq out")
    ws.check("sumsq partial_ws", [window(ws.buf, PAD, 1, REDUCE, REDUCE)])
    return out.t.clone()


@pytest.mark.parametrize("n", [1, 3, 4, 5, 7, 1000003])
def test_sumsq(ops, n):
    """out += sum x^2 against fp64, with a nonzero previous value; and with only the 1-3 tail elements nonzero."""
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, device="cuda", generator=g)
    L = 4 * -(-(n // 4) // (REDUCE * 256)) + 40
    for out0 in (0.0, 1.5):
        ref = (out0 + (x.double() ** 2).sum()).reshape(1)
        _bound("D sumsq", _sumsq_run(ops, x, n, out0), ref, L * 2.0 ** -24 * ref, f"sumsq n={n}")
    if n % 4:
        xt = torch.zeros(n, device="cuda")
        xt[n - n % 4:] = x[n - n % 4:] + 3
        ref = (xt.double() ** 2).sum().reshape(1)
        _bound("D sumsq", _sumsq_run(ops, xt, n, 0.0), ref, L * 2.0 ** -24 * ref, f"sumsq tail only n={n}")


def _adamw64(p, g, m, v, ss, max_norm, lr, b1, b2, eps, wd, step, gd):
    """fp64 replay of clip + AdamW from the fp32 inputs and hyper-parameters; returns (p, m, v, bounds)."""
    f = lambda z: float(torch.tensor(z, dtype=torch.float32))
    b1, b2, lr, eps, wd, gd = map(f, (b1, b2, lr, eps, wd, gd))
    coef = gd
    if max_norm > 0:
        coef *= min(1.0, f(max_norm) / (math.sqrt(ss) * gd + f(1e-6)))
    p, g, m, v = p.double(), g.double(), m.double(), v.double()
    gi = g * coef
    t1, t2 = b1 * m, (1 - b1) * gi
    m1 = t1 + t2
    u1, u2 = b2 * v, (1 - b2) * gi * gi
    v1 = u1 + u2
    bc1, bc2s = 1 - b1 ** step, math.sqrt(1 - b2 ** step)
    denom = v1.sqrt() / bc2s + eps
    p1 = p * (1 - lr * wd) - (lr / bc1) * m1 / denom
    # m1 may cancel: its error, and the update's, are relative to the magnitudes of its two terms
    return (p1, m1, v1, 2 * f32_ulp(p1) + 2.0 ** -18 * (lr / bc1) * (t1.abs() + t2.abs()) / denom,
            2 * f32_ulp(m1) + 2.0 ** -18 * (t1.abs() + t2.abs()), 2 * f32_ulp(v1) + 2.0 ** -18 * (u1.abs() + u2.abs()))


@pytest.mark.parametrize("n", [1, 2, 3, 5, 100003])
@pytest.mark.parametrize("case", ["clip", "no_clip", "max_norm_0", "max_norm_neg"])
@pytest.mark.parametrize("step,wd", [(1, 0.0), (1000, 0.01)])
def test_adamw_clip(ops, n, case, step, wd):
    """Clip active and inactive, and clipping off (max_norm <= 0) with grad_div != 1 and a NaN sumsq that must not be
    read; wd 0 and != 0; steps 1 and 1000 (non-zero moments).  p, g, m, v in sentinel buffers; g is zeroed on exactly n
    elements."""
    gen = torch.Generator(device="cuda").manual_seed(n + step)
    gd, lr, b1, b2, eps = 0.5, 1e-2, 0.9, 0.99, 1e-8
    p0 = torch.randn(n, device="cuda", generator=gen)
    g0 = torch.randn(n, device="cuda", generator=gen) * 0.05
    m0 = torch.randn(n, device="cuda", generator=gen) * 0.01 if step > 1 else torch.zeros(n, device="cuda")
    v0 = torch.rand(n, device="cuda", generator=gen) * 1e-3 if step > 1 else torch.zeros(n, device="cuda")
    norm = g0.double().norm().item() * gd
    max_norm = {"clip": norm / 3, "no_clip": norm * 3, "max_norm_0": 0.0, "max_norm_neg": -1.0}[case]
    ssv = float((g0.double() ** 2).sum().float())
    ss = torch.full((1,), NAN if max_norm <= 0 else ssv, device="cuda")
    bufs = [Guarded(n, torch.float32) for _ in range(4)]
    for b, t in zip(bufs, (p0, g0, m0, v0)):
        b.t.copy_(t)
    ops.adamw_clip(*(b.t for b in bufs), n, ss, max_norm, lr, b1, b2, eps, wd, step, grad_div=gd)
    p1, m1, v1, bp, bm, bv = _adamw64(p0, g0, m0, v0, ssv, max_norm, lr, b1, b2, eps, wd, step, gd)
    _bound("D adamw", bufs[0].t, p1, bp, f"p {case}")
    _bound("D adamw", bufs[2].t, m1, bm, f"m {case}")
    _bound("D adamw", bufs[3].t, v1, bv, f"v {case}")
    assert torch.equal(bufs[1].t, torch.zeros_like(bufs[1].t))
    for b, name in zip(bufs, "pgmv"):
        b.check(f"adamw {name}")


# ---------------------------------------------------------------------------------------------------------------------
# E. argument refusals: every misaligned vector operand, NULL head-split tensor, rope bit past nseg, empty shape.  Each
# refused call leaves every output untouched.
# ---------------------------------------------------------------------------------------------------------------------
ALIGN, SHAPE, ARG = -2, -1, -5


def _mis(t):
    """The same tensor one element (2 or 4 bytes) further into a larger allocation: not 16-byte aligned."""
    buf = torch.empty(t.numel() + 8, dtype=t.dtype, device="cuda")
    m = buf[1:1 + t.numel()].view(t.shape)
    m.copy_(t)
    return m


def test_refuse_norm_modulate_and_colscale(ops):
    R, D, rps, eps = 4, 72, 2, 1e-6
    x, dy, dxin = (torch.randn(R, D, device="cuda").bfloat16() for _ in range(3))
    tab, temb = torch.zeros(6, D, device="cuda").bfloat16(), torch.zeros(2, 6 * D, device="cuda").bfloat16()
    y, dx, o2 = Guarded(R * D), Guarded(R * D), Guarded(R * D)
    fwd = dict(x=x, y=y.view(R, D), shift_tab=tab[0], shift_emb=temb, scale_tab=tab[1], scale_emb=temb[:, D:],
               emb_stride=6 * D)
    runf = lambda **kw: ops.norm_modulate_fwd(**dict(fwd, **kw), rows=R, D=D, rows_per_sample=rps, eps=eps)
    for k in ("x", "shift_tab", "shift_emb", "scale_tab", "scale_emb"):
        _raises_code(ALIGN, lambda: runf(**{k: _mis(fwd[k])}))
    _raises_code(ALIGN, lambda: runf(y=_mis(y.view(R, D))))
    _raises_code(ALIGN, lambda: runf(emb_stride=6 * D + 4))
    y.check("norm_modulate_fwd refused", [])
    bwd = dict(dy=dy, x=x, dx_in=dxin, dx_out=dx.view(R, D), scale_tab=tab[1], scale_emb=temb[:, D:], gate2_tab=tab[5],
               gate2_emb=temb[:, 5 * D:], out2=o2.view(R, D), emb_stride=6 * D)
    runb = lambda **kw: ops.norm_modulate_bwd(**dict(bwd, **kw), rows=R, D=D, rows_per_sample=rps, eps=eps)
    for k in ("dy", "x", "dx_in", "scale_tab", "scale_emb", "gate2_tab", "gate2_emb"):
        _raises_code(ALIGN, lambda: runb(**{k: _mis(bwd[k])}))
    _raises_code(ALIGN, lambda: runb(dx_out=_mis(dx.view(R, D))))
    _raises_code(ALIGN, lambda: runb(out2=_mis(o2.view(R, D))))
    _raises_code(ALIGN, lambda: runb(emb_stride=6 * D - 2))
    dx.check("norm_modulate_bwd refused", [])
    o2.check("norm_modulate_bwd out2 refused", [])
    out = Guarded(R * D)
    cs = dict(x=x, out=out.view(R, D), tab=tab[5], emb=temb[:, 5 * D:], emb_stride=6 * D)
    runc = lambda **kw: ops.colscale(**dict(cs, **kw), rows=R, D=D, rows_per_sample=rps)
    for k in ("x", "tab", "emb"):
        _raises_code(ALIGN, lambda: runc(**{k: _mis(cs[k])}))
    _raises_code(ALIGN, lambda: runc(out=_mis(out.view(R, D))))
    _raises_code(ALIGN, lambda: runc(emb_stride=6 * D + 1))
    out.check("colscale refused", [])


def test_refuse_qkv(ops):
    p = QkvProblem(2, 7, 1, 3, 0b111, 0b011, seed=5)
    B, S, H, D = p.B, p.S, p.H, p.D
    n = B * H * S * 64
    dsts = [Guarded(n) for _ in range(3)]
    dv = [d.view(B, H, S, 64) for d in dsts]
    dx = Guarded(p.rows * p.ld_dx)

    def fwd(src=p.src, w=p.w, rope=0b011, cos=p.cos, sin=p.sin, d=dv):
        ops.qkv_norm_rope_fwd(src, p.ld, p.col_off, w, rope, cos, sin, d, B, S, H, p.eps)

    def bwd(x=p.src, w=p.w, rope=0b011, cos=p.cos, sin=p.sin, dy=p.dy, dxt=dx.view(p.rows, p.ld_dx)):
        ops.qkv_norm_rope_bwd(dy, x, p.ld, p.col_off, w, rope, cos, sin, dxt, p.ld_dx, p.dx_col_off, B, S, H, p.eps)

    _raises_code(ALIGN, lambda: fwd(src=_mis(p.src)))
    _raises_code(ALIGN, lambda: fwd(cos=_mis(p.cos)))
    _raises_code(ALIGN, lambda: fwd(sin=_mis(p.sin)))
    for i in range(3):
        _raises_code(ALIGN, lambda: fwd(w=[_mis(w) if j == i else w for j, w in enumerate(p.w)]))
        _raises_code(ALIGN, lambda: fwd(d=[_mis(t) if j == i else t for j, t in enumerate(dv)]))
        _raises_code(ARG, lambda: fwd(d=[None if j == i else t for j, t in enumerate(dv)]))
        _raises_code(ALIGN, lambda: bwd(w=[_mis(w) if j == i else w for j, w in enumerate(p.w)]))
        _raises_code(ALIGN, lambda: bwd(dy=[_mis(t) if j == i else t for j, t in enumerate(p.dy)]))
        if i > 0:   # dy_0 is the pointer the entry point binds the device with: NULL there fails before the checks
            _raises_code(ARG, lambda: bwd(dy=[None if j == i else t for j, t in enumerate(p.dy)]))
    _raises_code(ARG, lambda: ops.qkv_norm_rope_fwd(p.src, p.ld, p.col_off, p.w[:2], 0b100, p.cos, p.sin, dv[:2], B, S, H,
                                                   p.eps))
    _raises_code(ARG, lambda: fwd(rope=0b1000))
    _raises_code(ALIGN, lambda: bwd(x=_mis(p.src)))
    _raises_code(ALIGN, lambda: bwd(cos=_mis(p.cos)))
    _raises_code(ALIGN, lambda: bwd(sin=_mis(p.sin)))
    _raises_code(ALIGN, lambda: bwd(dxt=_mis(dx.view(p.rows, p.ld_dx))))
    _raises_code(ARG, lambda: ops.qkv_norm_rope_bwd(p.dy[:1], p.src, p.ld, p.col_off, p.w[:1], 0b10, p.cos, p.sin,
                                                   dx.view(p.rows, p.ld_dx), p.ld_dx, p.dx_col_off, B, S, H, p.eps))
    _raises_code(ARG, lambda: bwd(rope=-1))
    # the single-segment entry points share the checks
    w0 = p.w[0]
    _raises_code(ALIGN, lambda: ops.qknorm_rope_fwd(_mis(p.src), p.ld, p.col_off, w0, p.cos, p.sin, dv[0], B, S, H,
                                                    True, p.eps))
    _raises_code(ALIGN, lambda: ops.qknorm_rope_fwd(p.src, p.ld, p.col_off, _mis(w0), p.cos, p.sin, dv[0], B, S, H,
                                                    True, p.eps))
    _raises_code(ARG, lambda: ops.qknorm_rope_fwd(p.src, p.ld, p.col_off, w0, p.cos, p.sin, None, B, S, H, True, p.eps))
    _raises_code(ALIGN, lambda: ops.qknorm_rope_bwd(p.dy[0], p.src, p.ld, p.col_off, w0, p.cos, p.sin,
                                                    _mis(dx.view(p.rows, p.ld_dx)), p.ld_dx, p.dx_col_off, B, S, H,
                                                    True, p.eps))
    for d in dsts:
        d.check("qkv fwd refused", [])
    dx.check("qkv bwd refused", [])


def test_refuse_satellites(ops):
    B, per = 2, 64
    pred, tg = torch.randn(B * per, device="cuda").bfloat16(), torch.randn(B * per, device="cuda").bfloat16()
    loss, ws, dp = Guarded(1, torch.float32), Guarded(1024, torch.float32), Guarded(B * per)
    run = lambda pr=pred, t=tg, d=dp.t, b=B, ps=per: ops.loss_mse(pr, t, None, 1.0, loss.t, d, ws.t, b, ps)
    _raises_code(ALIGN, lambda: run(pr=_mis(pred)))
    _raises_code(ALIGN, lambda: run(t=_mis(tg)))
    _raises_code(ALIGN, lambda: run(d=_mis(dp.t)))
    _raises_code(SHAPE, lambda: run(b=0))
    _raises_code(SHAPE, lambda: run(b=-1))
    _raises_code(SHAPE, lambda: run(ps=0))
    _raises_code(SHAPE, lambda: run(ps=-8))
    for t, what in ((loss, "loss_out"), (ws, "partial_ws"), (dp, "dpred")):
        t.check(f"loss refused: {what}", [])
    x = torch.randn(64, device="cuda")
    out = Guarded(1, torch.float32)
    _raises_code(ALIGN, lambda: ops.sumsq(_mis(x), 63, out.t, ws.t))
    out.check("sumsq refused", [])
    ws.check("sumsq refused: partial_ws", [])
    dst = Guarded(64, shift=2)
    _raises_code(ALIGN, lambda: ops.cast_f32_bf16(_mis(x), Guarded(64).t, 63, 1.0))
    _raises_code(ALIGN, lambda: ops.cast_f32_bf16(x, dst.t, 64, 1.0))
    dst.check("cast refused", [])
    so = Guarded(256)
    for n in (0, -3):
        ops.timestep_sinusoid(torch.ones(1, device="cuda"), so.t, n)
    so.check("sinusoid n <= 0", [])
    cos, sin = Guarded(64 * 6, torch.float32), Guarded(64 * 6, torch.float32)
    for F, H, W in ((0, 4, 4), (2, 0, 4), (2, 4, -1)):
        _raises_code(SHAPE, lambda: ops.rope_table(cos.t, sin.t, F, H, W, 12, 0.1, 0.1, 0.1))
    cos.check("rope_table refused", [])
    sin.check("rope_table refused", [])
    p = [Guarded(8, torch.float32) for _ in range(4)]
    for i in range(4):
        args = [_mis(b.t) if j == i else b.t for j, b in enumerate(p)]
        _raises_code(ALIGN, lambda: ops.adamw_clip(*args, 7, torch.ones(1, device="cuda"), 1.0, 1e-3, 0.9, 0.99, 1e-8,
                                                   0.0, 1))
    for b in p:
        b.check("adamw refused", [])
