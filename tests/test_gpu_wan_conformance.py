"""Wan-2.1 kernel conformance: the seven entry points Wan's step adds to b2d_elem.cu (the affine LayerNorm, the per-head
q/k-norm + RoPE, the per-head RoPE table, the step prologue and the patch permutes) at every dispatch width and at the
1.3B and 14B call forms, with the outputs inside sentinel buffers and the inputs a kernel must not read poisoned.

Conventions as in test_gpu_elem.py: each element is checked against a reference computed on the GPU from the same
bf16 / fp32 inputs; every output buffer element outside the output window keeps the sentinel bit pattern
(_util.sentinel_buffer), with windows moved off the 16-byte alignment where the entry point stores scalars; every input
element a kernel must not read (weight and bias elements past D, table rows past S, temb chunks other than the gate's,
source columns outside the segment window) holds NaN, so reading one turns an output into NaN, which check_bound rejects.

Bounds (ulp16 / ulp32 = bf16 / fp32 spacing at the reference value, "rowmax" = the largest magnitude in the row):
  A  affine LayerNorm fwd:  ulp16(ref) + 2^-16 * rowmax(|xhat w| + |b|)
     affine LayerNorm bwd:  ulp16(ref) + 2^-16 * (|dx_in| + rstd * rowmax|g| * (1 + rowmax|xhat|)^2),  g = dy w
     out2:                  ulp16(ref) + 2^-22 |ref|  (two fp32 roundings of a product of bf16 values)
     These are test_gpu_elem.py part A's bounds with the modulation (1 + scale) replaced by the weight w: the kernels
     are the same row bodies.  The fp32 row statistics (a per-thread serial sum, then a warp and a block tree) carry a
     relative error below 2^-18 for D <= 8192, and the final (x - mean) rstd w + b and g - mean(g) - xhat mean(g xhat)
     steps scale it by at most the terms named; the rest is the final bf16 rounding, half an ulp16.
  B  per-head q/k fwd:  ulp16(ref) + 2^-16 * 2 rowmax|n|  (n = the normalized, unrotated segment row; the rotation by a
                        unit (cos, sin) pair adds two fp32 products and one sum, each relative to at most |n|)
     per-head q/k bwd:  ulp16(ref) + 2^-16 * rstd * rowmax|g| * (1 + rowmax|xhat|)^2,  g = rope^T(dy) w, or 2 rowmax|dy|
                        for a segment without a norm
     plus, bit for bit: the _ph entry points against the _hd ones given the per-head table tiled over the H heads.
  C  rope_table_wan:  |t - t64| <= ulp32(t64) / 2 + (|angle| + 1) 2^-50.  The kernel evaluates theta^(2i/n), 1 / that,
     pos * freq and cos / sin in float64 and rounds once to fp32 (half an ulp32).  The device's double pow, division
     and product put the angle within a few double ulps of the exact one, |d angle| <= 2^-50 |angle|, and its double
     cos / sin add at most 2^-52; both are far below the fp32 rounding.  The float64 reference itself is cross-checked
     against oracle.wan_independent_constants.wan_rope_entry at a few hundred entries under the same slack.
  D  wan_prep:       bit-exact against oracle.wan_oracle.prologue run on the GPU (NaN inputs: NaN outputs).
  E  patch_permute:  exact.

The worst error / bound ratio of each part is printed at the end of the module (pytest -s).  Measured on an H100 80GB
HBM3 at a 700 W power limit: see DESIGN.md section 4.13.
"""
import ctypes as C
import re

import pytest
import torch

from _util import bf16_ulp, check_bound, check_sentinel, f32_ulp, sentinel_buffer, window

pytestmark = pytest.mark.gpu

NAN = float("nan")
PAD = 64            # sentinel elements on each side of an output window
TAIL = 256          # sentinel elements after a RoPE table: a whole 256-thread block past the last entry
ALIGN, SHAPE, ARG = -2, -1, -5


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
    print("\nworst error/bound ratio per part:", {k: round(v, 6) for k, v in sorted(WORST.items())})


def _raises_code(code, fn):
    from finetrainers_b200.lib import B2DError
    with pytest.raises(B2DError, match=rf"\(code {code}\)"):
        fn()


def _bits(t):
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _same_bits(a, b, what):
    a, b = _bits(a), _bits(b)
    n = int((a != b).sum())
    assert n == 0, f"{what}: {n} element(s) differ"


class Guarded:
    """An output of `n` elements inside a sentinel-filled buffer with `pad` elements of margin on each side; `shift`
    elements move the window off the buffer's 16-byte alignment."""

    def __init__(self, n, dtype=torch.bfloat16, shift=0, pad=PAD):
        self.n, self.off = n, pad + shift
        self.buf = sentinel_buffer(n + 2 * pad + shift, dtype)
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


def _rowmax(t):
    return t.abs().amax(-1, keepdim=True)


def _mis(t):
    """The same tensor one element (2 or 4 bytes) further into a larger allocation: not 16-byte aligned."""
    buf = torch.empty(t.numel() + 8, dtype=t.dtype, device="cuda")
    m = buf[1:1 + t.numel()].view(t.shape)
    m.copy_(t)
    return m


# ---------------------------------------------------------------------------------------------------------------------
# A. layer_norm_affine_fwd / bwd
# ---------------------------------------------------------------------------------------------------------------------
def _rows_with_edges(g, R, D):
    """Random rows with the statistics edges in rows 1-3: a large common offset next to the spread (mean 32, std 1), a
    constant row (variance 0: eps decides), and tiny rows (|x| ~ 1e-4)."""
    x = torch.randn(R, D, device="cuda", generator=g)
    x[1] = 32 + torch.randn(D, device="cuda", generator=g)
    x[2] = 0.75
    x[3] = 1e-4 * torch.randn(D, device="cuda", generator=g)
    return x.bfloat16()


def _vec(g, D, mean, std):
    """[D] bf16 values followed by D NaN elements."""
    v = torch.full((2 * D,), NAN, device="cuda", dtype=torch.bfloat16)
    v[:D] = (mean + std * torch.randn(D, device="cuda", generator=g)).bfloat16()
    return v


def _affine_case(ops, R, D, rps, seed, emb_stride=None, gate=2, eps=1e-6):
    """Forward, then the backward with out2 (gate2 from table row `gate` and temb chunk `gate`, every other row and
    chunk NaN, emb_stride != 6 D by default), in place, with dx_in = NULL and with out2 = NULL."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    nb = R // rps
    es = emb_stride or 6 * D + 8
    x = _rows_with_edges(g, R, D)
    w, bias = _vec(g, D, 1.0, 0.2), _vec(g, D, 0.0, 0.1)
    wd, bd = w[:D].double(), bias[:D].double()
    y = Guarded(R * D)
    ops.layer_norm_affine_fwd(x, y.view(R, D), w, bias, R, D, eps)
    xd = x.double().requires_grad_(True)
    xc = xd - xd.mean(-1, keepdim=True)
    rstd = torch.rsqrt((xc * xc).mean(-1, keepdim=True) + eps)
    xhat = xc * rstd
    ref = (xhat * wd + bd).detach()
    _bound("A affine fwd", y.view(R, D), ref, bf16_ulp(ref) + 2.0 ** -16 * _rowmax(xhat.detach().abs() * wd.abs() + bd.abs()),
           f"fwd R={R} D={D}")
    y.check(f"affine fwd y D={D}")

    tab = torch.full((6, D), NAN, device="cuda", dtype=torch.bfloat16)
    tab[gate] = _rnd(g, D, scale=0.3)
    temb = torch.full((nb, es), NAN, device="cuda", dtype=torch.bfloat16)
    temb[:, gate * D:(gate + 1) * D] = _rnd(g, nb, D, scale=0.3)
    b = torch.arange(R, device="cuda") // rps
    gate64 = tab[gate].double()[None] + temb[:, gate * D:(gate + 1) * D].double()[b]
    dy, dxin = _rnd(g, R, D), _rnd(g, R, D)
    (xhat * wd).backward(dy.double())
    grad = xd.grad
    scl = rstd.detach() * _rowmax(dy.double() * wd) * (1 + _rowmax(xhat.detach())) ** 2
    gkw = dict(gate2_tab=tab[gate], gate2_emb=temb[:, gate * D:], emb_stride=es, rows_per_sample=rps)

    dx, o2 = Guarded(R * D), Guarded(R * D)
    ops.layer_norm_affine_bwd(dy, x, dxin, dx.view(R, D), w, R, D, eps, out2=o2.view(R, D), **gkw)
    refdx = dxin.double() + grad
    _bound("A affine bwd", dx.view(R, D), refdx, bf16_ulp(refdx) + 2.0 ** -16 * (dxin.double().abs() + scl),
           f"bwd R={R} D={D}")
    ref2 = dx.view(R, D).double() * gate64
    _bound("A affine bwd out2", o2.view(R, D), ref2, bf16_ulp(ref2) + 2.0 ** -22 * ref2.abs(), f"out2 R={R} D={D}")
    dx.check(f"affine bwd dx D={D}")
    o2.check(f"affine bwd out2 D={D}")

    # in place (dx_in == dx_out): the same bits as out of place
    inpl, o2i = dxin.clone(), Guarded(R * D)
    ops.layer_norm_affine_bwd(dy, x, inpl, inpl, w, R, D, eps, out2=o2i.view(R, D), **gkw)
    _same_bits(inpl, dx.view(R, D), f"in-place dx D={D}")
    _same_bits(o2i.buf, o2.buf, f"in-place out2 D={D}")

    # dx_in = NULL (with out2)
    dx0, o20 = Guarded(R * D), Guarded(R * D)
    ops.layer_norm_affine_bwd(dy, x, None, dx0.view(R, D), w, R, D, eps, out2=o20.view(R, D), **gkw)
    _bound("A affine bwd", dx0.view(R, D), grad, bf16_ulp(grad) + 2.0 ** -16 * scl, f"bwd dx_in=NULL D={D}")
    ref2 = dx0.view(R, D).double() * gate64
    _bound("A affine bwd out2", o20.view(R, D), ref2, bf16_ulp(ref2) + 2.0 ** -22 * ref2.abs(), f"out2 dx_in=NULL D={D}")
    dx0.check(f"affine bwd dx (dx_in = NULL) D={D}")
    o20.check(f"affine bwd out2 (dx_in = NULL) D={D}")

    # out2 = NULL, no gate pointers: dx the same bits as with out2
    dxn = Guarded(R * D)
    ops.layer_norm_affine_bwd(dy, x, dxin, dxn.view(R, D), w, R, D, eps, emb_stride=es, rows_per_sample=rps)
    _same_bits(dxn.buf, dx.buf, f"out2 = NULL dx D={D}")


@pytest.mark.parametrize("rps", [5, 1])
@pytest.mark.parametrize("D", [8, 72, 1536, 2048, 2056, 4096, 4104, 5120, 6144, 8192])
def test_layer_norm_affine(ops, D, rps):
    """Every AFFINE instantiation (nch = ceil(D / 2048)): 1 chunk (8, 72, 1536 = the 1.3B width, 2048), 2 chunks (2056,
    4096), the 4-chunk kernel with 3 chunks active (4104, 5120 = the 14B width, 6144) and 4 chunks (8192); four samples
    of 5 rows, or one row per sample."""
    _affine_case(ops, 4 * rps, D, rps, seed=D + rps)


@pytest.mark.parametrize("D", [1536, 5120])
def test_layer_norm_affine_step_shapes(ops, D):
    """Wan's own call forms: 1560 tokens of one sample (a 480 x 832 latent frame) at the 1.3B and 14B widths, the gate
    from table row 2 and temb chunk 2 with emb_stride = 6 D, as the cross-attention pre-norm's backward runs."""
    _affine_case(ops, 1560, D, 1560, seed=D, emb_stride=6 * D)


# ---------------------------------------------------------------------------------------------------------------------
# B. qkv_norm_rope_ph_fwd / bwd (per-head RoPE)
# ---------------------------------------------------------------------------------------------------------------------
class PhProblem:
    """nseg D-wide segments (D = H * hd) at col_off of rows [B*S, ld]; every other source column is NaN.  The per-head
    tables are [S + 1, hd/2] with row S NaN; weights are [D] followed by D NaN elements, or stacked per block of
    rows_per_w rows with stride w_stride."""

    def __init__(self, B, S, H, hd, nseg, wmask, rope, col_off=24, ld_extra=40, dx_col_off=16, ld_dx_extra=88,
                 rows_per_w=0, w_stride=0, eps=1e-6, seed=0):
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
        ang = torch.randn(S + 1, hd // 2, device="cuda", generator=g) * 3
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

    def tables(self, per_head=True):
        """The per-head tables, or the same tiled over the H heads into full-width [S + 1, D/2] tables (row S NaN)."""
        if not self.rope:
            return None, None
        if per_head:
            return self.cos, self.sin
        return self.cos.repeat(1, self.H).contiguous(), self.sin.repeat(1, self.H).contiguous()

    def reference(self, i):
        """(fwd ref [B,H,S,hd], dx ref [rows, D], fwd bound, dx bound) of segment i, fp64 with autograd; channel c of a
        row rotates by table pair (c mod hd) / 2."""
        x = self.seg(i).double().requires_grad_(True)
        n = x
        s_idx = torch.arange(self.rows, device="cuda") % self.S
        norm, rot = self.w[i] is not None, (self.rope >> i) & 1
        if norm:
            rstd = torch.rsqrt((x * x).mean(-1, keepdim=True) + self.eps)     # over all D channels: across heads
            n = x * rstd * self.weight_rows(i)
        o = n
        if rot:
            c = self.cos[:self.S].double()[s_idx].repeat(1, self.H)
            s = self.sin[:self.S].double()[s_idx].repeat(1, self.H)
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

    def run_fwd(self, ops, per_head=True):
        dsts = [Guarded(self.B * self.H * self.S * self.hd) for _ in range(self.nseg)]
        c, s = self.tables(per_head)
        ops.qkv_norm_rope_fwd(self.src, self.ld, self.col_off, self.w, self.rope, c, s,
                              [d.view(self.B, self.H, self.S, self.hd) for d in dsts], self.B, self.S, self.H, self.eps,
                              rows_per_w=self.rows_per_w, w_stride=self.w_stride, head_dim=self.hd, per_head=per_head)
        return dsts

    def run_bwd(self, ops, per_head=True):
        dx = Guarded(self.rows * self.ld_dx)
        c, s = self.tables(per_head)
        ops.qkv_norm_rope_bwd(self.dy, self.src, self.ld, self.col_off, self.w, self.rope, c, s,
                              dx.view(self.rows, self.ld_dx), self.ld_dx, self.dx_col_off, self.B, self.S, self.H,
                              self.eps, rows_per_w=self.rows_per_w, w_stride=self.w_stride, head_dim=self.hd,
                              per_head=per_head)
        return dx

    def check(self, ops, what):
        dsts, dx = self.run_fwd(ops), self.run_bwd(ops)
        dxw = window(dx.buf, dx.off + self.dx_col_off, self.rows, self.nseg * self.D, self.ld_dx)
        for i in range(self.nseg):
            f, gx, fb, gb = self.reference(i)
            out = dsts[i].view(self.B, self.H, self.S, self.hd)
            dxi = dxw[:, i * self.D:(i + 1) * self.D]
            tag = f"{what} hd={self.hd} H={self.H} seg {i} (w {self.wmask:03b}, rope {self.rope:03b})"
            _bound("B ph fwd", out, f, fb, tag + " fwd")
            _bound("B ph bwd", dxi, gx, gb, tag + " bwd")
            if self.w[i] is None and not (self.rope >> i) & 1:       # neither norm nor rope: a copy both ways
                _same_bits(out, self.heads(self.seg(i)), tag + " fwd copy")
                _same_bits(dxi, self.rows_of(self.dy[i]), tag + " bwd copy")
            dsts[i].check(tag + " dst")
        dx.check(what + " dx", [dxw])
        # the full-width entry points with the tiled table run the same row body: the same bits, sentinels included
        for a, b in zip(dsts, self.run_fwd(ops, per_head=False)):
            _same_bits(a.buf, b.buf, f"{what} hd={self.hd} H={self.H}: _ph fwd vs _hd fwd with the tiled table")
        _same_bits(dx.buf, self.run_bwd(ops, per_head=False).buf,
                   f"{what} hd={self.hd} H={self.H}: _ph bwd vs _hd bwd with the tiled table")


@pytest.mark.parametrize("nseg", [1, 2, 3])
@pytest.mark.parametrize("H", [1, 2])
@pytest.mark.parametrize("hd", [64, 128])
def test_ph_every_combination(ops, hd, H, nseg):
    """Every weight present / absent per segment x every rope_mask in 0 .. 2^nseg - 1, B = 2, S = 7."""
    for wmask in range(1 << nseg):
        for rope in range(1 << nseg):
            PhProblem(2, 7, H, hd, nseg, wmask, rope, seed=wmask * 8 + rope).check(ops, f"nseg={nseg}")


# a subset that still has every segment normed and not, rotated and not, and the third segment's norm with and without
# the first two
SUBSET = [(3, 0b011, 0b011), (3, 0b100, 0b100), (3, 0b101, 0b010), (3, 0b111, 0b111), (3, 0b000, 0b000),
          (2, 0b10, 0b01), (1, 0b1, 0b1)]


@pytest.mark.parametrize("hd,H", [(128, 12), (128, 16), (128, 17), (128, 32), (128, 40), (128, 64),
                                  (64, 32), (64, 33), (64, 65), (64, 128)])
def test_ph_widths(ops, hd, H):
    """Every chunk class at both head dimensions: 1 chunk (12 x 128 = the 1.3B width, 16 x 128, 32 x 64), 2 chunks
    (17 x 128, 32 x 128, 33 x 64), 3 of 4 chunks (40 x 128 = the 14B width, 65 x 64) and 4 chunks (64 x 128,
    128 x 64)."""
    for nseg, wmask, rope in SUBSET:
        PhProblem(2, 7, H, hd, nseg, wmask, rope, seed=H + wmask).check(ops, f"nseg={nseg}")


@pytest.mark.parametrize("hd,H", [(64, 2), (128, 2), (128, 40)])
def test_ph_stacked_weights(ops, hd, H):
    """rows_per_w > 0 (two blocks of 2 x 7 rows, w_stride != D) with a rotated normed segment, a normed unrotated one
    and a rotated copy."""
    PhProblem(4, 7, H, hd, 3, 0b011, 0b101, rows_per_w=14, w_stride=H * hd + 24, seed=11).check(ops, "stacked")


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("H", [12, 40])
def test_ph_step_shapes(ops, H, B):
    """Wan's self-attention call form: q|k|v of the fused projection (ld = 3 D, no offsets), q and k normed and
    rotated (mask 0b011 / 0b011), v copied, S = 1560 tokens, at the 1.3B (12 heads) and 14B (40 heads) widths."""
    PhProblem(B, 1560, H, 128, 3, 0b011, 0b011, col_off=0, ld_extra=0, dx_col_off=0, ld_dx_extra=0,
              seed=B * 100 + H).check(ops, f"step B={B}")


# ---------------------------------------------------------------------------------------------------------------------
# C. rope_table_wan
# ---------------------------------------------------------------------------------------------------------------------
def _wan_angles64(F, H, W, hd, theta=10000.0):
    """The table's angles [S, hd/2] in float64: pair j of the t / h / w part of n dims at grid position p along its
    axis rotates by p * theta^(-2i / n), i the pair's index inside its part."""
    pairs, nhw = hd // 2, hd // 6
    nt = pairs - 2 * nhw
    j = torch.arange(pairs, device="cuda")
    axis = (j >= nt).long() + (j >= nt + nhw).long()
    i = j - torch.tensor([0, nt, nt + nhw], device="cuda")[axis]
    n = torch.tensor([2 * nt, 2 * nhw, 2 * nhw], device="cuda", dtype=torch.float64)[axis]
    freq = 1.0 / theta ** ((2 * i).double() / n)
    f, h, w = torch.meshgrid(torch.arange(F), torch.arange(H), torch.arange(W), indexing="ij")
    pos = torch.stack([f, h, w], -1).reshape(-1, 3).cuda().double()
    return pos[:, axis] * freq[None]


@pytest.mark.parametrize("F,H,W", [(1, 1, 1), (3, 5, 7), (13, 30, 52), (21, 45, 80)])
@pytest.mark.parametrize("hd", [6, 10, 64, 96, 128])
def test_rope_table_wan(ops, hd, F, H, W):
    """head_dim 6 (the minimum: one pair per part), 10 and 96 (not multiples of 12 or 6), 64 (the 24 / 20 / 20 split)
    and 128 (44 / 42 / 42); one token, a small odd grid, the 1.3B step grid (13 x 30 x 52) and the 14B 720p grid
    (21 x 45 x 80: 4.8 M entries).  Both tables sit 4 / 12 bytes off the 16-byte alignment with TAIL sentinel entries
    after them."""
    from oracle.wan_independent_constants import wan_rope_entry
    S, P = F * H * W, hd // 2
    cos = Guarded(S * P, torch.float32, shift=1, pad=TAIL)
    sin = Guarded(S * P, torch.float32, shift=3, pad=TAIL)
    ops.rope_table_wan(cos.t, sin.t, F, H, W, hd)
    cos.check(f"rope_table_wan cos hd={hd}")
    sin.check(f"rope_table_wan sin hd={hd}")
    ang = _wan_angles64(F, H, W, hd)
    slack = (ang.abs() + 1) * 2.0 ** -50
    c64, s64 = ang.cos(), ang.sin()
    _bound("C rope_table_wan", cos.view(S, P), c64, f32_ulp(c64) / 2 + slack, f"cos hd={hd} grid={F}x{H}x{W}")
    _bound("C rope_table_wan", sin.view(S, P), s64, f32_ulp(s64) / 2 + slack, f"sin hd={hd} grid={F}x{H}x{W}")
    # the reference against the independent scalar derivation
    g = torch.Generator().manual_seed(S + hd)
    for k in torch.randint(0, S * P, (min(300, S * P),), generator=g).tolist():
        s, p = divmod(k, P)
        c, sn = wan_rope_entry(s // (H * W), (s // W) % H, s % W, p, hd)
        tol = (abs(ang[s, p].item()) + 1) * 2.0 ** -50
        assert abs(c64[s, p].item() - c) <= tol and abs(s64[s, p].item() - sn) <= tol, (hd, s, p)


# ---------------------------------------------------------------------------------------------------------------------
# D. wan_prep
# ---------------------------------------------------------------------------------------------------------------------
def _patchify_ref(x, out_order):
    """[B, C, F, H, W] -> [B, F (H/2) (W/2), 4C] in the Conv3d (c, kh, kw) or proj_out (kh, kw, c) channel order."""
    B, C, F, H, W = x.shape
    t = x.reshape(B, C, F, H // 2, 2, W // 2, 2)
    t = t.permute(0, 2, 3, 5, 4, 6, 1) if out_order else t.permute(0, 2, 3, 5, 1, 4, 6)
    return t.reshape(B, F * (H // 2) * (W // 2), 4 * C)


LOGVAR_EDGES = [-30.0, 20.0, -30.25, 20.25, float("inf"), -float("inf")]


@pytest.mark.parametrize("B,C,F,H,W", [(1, 1, 1, 2, 2), (3, 3, 2, 6, 10), (2, 16, 3, 6, 10), (1, 16, 13, 60, 104)])
def test_wan_prep(ops, B, C, F, H, W):
    """Bit-exact against the reference's prologue run per sample on the GPU, with a distinct mean and std per sample and
    channel ([B, C], not expanded), sigma exactly 0 and 1 among the samples, the normalised logvar exactly on both clamp
    bounds, just beyond them and at +-inf, and NaN in a mean, a logvar, an eps and a noise element.  x_t and target sit
    2 / 6 bytes off the 16-byte alignment inside sentinel buffers."""
    from oracle import wan_oracle as O
    g = torch.Generator().manual_seed(B * 1000 + C * 10 + F)
    S = F * H * W
    mom = torch.cat([torch.randn(B, C, F, H, W, generator=g), torch.rand(B, C, F, H, W, generator=g) * 60 - 35], 1)
    mean = torch.randn(B, C, generator=g) * 0.3
    std = 1.0 / (torch.rand(B, C, generator=g) + 0.5)
    # channel 0: exact mean and power-of-two std per sample, so the edge logvars normalise to exactly LOGVAR_EDGES
    mean[:, 0] = 0.25 * (torch.arange(B) + 1)
    std[:, 0] = 2.0 ** (torch.arange(B) % 2).float()
    k = min(len(LOGVAR_EDGES), S)
    for b in range(B):
        mom[b, C].view(-1)[:k] = torch.tensor(LOGVAR_EDGES[:k]) / std[b, 0] + mean[b, 0]
    mom = mom.bfloat16()
    for b in range(B):
        lv = O.normalize_latents(mom[b:b + 1, C:C + 1], mean[b, :1], std[b, :1])
        assert torch.equal(lv.reshape(-1)[:k].float(), torch.tensor(LOGVAR_EDGES[:k])), b
    eps = torch.randn(B, C, F, H, W, generator=g).bfloat16()
    noise = torch.randn(B, C, F, H, W, generator=g).bfloat16()
    mom[-1, C - 1].view(-1)[-1] = NAN          # a mean
    mom[-1, 2 * C - 1].view(-1)[0] = NAN       # a logvar
    eps[0, 0].view(-1)[-1] = NAN
    noise[-1, -1].view(-1)[S // 2] = NAN
    sig = torch.tensor([0.0, 1.0, 0.37][:B]) if B > 1 else torch.tensor([0.6])
    mom, eps, noise, mean, std, sig = (t.cuda() for t in (mom, eps, noise, mean, std, sig))
    n = B * C * S
    xt, tg = Guarded(n, shift=1), Guarded(n, shift=3)
    ops.wan_prep(mom, eps, noise, mean.contiguous(), std.contiguous(), sig, xt.t, tg.t, B, C, F, H, W)
    xt.check("wan_prep x_t")
    tg.check("wan_prep target")
    refs = [O.prologue(mom[b:b + 1], mean[b], std[b], eps[b:b + 1], noise[b:b + 1], sig[b:b + 1]) for b in range(B)]
    for got, ref, order, what in ((xt, torch.cat([r[0] for r in refs]), 0, "x_t"),
                                  (tg, torch.cat([r[1] for r in refs]), 1, "target")):
        ref = _patchify_ref(ref, order).reshape(-1)
        nan = torch.isnan(ref)
        assert nan.any() and torch.equal(torch.isnan(got.t), nan), what
        _same_bits(got.t[~nan], ref[~nan], what)


# ---------------------------------------------------------------------------------------------------------------------
# E. patch_permute
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,C,F,H,W", [(1, 1, 1, 2, 2), (3, 1, 2, 4, 6), (3, 2, 1, 2, 8), (2, 16, 3, 6, 10),
                                       (1, 16, 2, 60, 104), (1, 16, 21, 90, 160)])
@pytest.mark.parametrize("order", [0, 1])
def test_patch_permute(ops, order, B, C, F, H, W):
    """Patchify exact against the torch permute, unpatchify exact as its inverse (the patchify of its output is its
    input), and patchify then unpatchify the identity; C = 1, H = W = 2, B = 3, non-square grids and the 14B 720p latent
    (21 x 90 x 160).  Outputs sit 2 / 6 bytes off the 16-byte alignment inside sentinel buffers."""
    g = torch.Generator(device="cuda").manual_seed(B * C * F * H * W + order)
    n, Sp = B * C * F * H * W, F * (H // 2) * (W // 2)
    x = _rnd(g, B, C, F, H, W)
    p = Guarded(n, shift=1)
    ops.patch_permute(x, p.view(B, Sp, 4 * C), B, C, F, H, W, order, False)
    _same_bits(p.view(B, Sp, 4 * C), _patchify_ref(x, order), f"patchify order {order}")
    p.check("patchify")
    y = Guarded(n, shift=3)
    ops.patch_permute(p.view(B, Sp, 4 * C), y.view(B, C, F, H, W), B, C, F, H, W, order, True)
    _same_bits(y.view(B, C, F, H, W), x, f"unpatchify(patchify) order {order}")
    y.check("unpatchify")
    q = _rnd(g, B, Sp, 4 * C)
    z = Guarded(n, shift=1)
    ops.patch_permute(q, z.view(B, C, F, H, W), B, C, F, H, W, order, True)
    _same_bits(_patchify_ref(z.view(B, C, F, H, W), order), q, f"patchify(unpatchify) order {order}")
    z.check("unpatchify of rows")


# ---------------------------------------------------------------------------------------------------------------------
# F. refusals: every documented error code of the seven entry points; each refused call leaves every output untouched
# ---------------------------------------------------------------------------------------------------------------------
def test_refuse_layer_norm_affine(ops):
    R, D, eps = 4, 72, 1e-6
    x, dy, dxin = (torch.randn(R, D, device="cuda").bfloat16() for _ in range(3))
    w, b = torch.ones(D, device="cuda").bfloat16(), torch.zeros(D, device="cuda").bfloat16()
    tab, temb = torch.zeros(6, D, device="cuda").bfloat16(), torch.zeros(2, 6 * D, device="cuda").bfloat16()
    y, dx, o2 = Guarded(R * D), Guarded(R * D), Guarded(R * D)
    fwd = dict(x=x, y=y.view(R, D), weight=w, bias=b)
    runf = lambda rows=R, D=D, **kw: ops.layer_norm_affine_fwd(**dict(fwd, **kw), rows=rows, D=D, eps=eps)
    for k in ("y", "weight", "bias"):
        _raises_code(ARG, lambda: runf(**{k: None}))
    for k in ("x", "y", "weight", "bias"):
        _raises_code(ALIGN, lambda: runf(**{k: _mis(fwd[k])}))
    for r, d in ((0, D), (R, 0), (R, 68), (R, 8200)):
        _raises_code(SHAPE, lambda: runf(rows=r, D=d))
    y.check("layer_norm_affine_fwd refused", [])

    bwd = dict(dy=dy, x=x, dx_in=dxin, dx_out=dx.view(R, D), weight=w, gate2_tab=tab[2], gate2_emb=temb[:, 2 * D:],
               out2=o2.view(R, D), emb_stride=6 * D)
    runb = lambda rows=R, D=D, rps=2, **kw: ops.layer_norm_affine_bwd(**dict(bwd, **kw), rows=rows, D=D, eps=eps,
                                                                      rows_per_sample=rps)
    for k in ("x", "dx_out", "weight", "gate2_tab", "gate2_emb"):      # a missing gate pointer with out2 set
        _raises_code(ARG, lambda: runb(**{k: None}))
    for k in ("dy", "x", "dx_in", "dx_out", "weight", "gate2_tab", "gate2_emb", "out2"):
        _raises_code(ALIGN, lambda: runb(**{k: _mis(bwd[k])}))
    _raises_code(ALIGN, lambda: runb(emb_stride=6 * D + 4))
    for r, d, rps in ((0, D, 2), (R, 68, 2), (R, 8200, 2), (R, D, 0)):
        _raises_code(SHAPE, lambda: runb(rows=r, D=d, rps=rps))
    dx.check("layer_norm_affine_bwd refused dx", [])
    o2.check("layer_norm_affine_bwd refused out2", [])


@pytest.mark.parametrize("hd", [64, 128])
def test_refuse_qkv_ph(ops, hd):
    p = PhProblem(2, 7, 2, hd, 3, 0b111, 0b011, seed=5)
    B, S, H = p.B, p.S, p.H
    n = B * H * S * hd
    dsts = [Guarded(n) for _ in range(3)]
    dv = [d.view(B, H, S, hd) for d in dsts]
    dx = Guarded(p.rows * p.ld_dx)
    dxv = dx.view(p.rows, p.ld_dx)

    def fwd(src=p.src, ld=p.ld, col_off=p.col_off, w=p.w, rope=0b011, cos=p.cos, sin=p.sin, d=dv, H=H, head_dim=hd,
            rows_per_w=0, w_stride=0):
        ops.qkv_norm_rope_fwd(src, ld, col_off, w, rope, cos, sin, d, B, S, H, p.eps, rows_per_w=rows_per_w,
                              w_stride=w_stride, head_dim=head_dim, per_head=True)

    def bwd(x=p.src, ld=p.ld, col_off=p.col_off, w=p.w, rope=0b011, cos=p.cos, sin=p.sin, dy=p.dy, dxt=dxv,
            ld_dx=p.ld_dx, dx_col_off=p.dx_col_off, H=H, head_dim=hd, rows_per_w=0, w_stride=0):
        ops.qkv_norm_rope_bwd(dy, x, ld, col_off, w, rope, cos, sin, dxt, ld_dx, dx_col_off, B, S, H, p.eps,
                              rows_per_w=rows_per_w, w_stride=w_stride, head_dim=head_dim, per_head=True)

    for run in (fwd, bwd):
        for bad_hd in (96, 32, 256):
            _raises_code(SHAPE, lambda: run(head_dim=bad_hd))
        _raises_code(SHAPE, lambda: run(H=8192 // hd + 1))                      # D > 8192
        _raises_code(SHAPE, lambda: run(cos=None, sin=None))                    # rope without tables
        _raises_code(ARG, lambda: run(rope=0b1000))                             # a rope bit at nseg
        _raises_code(ARG, lambda: run(rope=-1))
        _raises_code(ARG, lambda: run(rows_per_w=-1))
        _raises_code(ARG, lambda: run(rows_per_w=7, w_stride=4))
        _raises_code(ALIGN, lambda: run(ld=p.ld + 4))
        _raises_code(ALIGN, lambda: run(col_off=p.col_off + 4))
        _raises_code(ALIGN, lambda: run(cos=_mis(p.cos)))
        _raises_code(ALIGN, lambda: run(sin=_mis(p.sin)))
        for i in range(3):
            _raises_code(ALIGN, lambda: run(w=[_mis(w) if j == i else w for j, w in enumerate(p.w)]))
    _raises_code(ALIGN, lambda: fwd(src=_mis(p.src)))
    _raises_code(ALIGN, lambda: bwd(x=_mis(p.src)))
    _raises_code(ALIGN, lambda: bwd(dxt=_mis(dxv)))
    _raises_code(ALIGN, lambda: bwd(ld_dx=p.ld_dx + 4))
    _raises_code(ALIGN, lambda: bwd(dx_col_off=p.dx_col_off + 4))
    for i in range(3):
        _raises_code(ALIGN, lambda: fwd(d=[_mis(t) if j == i else t for j, t in enumerate(dv)]))
        _raises_code(ARG, lambda: fwd(d=[None if j == i else t for j, t in enumerate(dv)]))
        _raises_code(ALIGN, lambda: bwd(dy=[_mis(t) if j == i else t for j, t in enumerate(p.dy)]))
        if i > 0:   # dy_0 is the pointer the entry point binds the device with: NULL there fails before the checks
            _raises_code(ARG, lambda: bwd(dy=[None if j == i else t for j, t in enumerate(p.dy)]))
    _raises_code(ARG, lambda: fwd(w=p.w[:2], d=dv[:2], rope=0b100))           # a rope bit at nseg = 2
    _raises_code(ARG, lambda: bwd(w=p.w[:1], dy=p.dy[:1], rope=0b10))
    for d in dsts:
        d.check("qkv_norm_rope_ph_fwd refused", [])
    dx.check("qkv_norm_rope_ph_bwd refused", [])


def test_refuse_rope_table_prep_permute(ops):
    from finetrainers_b200 import lib
    cos, sin = Guarded(8 * 64, torch.float32), Guarded(8 * 64, torch.float32)
    for hd in (7, 4, 0, -6):
        _raises_code(SHAPE, lambda: ops.rope_table_wan(cos.t, sin.t, 2, 2, 2, hd))
    for F, H, W in ((0, 2, 2), (2, -1, 2), (2, 2, 0)):
        _raises_code(SHAPE, lambda: ops.rope_table_wan(cos.t, sin.t, F, H, W, 128))
    _raises_code(ARG, lambda: ops.rope_table_wan(cos.t, None, 2, 2, 2, 128))
    cos.check("rope_table_wan refused cos", [])
    sin.check("rope_table_wan refused sin", [])

    B, Cc, F, H, W = 2, 3, 2, 4, 6
    n = B * Cc * F * H * W
    bf = lambda *s: torch.randn(*s, device="cuda").bfloat16()
    mom, eps, noise = bf(B, 2 * Cc, F, H, W), bf(B, Cc, F, H, W), bf(B, Cc, F, H, W)
    mean, std, sig = torch.zeros(B, Cc, device="cuda"), torch.ones(B, Cc, device="cuda"), torch.rand(B, device="cuda")
    xt, tg = Guarded(n), Guarded(n)
    prep = dict(moments=mom, eps=eps, noise=noise, mean=mean, std=std, sigma=sig, x_t=xt.t, target=tg.t)
    runp = lambda shape=(B, Cc, F, H, W), **kw: ops.wan_prep(*dict(prep, **kw).values(), *shape)
    for k in ("eps", "noise", "mean", "std", "sigma", "x_t", "target"):
        _raises_code(ARG, lambda: runp(**{k: None}))
    for shape in ((B, Cc, F, 3, W), (B, Cc, F, H, 5), (0, Cc, F, H, W), (B, 0, F, H, W), (B, Cc, 0, H, W),
                  (B, Cc, F, 0, W), (B, Cc, F, H, -2)):
        _raises_code(SHAPE, lambda: runp(shape))
    xt.check("wan_prep refused x_t", [])
    tg.check("wan_prep refused target", [])

    x = bf(B, Cc, F, H, W)
    x0 = x.clone()
    dst = Guarded(n)

    def perm(src=x, d=dst.t, shape=(B, Cc, F, H, W), order=0, unpatchify=0):
        lib.check(lib.load().b2d_patch_permute(C.c_void_p(src.data_ptr()), C.c_void_p(d.data_ptr()) if d is not None
                                               else None, *shape, order, unpatchify, ops._stream()), "patch_permute")

    for order, unp in ((2, 0), (-1, 0), (0, 2), (1, -1)):
        _raises_code(ARG, lambda: perm(order=order, unpatchify=unp))
    _raises_code(ARG, lambda: perm(d=None))
    _raises_code(ARG, lambda: perm(d=x))                                       # src == dst
    for shape in ((B, Cc, F, 3, W), (B, Cc, F, H, 7), (0, Cc, F, H, W), (B, Cc, F, 0, W), (B, -1, F, H, W)):
        _raises_code(SHAPE, lambda: perm(shape=shape))
    dst.check("patch_permute refused", [])
    _same_bits(x, x0, "patch_permute src == dst refused")


# ---------------------------------------------------------------------------------------------------------------------
# G. coverage: the widths above reach every instantiation they claim to
# ---------------------------------------------------------------------------------------------------------------------
def test_every_instantiation_launches(ops):
    """One small case per instantiation under torch.profiler: the 12 per_head_rope_qk_norm_{fwd,bwd}_kernel<NCH, HD>
    (NCH 1, 2, 4; HD 64, 128) and the 6 affine norm_modulate_{fwd,bwd}_kernel<NCH, true> all launch."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for hd, heads in ((64, (32, 33, 128)), (128, (16, 17, 64))):
            for H in heads:
                p = PhProblem(1, 3, H, hd, 3, 0b011, 0b011, seed=H)
                p.run_fwd(ops)
                p.run_bwd(ops)
        for D in (2048, 2056, 8192):
            _affine_case(ops, 4, D, 2, seed=D)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    ph = {(m[1], int(m[2]), int(m[3])) for nm in names
          for m in [re.search(r"per_head_rope_qk_norm_(fwd|bwd)_kernel<(\d+), (\d+)>", nm)] if m}
    aff = {(m[1], int(m[2])) for nm in names for m in [re.search(r"norm_modulate_(fwd|bwd)_kernel<(\d+), true>", nm)] if m}
    print("\nlaunched:", sorted(ph), sorted(aff))
    assert ph == {(d, n, hd) for d in ("fwd", "bwd") for n in (1, 2, 4) for hd in (64, 128)}, sorted(ph)
    assert aff == {(d, n) for d in ("fwd", "bwd") for n in (1, 2, 4)}, sorted(aff)
