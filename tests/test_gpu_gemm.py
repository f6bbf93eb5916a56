"""GEMM conformance: b2d_gemm against fp64 references computed on the GPU from the same bf16 operands.

Three layers, each with its own bound:
  (a) accumulation - EPI_F32_STORE / EPI_STORE against the exact fp64 product, per element:
      |got - ref| <= ulp_out(ref) + GAMMA * |alpha| * (|A| |B|^T + |A2| |B2|^T)
  (b) epilogues - every other epilogue against its formula applied in fp64 to the kernel's own EPI_F32_STORE result of
      the same launch configuration (same operands, block_n, cta_pair and layout run the same main loop, which (c) pins)
  (c) bounds, determinism and equivalences - every output lives inside a larger buffer filled with a sentinel bit
      pattern that must survive outside the logical output windows; repeated and paired launches are bitwise equal.

Shapes are ragged in M, N and K at once unless a case says otherwise (M % 128, N % block_n and K % 64 all nonzero), and
the leading dimensions of out/out2/res/aux differ from each other and from N, so that an index that uses the wrong one
fails."""
import math

import pytest
import torch

from _gemm_case import assert_same, load_ops
from _util import absmm64, bf16_ulp, check_bound, check_sentinel, f32_ulp, mm64, sentinel_buffer, window

pytestmark = pytest.mark.gpu

# Accumulation error per unit of |A| |B|^T.  Measured on an H100 80GB HBM3 at a 400 W power limit, the worst
# error / bound ratio of EPI_F32_STORE over every case of test_accumulation was 0.066 (errors below 2^-19.9 |A| |B|^T);
# EPI_STORE reached 0.498, its bf16 rounding.  Every epilogue bound of part (b) stayed at or below 0.5 (its rounding).
GAMMA = 2.0 ** -16

EPI = dict(STORE=0, GELU=1, SILU=2, GATE_RES=3, MUL_DGELU=4, F32_ATOMIC=5, F32_ATOMIC_T=6, F32_STORE=7)


@pytest.fixture(scope="module")
def ops():
    return load_ops()


WORST = {}   # layer -> worst error / bound ratio seen in this run (printed at the end of the module)


def _bound(layer, got, ref, bound, what):
    r = check_bound(got, ref, bound, what)
    WORST[layer] = max(WORST.get(layer, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst error/bound ratio per layer:", {k: round(v, 4) for k, v in sorted(WORST.items())})


def _up8(x):
    return (x + 7) // 8 * 8


class Problem:
    """Operands of one (possibly batched, possibly LoRA-extended) GEMM and its fp64 reference.

    Batch z reads the window of each operand's storage that starts z * (row offset) rows and z * (column offset) columns
    further in; storage columns beyond a window (leading-dimension padding, neighbouring batches) hold random values, so
    reading them changes the result."""

    def __init__(self, M, N, K, a_mn=False, b_mn=False, K2=0, group=0, batch=1, a_boff=(0, 0), b_boff=(0, 0),
                 a2_boff_row=0, b2_boff_row=0, bias=True, bias_boff=0, alpha=0.75, seed=0):
        self.M, self.N, self.K, self.K2, self.group, self.batch = M, N, K, K2, group, batch
        self.a_mn, self.b_mn, self.a_boff, self.b_boff = a_mn, b_mn, a_boff, b_boff
        self.a2_boff_row, self.b2_boff_row, self.bias_boff, self.alpha = a2_boff_row, b2_boff_row, bias_boff, alpha
        g = torch.Generator(device="cuda").manual_seed(seed)

        def rnd(r, c, s):
            return (torch.randn(r, _up8(c), device="cuda", generator=g) * s).bfloat16()

        self.ashape = (K, M) if a_mn else (M, K)
        self.bshape = (K, N) if b_mn else (N, K)
        z = batch - 1
        self.A = rnd(self.ashape[0] + z * a_boff[0], self.ashape[1] + z * a_boff[1], 1.0)
        self.B = rnd(self.bshape[0] + z * b_boff[0], self.bshape[1] + z * b_boff[1], K ** -0.5)
        self.groups = (N + group - 1) // group if group else 1
        if K2:
            self.A2 = rnd(M + z * a2_boff_row, K2 * self.groups, 1.0)
            self.B2 = rnd(K2 + z * b2_boff_row, N, K2 ** -0.5) if b_mn else rnd(N + z * b2_boff_row, K2, K2 ** -0.5)
        self.bias = (torch.randn(N + z * bias_boff, device="cuda", generator=g)).bfloat16() if bias else None

    def a(self, z):  # [M, K] view of batch z
        r0, c0 = z * self.a_boff[0], z * self.a_boff[1]
        v = self.A[r0:r0 + self.ashape[0], c0:c0 + self.ashape[1]]
        return v.t() if self.a_mn else v

    def b(self, z):  # [N, K]
        r0, c0 = z * self.b_boff[0], z * self.b_boff[1]
        v = self.B[r0:r0 + self.bshape[0], c0:c0 + self.bshape[1]]
        return v.t() if self.b_mn else v

    def ref(self, z):
        """(alpha * (A B^T + A2 B2^T) + bias, |alpha| (|A| |B|^T + |A2| |B2|^T)) of batch z, fp64."""
        acc, scl = mm64(self.a(z), self.b(z)), absmm64(self.a(z), self.b(z))
        if self.K2:
            a2 = self.A2[z * self.a2_boff_row:z * self.a2_boff_row + self.M]
            r0 = z * self.b2_boff_row
            b2 = self.B2[r0:r0 + self.K2].t() if self.b_mn else self.B2[r0:r0 + self.N]
            gw = self.group or self.N
            for gi in range(self.groups):
                cols = slice(gi * gw, min(self.N, (gi + 1) * gw))
                acc[:, cols] += mm64(a2[:, gi * self.K2:(gi + 1) * self.K2], b2[cols])
                scl[:, cols] += absmm64(a2[:, gi * self.K2:(gi + 1) * self.K2], b2[cols])
        pre = self.alpha * acc
        if self.bias is not None:
            pre = pre + self.bias[z * self.bias_boff:z * self.bias_boff + self.N].double()
        return pre, abs(self.alpha) * scl

    def run(self, ops, out, ldc, epi="STORE", c_boff=0, bias=True, **kw):
        """Launch into `out` (a flat buffer: batch z's [M, N] window starts at z * c_boff, leading dimension ldc)."""
        ext = {}
        if self.K2:
            ext = dict(A2=self.A2, B2=self.B2, K2=self.K2, a2_group_n=self.group, a2_boff_row=self.a2_boff_row,
                       b2_boff_row=self.b2_boff_row)
        ops.gemm(self.A, self.B, out, M=self.M, N=self.N, K=self.K, ldc=ldc, a_mn=self.a_mn, b_mn=self.b_mn,
                 batch=self.batch, a_boff=self.a_boff, b_boff=self.b_boff, c_boff=c_boff, epi=EPI[epi], alpha=self.alpha,
                 bias=self.bias if bias else None, bias_boff=self.bias_boff, **ext, **kw)
        return out


def out_buffer(rows, cols, ld, dtype, batch=1, c_boff=0, zero=False):
    """Sentinel-filled flat buffer holding `batch` [rows, cols] windows (leading dimension ld, batch stride c_boff), with
    32 elements of margin after the last; returns (buffer, windows)."""
    n = (batch - 1) * c_boff + rows * ld + 32
    buf = sentinel_buffer(n, dtype)
    wins = [window(buf, z * c_boff, rows, cols, ld) for z in range(batch)]
    if zero:
        for w in wins:
            w.zero_()
    return buf, wins


# ---------------------------------------------------------------------------------------------------------------------
# (a) accumulation
# ---------------------------------------------------------------------------------------------------------------------
def _acc_cases():
    cases = []
    M, N, K = 300, 200, 200          # M % 128 = 44, N % bn != 0 for every bn, K % 64 = 8
    for a_mn in (False, True):
        for b_mn in (False, True):
            for bn in (64, 128, 160, 192, 256):
                if a_mn and bn == 160:
                    continue
                for pair in (1, 2):
                    if pair == 2 and (a_mn or bn == 64):
                        continue
                    cases.append(pytest.param(dict(M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn), dict(block_n=bn, cta_pair=pair),
                                              id=f"a{int(a_mn)}b{int(b_mn)}-bn{bn}-p{pair}"))
    # M <= 128 (one M tile), K below one k-block, alpha = 1 without bias
    cases.append(pytest.param(dict(M=100, N=136, K=40, alpha=1.0, bias=False), dict(block_n=128), id="m100-k40"))
    cases.append(pytest.param(dict(M=128, N=72, K=520, b_mn=True, alpha=-1.5), dict(block_n=64), id="m128-bmn"))
    # LoRA extension, with and without per-group A2 slices
    for b_mn in (False, True):
        for pair in (1, 2):
            cases.append(pytest.param(dict(M=300, N=200, K=200, b_mn=b_mn, K2=64), dict(block_n=128, cta_pair=pair),
                                      id=f"k2-b{int(b_mn)}-p{pair}"))
            cases.append(pytest.param(dict(M=300, N=712, K=200, b_mn=b_mn, K2=128, group=256),
                                      dict(block_n=256 if pair == 2 else 128, cta_pair=pair),
                                      id=f"k2group-b{int(b_mn)}-p{pair}"))
    # batched: every offset at once (K a whole number of k-blocks, so offsets may run along K); ragged K with offsets
    # along M / N only
    for a_mn in (False, True):
        for b_mn in (False, True):
            bo = dict(batch=3, a_boff=(40, 64) if not a_mn else (64, 40), b_boff=(24, 128) if not b_mn else (128, 24),
                      bias_boff=16)
            cases.append(pytest.param(dict(M=300, N=200, K=192, a_mn=a_mn, b_mn=b_mn, **bo), dict(block_n=64 if a_mn else 192),
                                      id=f"batch-a{int(a_mn)}b{int(b_mn)}"))
            bo = dict(batch=2, a_boff=(310, 0) if not a_mn else (0, 312), b_boff=(208, 0) if not b_mn else (0, 208))
            cases.append(pytest.param(dict(M=300, N=200, K=200, a_mn=a_mn, b_mn=b_mn, **bo), dict(block_n=128),
                                      id=f"batch-ktail-a{int(a_mn)}b{int(b_mn)}"))
    for b_mn in (False, True):
        bo = dict(batch=3, a_boff=(0, 64), b_boff=(128, 0) if b_mn else (208, 0), K2=64, a2_boff_row=300,
                  b2_boff_row=64 if b_mn else 200, bias_boff=8)
        cases.append(pytest.param(dict(M=300, N=200, K=192, b_mn=b_mn, **bo), dict(block_n=128, cta_pair=2),
                                  id=f"batch-pairs-k2-b{int(b_mn)}"))
    # long LoRA extensions (adapter ranks padded to 192 and 256).  The forward QKV / kv2 form: per-group A2 slices of
    # K2 = rp columns each
    for K2 in (192, 256):
        cases.append(pytest.param(dict(M=300, N=712, K=200, K2=K2, group=256), dict(block_n=128), id=f"k2group-{K2}"))
    # the backward dX form (MN-major B, K2 = 3 rp): with K = 200 (four k-blocks, the last ragged) the 6, 9 and 12
    # extension k-blocks alone wrap the 5-stage ring of block_n 128, and at 9 and 12 also the 8-stage ring of block_n 64
    for K2 in (384, 576, 768):
        for bn in (64, 128):
            cases.append(pytest.param(dict(M=300, N=200, K=200, b_mn=True, K2=K2), dict(block_n=bn),
                                      id=f"k2long-{K2}-bn{bn}"))
    # the kv2 form: one batched launch over blocks, each with its own B, A2 rows and B2 rows, shared A, per-group A2 slices
    cases.append(pytest.param(dict(M=300, N=512, K=192, batch=3, b_boff=(520, 0), K2=256, group=256, a2_boff_row=300,
                                   b2_boff_row=528, bias_boff=512), dict(block_n=128), id="batch-kv2-k2-256"))
    # the step's shapes, automatic tile
    for N in (2048, 6144, 8192):
        for K in (2048, 8192):
            cases.append(pytest.param(dict(M=2688, N=N, K=K, alpha=1.0), dict(), id=f"step-{N}x{K}"))
    return cases


@pytest.mark.parametrize("prob,launch", _acc_cases())
def test_accumulation(ops, prob, launch):
    """EPI_F32_STORE and EPI_STORE against the fp64 product.  Worst error / bound ratio on an H100 80GB HBM3 with
    GAMMA = 2^-16: 0.066 for EPI_F32_STORE, 0.498 for EPI_STORE (see GAMMA)."""
    p = Problem(**prob)
    M, N, batch = p.M, p.N, p.batch
    ldc = _up8(N + 24)
    c_boff = M * ldc + 40 if batch > 1 else 0      # gaps between the batch slices
    refs = [p.ref(z) for z in range(batch)]
    for epi, dtype, ulp in (("F32_STORE", torch.float32, f32_ulp), ("STORE", torch.bfloat16, bf16_ulp)):
        buf, wins = out_buffer(M, N, ldc, dtype, batch, c_boff)
        p.run(ops, buf, ldc, epi, c_boff=c_boff, **launch)
        check_sentinel(buf, wins, epi)
        for z, (pre, scl) in enumerate(refs):
            _bound(f"acc {epi}", wins[z], pre, ulp(pre) + GAMMA * scl, f"{epi} batch {z}")


@pytest.mark.parametrize("a_mn,b_mn", [(True, True), (False, False), (False, True)])
@pytest.mark.parametrize("splits", [1, 2, 3])
@pytest.mark.parametrize("bn", [64, 128])
def test_split_k_atomics(ops, a_mn, b_mn, splits, bn):
    """EPI_F32_ATOMIC (out[row, col] +=) and EPI_F32_ATOMIC_T (out[col, row] +=) over 1..3 k-splits, into a nonzero
    accumulator, against the fp64 product."""
    p = Problem(M=300, N=200, K=392, a_mn=a_mn, b_mn=b_mn, bias=False, alpha=0.625, seed=splits)
    pre, scl = p.ref(0)
    init = torch.randn(p.M, p.N, device="cuda")
    buf, (w,) = out_buffer(p.M, p.N, 216, torch.float32)
    w.copy_(init)
    p.run(ops, buf, 216, "F32_ATOMIC", splits=splits, block_n=bn)
    check_sentinel(buf, [w], "F32_ATOMIC")
    _bound("F32_ATOMIC", w, pre + init.double(), f32_ulp(pre + init.double()) + f32_ulp(init) + GAMMA * scl, "F32_ATOMIC")
    bufT, (wT,) = out_buffer(p.N, p.M, 312, torch.float32)
    wT.copy_(init.t())
    p.run(ops, bufT, 312, "F32_ATOMIC_T", splits=splits, block_n=bn)
    check_sentinel(bufT, [wT], "F32_ATOMIC_T")
    ref = (pre + init.double()).t()
    _bound("F32_ATOMIC_T", wT, ref, f32_ulp(ref) + f32_ulp(init.t()) + GAMMA * scl.t(), "F32_ATOMIC_T")


# ---------------------------------------------------------------------------------------------------------------------
# (b) epilogues
# ---------------------------------------------------------------------------------------------------------------------
# Samples of 197 rows: a sample boundary falls inside 128-row tiles and between the two rows (row0, row0 + 8) one thread
# stores whenever it is not a multiple of 16.
RPS, NB = 197, 3
EPI_CASES = [
    pytest.param((dict(), dict(block_n=128)), id="a0b0-bn128"),
    pytest.param((dict(b_mn=True, K2=64), dict(block_n=128, cta_pair=2)), id="a0b1-k2-bn128-p2"),
    pytest.param((dict(b_mn=True), dict(block_n=160)), id="a0b1-bn160"),
    pytest.param((dict(a_mn=True), dict(block_n=192)), id="a1b0-bn192"),
    pytest.param((dict(a_mn=True, b_mn=True), dict(block_n=64)), id="a1b1-bn64"),
    pytest.param((dict(K2=128, group=256, N=712), dict(block_n=256, cta_pair=2)), id="a0b0-k2group-bn256-p2"),
    # the backward dh GEMM of an adapter padded to rank 128 (K2 = 3 rp = 384): the extension wraps the ring on its own
    pytest.param((dict(b_mn=True, K2=384), dict(block_n=128)), id="a0b1-k2long384-bn128"),
]
LDC, LDC2, LDRES, LDAUX = 24, 40, 56, 72   # added to N: all different, ldres and ldaux the largest


def _gelu64(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))


def _dgelu64(x):
    u = math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)
    t = torch.tanh(u)
    return 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * math.sqrt(2 / math.pi) * (1 + 3 * 0.044715 * x * x)


class EpiRun:
    """One configuration of part (b): the problem, its pre-activation from EPI_F32_STORE, and a launcher."""

    def __init__(self, ops, prob, launch):
        kw = dict(M=NB * RPS, N=200, K=200)
        kw.update(prob)
        self.ops, self.p, self.launch = ops, Problem(**kw, seed=11), launch
        p = self.p
        self.M, self.N = p.M, p.N
        self.ldc, self.ldc2, self.ldres, self.ldaux = (p.N + d for d in (LDC, LDC2, LDRES, LDAUX))
        buf, (w,) = out_buffer(p.M, p.N, self.ldc, torch.float32)
        p.run(ops, buf, self.ldc, "F32_STORE", **launch)
        check_sentinel(buf, [w], "F32_STORE")
        self.pre32 = w.clone()
        self.pre = self.pre32.double()

    def run(self, epi, out2=False, **kw):
        buf, (w,) = out_buffer(self.M, self.N, self.ldc, torch.bfloat16)
        wins2 = None
        if out2:
            buf2, wins2 = out_buffer(self.M, self.N, self.ldc2, torch.bfloat16)
            kw.update(out2=buf2, ldc2=self.ldc2)
        self.p.run(self.ops, buf, self.ldc, epi, **self.launch, **kw)
        check_sentinel(buf, [w], f"{epi} out")
        if out2:
            check_sentinel(buf2, wins2, f"{epi} out2")
            return w, wins2[0]
        return w


@pytest.fixture(scope="module", params=EPI_CASES)
def epi_run(ops, request):
    prob, launch = request.param
    return EpiRun(ops, prob, launch)


def test_epilogue_store_and_activations(epi_run):
    """EPI_STORE and the out2 of GELU/SILU are the fp32 pre-activation rounded to bf16, bit for bit.  GELU is within
    1 bf16 ulp + 2^-12 |pre|: tanh.approx.f32 has an absolute error below 2^-11 and gelu = x/2 (1 + tanh(.)).  SILU is
    within 1 ulp + 2^-20 |pre| (__expf and __fdividef: a few fp32 ulps)."""
    r = epi_run
    want = r.pre32.bfloat16()
    assert_same([r.run("STORE")], [want], "STORE")
    out, o2 = r.run("GELU", out2=True)
    assert_same([o2], [want], "GELU out2")
    ref = _gelu64(r.pre)
    _bound("GELU", out, ref, bf16_ulp(ref) + 2.0 ** -12 * r.pre.abs(), "GELU")
    out, o2 = r.run("SILU", out2=True)
    assert_same([o2], [want], "SILU out2")
    ref = r.pre * torch.sigmoid(r.pre)
    _bound("SILU", out, ref, bf16_ulp(ref) + 2.0 ** -20 * r.pre.abs(), "SILU")
    out = r.run("GELU")           # without out2
    _bound("GELU", out, _gelu64(r.pre), bf16_ulp(_gelu64(r.pre)) + 2.0 ** -12 * r.pre.abs(), "GELU no out2")


def test_epilogue_mul_dgelu(epi_run):
    """out = pre * gelu_tanh'(aux) within 1 ulp + 2^-10 |pre| (1 + |aux|): the tanh.approx error (< 2^-11) enters
    gelu'(x) = (1 + t) / 2 + x (1 - t^2) (k0 + 3 k0 k1 x^2) / 2 with weight |1/2 - x t (k0 + 3 k0 k1 x^2)|, which stays
    below 2 (1 + |x|) while tanh is not saturated (|x| < 4)."""
    r = epi_run
    g = torch.Generator(device="cuda").manual_seed(5)
    aux = torch.randn(r.M, r.ldaux, device="cuda", generator=g).bfloat16()
    out = r.run("MUL_DGELU", aux=aux, ldaux=r.ldaux)
    x = aux[:, :r.N].double()
    ref = r.pre * _dgelu64(x)
    _bound("MUL_DGELU", out, ref, bf16_ulp(ref) + 2.0 ** -10 * r.pre.abs() * (1 + x.abs()), "MUL_DGELU")


GATE_VARIANTS = ["gate+gate2", "gate", "none", "gate2"]


@pytest.mark.parametrize("variant", GATE_VARIANTS + ["in-place"])
def test_epilogue_gate_res(epi_run, variant):
    """out = res + g * pre (g = gate_table + gate_temb[sample], or 1 without a gate) within 1 bf16 ulp + 2^-22 of the
    terms' magnitudes (fp32 gate sum and fma); out2 = bf16(out) * g2 within 1 ulp of the kernel's own primary output
    times the second gate: what is gated is the rounded primary."""
    r = epi_run
    g = torch.Generator(device="cuda").manual_seed(7)
    M, N = r.M, r.N
    res = (torch.randn(M, r.ldres, device="cuda", generator=g)).bfloat16()
    tab = (torch.randn(6, N, device="cuda", generator=g) * 0.5).bfloat16()
    ts = 6 * N + 8
    temb = (torch.randn(NB, ts, device="cuda", generator=g) * 0.5).bfloat16()
    smp = torch.arange(M, device="cuda") // RPS

    def gate(row):
        return tab[row].double()[None] + temb[:, row * N:(row + 1) * N].double()[smp]

    kw = dict(temb_stride=ts, rows_per_sample=RPS)
    use_g = variant in ("gate+gate2", "gate", "in-place")
    use_g2 = variant in ("gate+gate2", "gate2")
    if use_g:
        kw.update(gate_table=tab[2], gate_temb=temb[:, 2 * N:])
    if use_g2:
        kw.update(gate2_table=tab[5], gate2_temb=temb[:, 5 * N:])
    gv = gate(2) if use_g else torch.ones_like(r.pre)
    if variant == "in-place":
        buf, (w,) = out_buffer(M, N, r.ldc, torch.bfloat16)
        w.copy_(res[:, :N])
        resv = w.double().clone()
        r.p.run(r.ops, buf, r.ldc, "GATE_RES", res=buf, ldres=r.ldc, **r.launch, **kw)
        check_sentinel(buf, [w], "GATE_RES in place")
        out = w
    else:
        resv = res[:, :N].double()
        got = r.run("GATE_RES", out2=use_g2, res=res, ldres=r.ldres, **kw)
        out, o2 = got if use_g2 else (got, None)
    gp = gv * r.pre
    ref = resv + gp
    _bound("GATE_RES", out, ref, bf16_ulp(ref) + 2.0 ** -22 * (resv.abs() + gp.abs()), f"GATE_RES {variant}")
    if use_g2:
        ref2 = out.double() * gate(5)
        _bound("GATE_RES", o2, ref2, bf16_ulp(ref2) + 2.0 ** -22 * ref2.abs(), f"GATE_RES {variant} out2")


def test_epilogue_batched_bias_and_out2(ops):
    """Batched launch: batch z adds bias + z * bias_boff and stores out and out2 at z * c_boff (gaps between slices stay
    untouched); out2 of GELU is bitwise the rounded EPI_F32_STORE result of the same launch."""
    p = Problem(M=300, N=200, K=192, batch=3, a_boff=(0, 64), b_boff=(208, 0), bias_boff=24, seed=3)
    ldc, ldc2 = 224, 232
    c32, c16 = 300 * ldc + 8, 300 * ldc2 + 16      # out and out2 share c_boff
    b32, w32 = out_buffer(300, 200, ldc, torch.float32, 3, c32)
    p.run(ops, b32, ldc, "F32_STORE", c_boff=c32, block_n=128)
    check_sentinel(b32, w32, "F32_STORE")
    b16, w16 = out_buffer(300, 200, ldc, torch.bfloat16, 3, c16)
    b2, w2 = out_buffer(300, 200, ldc2, torch.bfloat16, 3, c16)
    p.run(ops, b16, ldc, "GELU", c_boff=c16, out2=b2, ldc2=ldc2, block_n=128)
    check_sentinel(b16, w16, "GELU out")
    check_sentinel(b2, w2, "GELU out2")
    for z in range(3):
        pre, scl = p.ref(z)
        _bound("F32_STORE", w32[z], pre, f32_ulp(pre) + GAMMA * scl, f"F32_STORE batch {z}")
        assert_same([w2[z]], [w32[z].bfloat16()], f"GELU out2 batch {z}")
        ref = _gelu64(w32[z].double())
        _bound("GELU", w16[z], ref, bf16_ulp(ref) + 2.0 ** -12 * w32[z].double().abs(), f"GELU batch {z}")


# ---------------------------------------------------------------------------------------------------------------------
# (c) determinism and equivalences
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn", [128, 160, 192, 256])
@pytest.mark.parametrize("b_mn", [False, True])
def test_pairs_equal_single_ctas_and_repeat_bitwise(ops, bn, b_mn):
    """A CTA pair computes exactly what two single CTAs compute at the same tile width, and a launch repeated gives the
    same bits (GATE_RES with both gates, the LoRA extension and ragged M/N/K: the model's backward dX launch)."""
    p = Problem(M=NB * RPS, N=200, K=200, b_mn=b_mn, K2=64, seed=bn)
    N, M = p.N, p.M
    g = torch.Generator(device="cuda").manual_seed(1)
    res = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    tab = torch.randn(2, N, device="cuda", generator=g).bfloat16()
    temb = torch.randn(NB, 2 * N, device="cuda", generator=g).bfloat16()
    kw = dict(res=res, gate_table=tab[0], gate_temb=temb, gate2_table=tab[1], gate2_temb=temb[:, N:], temb_stride=2 * N,
              rows_per_sample=RPS)
    outs = []
    for pair in (1, 2, 2):
        o, o2 = torch.empty(M, N, device="cuda", dtype=torch.bfloat16), torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        p.run(ops, o, N, "GATE_RES", out2=o2, block_n=bn, cta_pair=pair, **kw)
        o32 = torch.empty(M, N, device="cuda")
        p.run(ops, o32, N, "F32_STORE", block_n=bn, cta_pair=pair)
        outs.append((o, o2, o32))
    for i, what in enumerate(("out", "out2", "f32")):
        assert_same([outs[1][i]], [outs[0][i]], f"pair vs single {what}")
        assert_same([outs[2][i]], [outs[1][i]], f"repeat {what}")


@pytest.mark.parametrize("a_mn,b_mn,bn", [(True, True, 64), (False, False, 128), (False, True, 192)])
def test_atomic_equals_store(ops, a_mn, b_mn, bn):
    """With one split, EPI_F32_ATOMIC into zeros equals EPI_F32_STORE without bias, and EPI_F32_ATOMIC_T equals its
    transpose (0 + v = v, and every element is added once)."""
    p = Problem(M=300, N=200, K=200, a_mn=a_mn, b_mn=b_mn, bias=False, seed=9)
    st = torch.empty(300, 200, device="cuda")
    p.run(ops, st, 200, "F32_STORE", block_n=bn)
    at = torch.zeros(300, 200, device="cuda")
    p.run(ops, at, 200, "F32_ATOMIC", block_n=bn)
    atT = torch.zeros(200, 304, device="cuda")
    p.run(ops, atT, 304, "F32_ATOMIC_T", block_n=bn)
    assert torch.equal(at, st)
    assert torch.equal(atT[:, :300].t(), st) and atT[:, 300:].abs().max() == 0


# ---------------------------------------------------------------------------------------------------------------------
# contract: batched launches whose batch offset runs along a ragged K
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("a_mn,b_mn,along", [(False, False, "a"), (True, True, "a"), (False, False, "b"),
                                             (True, True, "b"), (False, False, "ab"), (True, True, "ab")])
def test_batched_k_tail_offset_along_k_is_rejected(ops, a_mn, b_mn, along):
    """Batched launches widen the tensor-map extents over all batches, so with K % 64 != 0 the last k-block of batch z
    reads batch z + 1's elements instead of zero fill in every operand whose batch offset runs along K.  With both
    operands offset along K that product is wrong (up to 0.29 |A| |B|^T in batch 0 before the check existed).  With one,
    the other operand's tail is zero fill and finite data still give the right result, but a non-finite value in the
    neighbouring batch would turn into 0 * Inf = NaN; the rule stays simple and refuses every such launch with
    B2D_ERR_SHAPE."""
    from finetrainers_b200.lib import B2DError
    K = 200
    ka = (K, 0) if a_mn else (0, K)        # a_boff along K: rows of an MN-major A, columns of a K-major A
    kb = (K, 0) if b_mn else (0, K)
    p = Problem(M=256, N=128, K=K, a_mn=a_mn, b_mn=b_mn, batch=2, bias=False, alpha=1.0,
                a_boff=ka if "a" in along else (0, 0), b_boff=kb if "b" in along else (0, 0))
    out = torch.zeros(2 * 256, 128, device="cuda", dtype=torch.float32)
    try:
        p.run(ops, out, 128, "F32_STORE", c_boff=256 * 128, block_n=128)
    except B2DError as e:
        assert "(code -1)" in str(e), e
        return
    torch.cuda.synchronize()
    errs = []
    for z in range(2):
        pre, scl = p.ref(z)
        errs.append(((out[z * 256:(z + 1) * 256] - pre).abs() / scl.clamp_min(1e-30)).max().item())
    pytest.fail(f"accepted; worst |error| / (|A||B|) per batch: {errs}")
