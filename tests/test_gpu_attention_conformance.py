"""Attention conformance: the forward and backward kernels at head_dim 64 and 128 against an fp64 reference computed on
the GPU from the same bf16 q, k, v, dout and fp32 key bias, with a bound for every output element.

Notation: u = 2^-9 (bf16 rounding unit), GAMMA = fp32 MMA accumulation constant, ulp = bf16 spacing at the reference.
All terms are fp64 matrices built from the same inputs; a row whose keys are all -inf has P = 0 and out = 0 ("safe
softmax", as torch's math SDPA computes it), and the kernel must give it lse = +inf.

  score error      eps_S = GAMMA (scale |Q| |K|^T + |bias|)
  P (relative)     eta_i = u + 2 max_j eps_S,ij + 2^-20   (max over the keys with P_ij > 0)
  out              ulp(O) + 2 eta_i (P |V|) + UF sum_j |V_j|
  lse              4 f32_ulp(lse) + 2 max_j eps_S,ij
  dV               ulp(dV) + 2 (diag(eta) P)^T |dO| + UF sum_i |dO_i|
  delta            Ddelta_i = sum_d |dO| bound_out + GAMMA sum_d |O| |dO|
  dS error         E = u |dS| + P o (GAMMA |dO| |V|^T + Ddelta) + eta o P o |dP - delta| + UF (|dP - delta| + 1)
  dQ               ulp(dQ) + scale (E |K| + GAMMA |dS| |K|)
  dK               ulp(dK) + scale (E^T |Q| + GAMMA |dS|^T |Q|)

Every case scales q, k, v and dout of each (sample, head) by its own power of two, so a lse, delta or bias read for
the wrong (sample, head) fails element-wise.  The worst error/bound ratio per output is printed at the end."""
import math

import pytest
import torch
import torch.nn.functional as F

from _util import bf16_ulp, check_bound, check_sentinel, f32_ulp, sentinel_buffer, window

pytestmark = pytest.mark.gpu

U = 2.0 ** -9
# fp32 accumulation error per unit of the magnitude terms, as in the GEMM suite.  Measured on an H100 80GB HBM3 at a
# 700 W power limit, the worst error/bound ratio over the whole module was out 0.548, lse 0.637, dq 0.216, dk 0.719
# and dv 0.851, with u, GAMMA and the factors of 2 at their first-principles values.
GAMMA = 2.0 ** -16
# The kernels compute exponentials and products with fp32 denormals flushed to zero: every P, dS and product below
# 2^-126 may become 0.  That absolute term only matters where an output is itself near 1e-38.
UF = 2.0 ** -126
WORST = {}


def _check(name, got, ref, bound, what):
    r = check_bound(got, ref, bound, f"{name} {what}")
    WORST[name] = max(WORST.get(name, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst error/bound ratio per output:", {k: round(v, 4) for k, v in sorted(WORST.items())})


def reference(q, k, v, kb, scale, g):
    """fp64 attention, its gradients and their element-wise bounds, query block by query block.
    q [B,H,Sq,d], k/v [B,H,Sk,d], kb [B,Sk] fp32 or None, g = dout [B,H,Sq,d] -> dict of (value, bound) pairs."""
    B, H, Sq, d = q.shape
    Sk = k.shape[2]
    Q, K, V, G = q.double(), k.double(), v.double(), g.double()
    aK, aV = K.abs(), V.abs()
    if kb is None:
        bias = absb = torch.zeros(B, 1, 1, Sk, dtype=torch.float64, device=q.device)
    else:
        bias = kb.double()[:, None, None, :]
        absb = torch.where(torch.isinf(bias), torch.zeros_like(bias), bias.abs())
    out, bout = torch.empty_like(Q), torch.empty_like(Q)
    lse, blse = torch.empty(B, H, Sq, dtype=torch.float64, device=q.device), torch.empty(B, H, Sq, dtype=torch.float64,
                                                                                          device=q.device)
    dq, bdq = torch.empty_like(Q), torch.empty_like(Q)
    dk, bdk, dv, bdv = torch.zeros_like(K), torch.zeros_like(K), torch.zeros_like(V), torch.zeros_like(V)
    chunk = max(1, min(Sq, (1 << 25) // (B * H * Sk)))
    for i in range(0, Sq, chunk):
        sl = slice(i, i + chunk)
        Qi, Gi = Q[:, :, sl], G[:, :, sl]
        aQi, aGi = Qi.abs(), Gi.abs()
        S = Qi @ K.transpose(-1, -2) * scale + bias
        mx = S.amax(-1, keepdim=True)
        off = torch.where(torch.isinf(mx), torch.zeros_like(mx), mx)
        P = torch.exp(S - off)
        del S
        # the score error of keys whose probability underflows to 0 (masked ones) does not reach any output
        eps = GAMMA * (aQi @ aK.transpose(-1, -2) * scale + absb)
        meps = torch.where(P > 0, eps, torch.zeros_like(eps)).amax(-1, keepdim=True)
        del eps
        l = P.sum(-1, keepdim=True)
        P = P / torch.where(l > 0, l, torch.ones_like(l))
        lse[:, :, sl] = torch.where(l > 0, off + torch.log(l), torch.full_like(l, math.inf)).squeeze(-1)
        blse[:, :, sl] = (4 * f32_ulp(torch.where(l > 0, off + torch.log(l), torch.zeros_like(l))) + 2 * meps).squeeze(-1)
        eta = U + 2 * meps + 2.0 ** -20
        O = P @ V
        bO = bf16_ulp(O) + 2 * eta * (P @ aV) + UF * aV.sum(-2, keepdim=True)
        out[:, :, sl], bout[:, :, sl] = O, bO
        dv += P.transpose(-1, -2) @ Gi
        bdv += (eta * P).transpose(-1, -2) @ aGi
        delta = (O * Gi).sum(-1, keepdim=True)
        ddelta = (aGi * bO).sum(-1, keepdim=True) + GAMMA * (O.abs() * aGi).sum(-1, keepdim=True)
        dPd = Gi @ V.transpose(-1, -2) - delta
        dS = P * dPd
        E = U * dS.abs() + P * (GAMMA * (aGi @ aV.transpose(-1, -2)) + ddelta) + eta * P * dPd.abs() + UF * (dPd.abs() + 1)
        del dPd
        aS = dS.abs()
        dq[:, :, sl] = dS @ K * scale
        bdq[:, :, sl] = scale * ((E + GAMMA * aS) @ aK)
        dk += dS.transpose(-1, -2) @ Qi * scale
        bdk += scale * ((E + GAMMA * aS).transpose(-1, -2) @ aQi)
        del P, dS, aS, E
    bdv = 2 * bdv + UF * G.abs().sum(-2, keepdim=True)
    return {"out": (out, bout), "lse": (lse, blse), "dq": (dq, bdq + bf16_ulp(dq)), "dk": (dk, bdk + bf16_ulp(dk)),
            "dv": (dv, bdv + bf16_ulp(dv))}


def check_all(got, ref, what, heads=None):
    """got = (out [B,Sq,H*d] token-major, lse, dq, dk, dv) from the kernels; ref = reference(...) on heads[0:n]."""
    out, lse, dq, dk, dv = got
    B, H, Sq = lse.shape
    d = dq.shape[-1]
    n = H if heads is None else heads
    got = {"out": out.view(B, Sq, H, d).transpose(1, 2)[:, :n], "lse": lse[:, :n], "dq": dq[:, :n], "dk": dk[:, :n],
           "dv": dv[:, :n]}
    r_lse, b_lse = ref["lse"]
    dead = torch.isinf(r_lse)
    assert (got["lse"][dead] == math.inf).all(), f"lse {what}: a row with every key masked must give lse = +inf"
    zero = torch.zeros_like(r_lse)
    _check("lse", torch.where(dead, zero, got["lse"].double()), torch.where(dead, zero, r_lse), b_lse, what)
    for name in ("out", "dq", "dk", "dv"):
        _check(name, got[name], *ref[name], what)


def _run(q, k, v, kb, scale, dout_tok, head_dim):
    """fwd + bwd through ops; out, lse, dq, dk and dv start NaN-filled, so an element the kernels skip fails its
    bound.  Returns out [B,Sq,H*d], lse, dq, dk, dv."""
    from finetrainers_b200 import ops
    B, H, Sq, d = q.shape
    Sk = k.shape[2]
    nan = float("nan")
    out = torch.full((B, Sq, H * d), nan, device="cuda", dtype=torch.bfloat16)
    lse = torch.full((B, H, Sq), nan, device="cuda")
    ops.attn_fwd(q, k, v, kb, out, lse, B, H, Sq, Sk, scale, head_dim=head_dim)
    dq, dk, dv = torch.full_like(q, nan), torch.full_like(k, nan), torch.full_like(v, nan)
    ws = torch.full((ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=head_dim),), nan, device="cuda")
    ops.attn_bwd(q, k, v, kb, out, dout_tok, lse, ws, dq, dk, dv, B, H, Sq, Sk, scale, head_dim=head_dim)
    return out, lse, dq, dk, dv


def mags(B, H, lo=-6, hi=3, gen=None):
    """a power of two per (sample, head), [B, H, 1, 1]"""
    e = torch.randint(lo, hi + 1, (B, H, 1, 1), generator=gen)
    return torch.pow(2.0, e.float()).cuda()


def inputs(B, H, Sq, Sk, d, seed, mag=True):
    """bf16 q, k, v [B,H,S,d] and dout (head-major g, token-major copy), each (b, h) scaled by its own 2^e"""
    gen = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    out = []
    for S in (Sq, Sk, Sk, Sq):
        x = torch.randn(B, H, S, d, device="cuda")
        out.append((x * mags(B, H, gen=gen) if mag else x).bfloat16())
    q, k, v, g = out
    return q, k, v, g, g.transpose(1, 2).reshape(B, Sq, H * d).contiguous()


def key_bias(kind, B, Sk, seed=0):
    """fp32 key bias [B, Sk] of one kind, or None"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    ar = torch.arange(Sk, device="cuda")[None]
    if kind == "none":
        return None
    if kind == "ltx":   # 0 on the kept keys, -10000 on right padding, as the step builds it
        lens = torch.randint(1, Sk + 1, (B,), device="cuda", generator=gen)
        return ((ar >= lens[:, None]).float() * -10000.0).contiguous()
    if kind == "cont":  # moderate values, different per sample (ALiBi-like)
        return (torch.rand(B, Sk, device="cuda", generator=gen) * 16 - 8).contiguous()
    if kind == "dominant":  # one key far above the others, in the ragged last tile
        kb = torch.zeros(B, Sk, device="cuda")
        kb[:, Sk - 1 - (Sk - 1) % 128 + ((Sk - 1) % 128) // 2] = 20.0
        return kb
    if kind.startswith("left"):  # -inf on the first n keys (left padding)
        n = int(kind[4:])
        return torch.zeros(B, Sk, device="cuda").masked_fill(ar < n, float("-inf")).contiguous()
    if kind == "dead":  # sample 0 has every key masked, sample 1 none
        kb = torch.zeros(B, Sk, device="cuda")
        kb[0] = float("-inf")
        return kb
    raise ValueError(kind)


def run_case(B, H, Sq, Sk, d, kind="cont", scale=0.125, seed=0, heads=None, mag=True):
    q, k, v, g, g_tok = inputs(B, H, Sq, Sk, d, seed, mag)
    kb = key_bias(kind, B, Sk, seed)
    got = _run(q, k, v, kb, scale, g_tok, head_dim=d)
    n = H if heads is None else heads
    ref = reference(q[:, :n], k[:, :n], v[:, :n], kb, scale, g[:, :n])
    check_all(got, ref, f"B{B} H{H} Sq{Sq} Sk{Sk} d{d} {kind} scale {scale}", heads)
    return got


# --- dispatch branches: ragged and full key tiles, one query, a ragged query tile, long queries; B = 2, H = 3 takes
# the split dK/dV path at Sk <= 512 and Sq = 1000
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("Sq", [1, 127, 1000])
@pytest.mark.parametrize("Sk", [1, 64, 128, 129, 320, 383, 512, 513, 1023])
def test_dispatch_branches(Sk, Sq, d):
    run_case(2, 3, Sq, Sk, d, "cont", seed=Sk * 7 + Sq)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("Sk", [128, 383, 512])
def test_unsplit_dkv_path_many_heads(Sk, d):
    """B = 4, H = 40: at least one key-tile CTA per SM, so the dK/dV pass runs unsplit at Sk <= 512"""
    run_case(4, 40, 600, Sk, d, "cont", seed=Sk)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("scale", [0.125, None, 0.3, 1.0], ids=["0.125", "rsqrt_d", "0.3", "1.0"])
def test_softmax_scales(scale, d):
    run_case(2, 3, 700, 383, d, "cont", scale=d ** -0.5 if scale is None else scale, seed=3, mag=scale != 1.0)


KINDS = ["none", "ltx", "cont", "dominant", "left1", "left127", "left128", "left200", "left256", "dead"]


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B,H,Sq,Sk", [(2, 3, 1000, 383), (2, 40, 300, 320), (2, 3, 577, 700)],
                         ids=["split", "nosplit", "long"])
def test_key_biases(B, H, Sq, Sk, kind, d):
    """Every kind of key bias on the split and unsplit dK/dV paths and on long keys.  Masks hiding the first 128 or more
    keys leave a row's first key tile entirely -inf; 'dead' masks every key of one sample next to an unmasked one, whose
    out and gradients must be written as exact zeros (the outputs start NaN-filled)."""
    out, lse, dq, dk, dv = run_case(B, H, Sq, Sk, d, kind, seed=5)
    if kind == "dead":
        assert (out[0].view(torch.int16) == 0).all() and (dq[0].float() == 0).all()
        assert (dk[0].float() == 0).all() and (dv[0].float() == 0).all()


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("growth", [0.02, 0.2])
def test_running_max_growth_with_backward(growth, d):
    """Scores that keep growing along the keys take the online softmax through its rescale on every tile; the backward
    is checked too."""
    B, H, S = 2, 3, 1024
    torch.manual_seed(2)
    q = (torch.randn(B, H, S, d, device="cuda") * 0.3 + 1.0).bfloat16()
    ramp = torch.arange(S, device="cuda", dtype=torch.float32).view(1, 1, S, 1) * growth / d * 8
    k = (torch.randn(B, H, S, d, device="cuda") * 0.3 + ramp).bfloat16()
    v, g = torch.randn(B, H, S, d, device="cuda").bfloat16(), torch.randn(B, H, S, d, device="cuda").bfloat16()
    got = _run(q, k, v, None, 0.125, g.transpose(1, 2).reshape(B, S, H * d).contiguous(), head_dim=d)
    check_all(got, reference(q, k, v, None, 0.125, g), f"growth {growth} d{d}")


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("kind", ["none", "cont"])
def test_peaky_softmax(kind, d):
    """q and k scaled so that scale |q.k| is about 40: P is nearly one-hot and exp of the score error is large."""
    B, H, Sq, Sk = 2, 3, 500, 700
    torch.manual_seed(9)
    q, k = torch.randn(B, H, Sq, d, device="cuda"), torch.randn(B, H, Sk, d, device="cuda")
    c = math.sqrt(40 / (0.125 * math.sqrt(d)))
    q, k = (q * c).bfloat16(), (k * c).bfloat16()
    v, g = torch.randn(B, H, Sk, d, device="cuda").bfloat16(), torch.randn(B, H, Sq, d, device="cuda").bfloat16()
    kb = key_bias(kind, B, Sk, 9)
    got = _run(q, k, v, kb, 0.125, g.transpose(1, 2).reshape(B, Sq, H * d).contiguous(), head_dim=d)
    check_all(got, reference(q, k, v, kb, 0.125, g), f"peaky {kind} d{d}")


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("Sk", [100, 383, 1023])
def test_zero_query_gives_key_mean_and_zero_dk(Sk, d):
    """q = 0 and no bias: P is uniform, so out is the key-mean of V; dK = scale dS^T Q is exactly 0."""
    B, H, Sq = 2, 3, 300
    q, k, v, g, g_tok = inputs(B, H, Sq, Sk, d, 13)
    q = torch.zeros_like(q)
    got = _run(q, k, v, None, 0.125, g_tok, head_dim=d)
    ref = reference(q, k, v, None, 0.125, g)
    mean = v.double().mean(2, keepdim=True)
    assert ((ref["out"][0] - mean).abs() <= 1e-12 * v.double().abs().mean(2, keepdim=True)).all()
    check_all(got, ref, f"q=0 Sk{Sk} d{d}")
    assert ((got[3].view(torch.int16) & 0x7FFF) == 0).all(), "dK must be exactly zero when q = 0"


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("Sk,kind", [(2688, "none"), (128, "step")], ids=["self", "cross"])
def test_ltx_full_size(Sk, kind, d):
    """The LTX self-attention shape (1, 32, 2688, 2688) and the cross-attention shape Sk = 128 with the step's mask
    (77 kept keys, -10000 on the rest), all heads computed, three checked."""
    B, H, Sq = 1, 32, 2688
    q, k, v, g, g_tok = inputs(B, H, Sq, Sk, d, 17)
    kb = None
    if kind == "step":
        kb = (torch.arange(Sk, device="cuda")[None] >= 77).float() * -10000.0
    got = _run(q, k, v, kb, d ** -0.5, g_tok, head_dim=d)
    check_all(got, reference(q[:, :3], k[:, :3], v[:, :3], kb, d ** -0.5, g[:, :3]), f"LTX {kind} d{d}", heads=3)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("kind", ["left200", "dead"])
@pytest.mark.parametrize("B,H,Sq,Sk", [(2, 3, 1000, 320), (2, 40, 300, 383)], ids=["split", "nosplit"])
def test_masked_outputs_stay_inside_and_repeat_bitwise(B, H, Sq, Sk, kind, d):
    """Left padding and a fully masked sample: out, lse, dq, dk and dv inside NaN-patterned buffers, nothing outside
    them changes, and a second launch (its workspace NaN-filled) gives the same bits."""
    from finetrainers_b200 import ops
    pad = 4096
    q, k, v, g, g_tok = inputs(B, H, Sq, Sk, d, 21)
    kb = key_bias(kind, B, Sk, 21)
    runs = []
    for ws_fill in (0.0, float("nan")):
        bufs, views = {}, {}
        for name, shape, dt in (("out", (B, Sq, H * d), torch.bfloat16), ("lse", (B, H, Sq), torch.float32),
                                ("dq", (B, H, Sq, d), torch.bfloat16), ("dk", (B, H, Sk, d), torch.bfloat16),
                                ("dv", (B, H, Sk, d), torch.bfloat16)):
            n = math.prod(shape)
            bufs[name] = sentinel_buffer(n + 2 * pad, dt)
            views[name] = bufs[name][pad:pad + n].view(shape)
        ops.attn_fwd(q, k, v, kb, views["out"], views["lse"], B, H, Sq, Sk, 0.125, head_dim=d)
        ws = torch.full((ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=d),), ws_fill, device="cuda")
        ops.attn_bwd(q, k, v, kb, views["out"], g_tok, views["lse"], ws, views["dq"], views["dk"], views["dv"], B, H,
                     Sq, Sk, 0.125, head_dim=d)
        torch.cuda.synchronize()
        for name, buf in bufs.items():
            n = views[name].numel()
            check_sentinel(buf, [window(buf, pad, 1, n, n)], name)
        runs.append(views)
    for name in runs[0]:
        x, y = runs[0][name], runs[1][name]
        it = torch.int16 if x.dtype == torch.bfloat16 else torch.int32
        assert torch.equal(x.view(it), y.view(it)), name
    r = runs[0]
    check_all((r["out"], r["lse"], r["dq"], r["dk"], r["dv"]), reference(q, k, v, kb, 0.125, g), f"sentinel {kind} d{d}")


# --- the provider, through attention_dispatch with autograd, against torch's math SDPA in fp64 on the same values
def _math_sdpa64(q, k, v, mask, scale, g):
    qq, kk, vv = (t.double().requires_grad_(True) for t in (q, k, v))
    m = mask if mask is None or mask.dtype == torch.bool else mask.double()
    with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.MATH):
        o = F.scaled_dot_product_attention(qq, kk, vv, attn_mask=m, scale=scale)
    o.backward(g.double())
    return o.detach(), qq.grad, kk.grad, vv.grad


def _provider(q, k, v, mask, scale, g):
    from finetrainers_b200.attention import attention_dispatch
    qq, kk, vv = (t.clone().requires_grad_(True) for t in (q, k, v))
    o = attention_dispatch(qq, kk, vv, attn_mask=mask, scale=scale)
    o.backward(g)
    return o.detach(), qq.grad, kk.grad, vv.grad


def _mask(form, B, Sk):
    ar = torch.arange(Sk, device="cuda")
    keep = ar[None] >= torch.tensor([[0], [150]], device="cuda")[:B]        # sample 1 left-padded by 150 keys
    if form == "bool":
        return keep[:, None, None, :]
    if form == "bool_broadcast":
        return (ar >= 37)[None, None, None, :]
    if form == "left_pad":
        return (ar[None] >= torch.tensor([[128], [200]], device="cuda"))[:, None, None, :]
    if form == "dead":
        k2 = keep.clone()
        k2[0] = False
        return k2[:, None, None, :]
    gen = torch.Generator(device="cuda").manual_seed(4)
    cont = torch.rand(B, 1, 1, Sk, device="cuda", generator=gen) * 16 - 8
    if form in ("f32", "bf16"):
        return cont.to(torch.float32 if form == "f32" else torch.bfloat16)
    if form in ("finfo_f32", "finfo_bf16"):
        dt = torch.float32 if form == "finfo_f32" else torch.bfloat16
        return torch.zeros(B, 1, 1, Sk, device="cuda", dtype=dt).masked_fill(~keep[:, None, None, :], torch.finfo(dt).min)
    raise ValueError(form)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("form", ["bool", "bool_broadcast", "left_pad", "dead", "f32", "bf16", "finfo_f32",
                                  "finfo_bf16"])
def test_provider_masks(form, d):
    from finetrainers_b200.attention import mask_to_key_bias
    B, H, Sq, Sk = 2, 3, 300, 320
    q, k, v, g, _ = inputs(B, H, Sq, Sk, d, 31)
    mask = _mask(form, B, Sk)
    scale = d ** -0.5
    got = _provider(q, k, v, mask, scale, g)
    want = _math_sdpa64(q, k, v, mask, scale, g)
    kb = mask_to_key_bias(mask, B, Sk)
    ref = reference(q, k, v, kb, scale, g)
    for name, a, w in zip(("out", "dq", "dk", "dv"), got, want):
        assert torch.isfinite(a.float()).all(), name
        _check(name, a, w, ref[name][1], f"provider {form} d{d}")
    if form == "dead":
        for a in got:
            assert (a[0].float() == 0).all()


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("form", ["finfo_f32", "finfo_bf16", "minus_1e9"])
def test_provider_sample_masked_by_a_large_finite_value(form, d):
    """Sample 0 has every key at one large finite value, sample 1 its first 150 keys.  Scores reach a few hundred (natural
    log), so a backward that rebuilt P as an unnormalised exp of the score (what an lse that absorbed a huge bias
    gives) would overflow.  finfo.min masks like -inf: sample 0 gets out = 0 and zero gradients.  A common -1e9 is
    removed before the kernel: sample 0 attends as with no mask (bit for bit), which is what fp64 SDPA computes with
    that mask.  Everything else is held to its bound against fp64 SDPA."""
    from finetrainers_b200.attention import mask_to_key_bias
    B, H, Sq, Sk = 2, 3, 200, 300
    torch.manual_seed(37)
    q, k = ((torch.randn(B, H, S, d, device="cuda") * 12).bfloat16() for S in (Sq, Sk))
    v, g = torch.randn(B, H, Sk, d, device="cuda").bfloat16(), torch.randn(B, H, Sq, d, device="cuda").bfloat16()
    dt = {"finfo_f32": torch.float32, "finfo_bf16": torch.bfloat16, "minus_1e9": torch.float32}[form]
    val = -1e9 if form == "minus_1e9" else torch.finfo(dt).min
    mask = torch.zeros(B, 1, 1, Sk, device="cuda", dtype=dt)
    mask[0] = val
    mask[1, ..., :150] = val
    scale = d ** -0.5
    got = _provider(q, k, v, mask, scale, g)
    for a in got:
        assert torch.isfinite(a.float()).all()
    if form == "minus_1e9":
        free = mask.clone()
        free[0] = 0
        for a, b in zip(got, _provider(q, k, v, free, scale, g)):
            assert torch.equal(a[0].view(torch.int16), b[0].view(torch.int16))
        rows = slice(0, B)
    else:
        for a in got:
            assert (a[0].view(torch.int16) & 0x7FFF == 0).all()
        rows = slice(1, B)
    want = _math_sdpa64(q, k, v, mask, scale, g)
    ref = reference(q, k, v, mask_to_key_bias(mask, B, Sk), scale, g)
    for name, a, w in zip(("out", "dq", "dk", "dv"), got, want):
        _check(name, a[rows], w[rows], ref[name][1][rows], f"provider {form} d{d}")


@pytest.mark.parametrize("d", [64, 128])
def test_provider_per_head_masks(d):
    """A mask that differs between heads is refused; one repeated over the heads gives the bits of its [B,1,1,Sk] form."""
    from finetrainers_b200.attention import attention_dispatch
    B, H, Sq, Sk = 2, 3, 130, 200
    q, k, v, g, _ = inputs(B, H, Sq, Sk, d, 35)
    keep = torch.arange(Sk, device="cuda")[None, None, None, :] < torch.tensor([150, 200], device="cuda").view(B, 1, 1, 1)
    per_head = keep.expand(B, H, 1, Sk).clone()
    per_head[1, 2, 0, :10] = False
    with pytest.raises(ValueError, match="every head"):
        attention_dispatch(q, k, v, attn_mask=per_head)
    a = _provider(q, k, v, keep, None, g)
    b = _provider(q, k, v, keep.expand(B, H, 1, Sk).contiguous(), None, g)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16))
