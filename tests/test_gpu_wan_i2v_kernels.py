"""Wan-2.1 image-to-video kernels: the I2V step prologue (b2d_wan_i2v_prep), the exact GELU of the image embedder
(b2d_gelu_erf) and the K = 144 patch-embedding GEMM of the 36-channel input.

  wan_i2v_prep: bit-exact against tests/golden/wan_i2v_golden.pt (the reference's own prologue code, run on the
                CPU); at larger shapes bit-exact against the reference's arithmetic restated on the GPU
                (oracle.wan_oracle.prologue for x_t and target, oracle.wan_oracle.normalize_latents for the condition
                mean, the mask copied), patchified as cat([x_t, mask, condition], dim=1) through a Conv3d weight viewed
                as [D, 144]; x_t and target also bit for bit against b2d_wan_prep on the same inputs.  Outputs inside
                sentinel buffers.
  gelu_erf:     against torch's F.gelu(approximate="none") on the same bf16 tensor on the GPU: bit-exact expected; any
                differing element is reported and must be within one bf16 ulp.
  K = 144 GEMM: within ulp16(ref) + 2^-16 |A| |W|^T of the fp64 product (the GEMM suite's accumulation bound)."""
import pytest
import torch
import torch.nn.functional as F

from _util import absmm64, bf16_ulp, check_bound, check_sentinel, mm64, sentinel_buffer, window

pytestmark = pytest.mark.gpu

PAD = 64


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


def _bits(t):
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _guarded(n, shift=0):
    buf = sentinel_buffer(n + 2 * PAD + shift, torch.bfloat16)
    return buf, buf[PAD + shift:PAD + shift + n]


def _patchify_conv(x):
    """[B, C, F, H, W] -> [B, F (H/2) (W/2), 4C] with k = c*4 + kh*2 + kw (Conv3d weight [D, C, 1, 2, 2] as [D, 4C])."""
    B, C, Fr, H, W = x.shape
    t = x.reshape(B, C, Fr, H // 2, 2, W // 2, 2).permute(0, 2, 3, 5, 1, 4, 6)
    return t.reshape(B, Fr * (H // 2) * (W // 2), 4 * C)


def _mask(B, Fr, H, W):
    """WanImageConditioningLatentEncodeProcessor's mask [B, 4, F, H, W]: the first latent frame 1, the others 0."""
    m = torch.zeros(B, 4, Fr, H, W, dtype=torch.bfloat16, device="cuda")
    m[:, :, 0] = 1
    return m


@pytest.mark.parametrize("B,C,F,H,W", [(1, 16, 2, 4, 6), (2, 16, 3, 6, 10), (1, 16, 13, 60, 104), (2, 5, 2, 2, 2)])
def test_wan_i2v_prep(ops, B, C, F, H, W):
    from oracle import wan_oracle as O
    g = torch.Generator().manual_seed(B * 100 + C + F)
    Cm = 4
    mom = torch.cat([torch.randn(B, C, F, H, W, generator=g), torch.rand(B, C, F, H, W, generator=g) * 10 - 5], 1)
    cond = torch.cat([torch.randn(B, C, F, H, W, generator=g) * 2, torch.full((B, C, F, H, W), float("nan"))], 1)
    mean = torch.randn(B, C, generator=g) * 0.3
    std = 1.0 / (torch.rand(B, C, generator=g) + 0.5)
    eps, noise = torch.randn(B, C, F, H, W, generator=g), torch.randn(B, C, F, H, W, generator=g)
    sig = torch.rand(B, generator=g)
    mom, cond, eps, noise = (t.bfloat16().cuda() for t in (mom, cond, eps, noise))
    mean, std, sig = mean.cuda(), std.cuda(), sig.cuda()
    mask = _mask(B, F, H, W)
    S = F * (H // 2) * (W // 2)
    n_in, n_t = B * S * 4 * (2 * C + Cm), B * S * 4 * C
    xb, x_in = _guarded(n_in, shift=1)
    tb, tg = _guarded(n_t, shift=3)
    ops.wan_i2v_prep(mom, cond, mask, eps, noise, mean, std, sig, x_in, tg, B, C, Cm, F, H, W)
    torch.cuda.synchronize()
    check_sentinel(xb, [window(xb, PAD + 1, 1, n_in, n_in)], "x_in")
    check_sentinel(tb, [window(tb, PAD + 3, 1, n_t, n_t)], "target")
    # the reference's arithmetic: x_t and target per sample, the condition as the normalised mean (its logvar, NaN here,
    # must not be read), then cat([x_t, mask, condition], dim=1) patchified in the Conv3d order
    xt_ref, tg_ref, c_ref = [], [], []
    for b in range(B):
        x_t, target = O.prologue(mom[b:b + 1], mean[b], std[b], eps[b:b + 1], noise[b:b + 1], sig[b:b + 1])
        xt_ref.append(x_t)
        tg_ref.append(target)
        c_ref.append(O.normalize_latents(cond[b:b + 1, :C], mean[b], std[b]))
    x5 = torch.cat([torch.cat(xt_ref), mask, torch.cat(c_ref)], 1)
    ref = _patchify_conv(x5).reshape(-1)
    assert torch.equal(_bits(x_in), _bits(ref)), f"x_in: {(_bits(x_in) != _bits(ref)).sum().item()} elements differ"
    t_ref = torch.cat(tg_ref).reshape(B, C, F, H // 2, 2, W // 2, 2).permute(0, 2, 3, 5, 4, 6, 1).reshape(-1)
    assert torch.equal(_bits(tg), _bits(t_ref)), "target"
    # against the text-to-video prologue on the same inputs
    xt2, tg2 = torch.empty(B, S, 4 * C, dtype=torch.bfloat16, device="cuda"), torch.empty(n_t, dtype=torch.bfloat16,
                                                                                          device="cuda")
    ops.wan_prep(mom, eps, noise, mean, std, sig, xt2, tg2, B, C, F, H, W)
    xin = x_in.view(B, S, 2 * C + Cm, 4)
    assert torch.equal(_bits(xin[:, :, :C].reshape(B, S, 4 * C)), _bits(xt2)), "x_t vs wan_prep"
    assert torch.equal(_bits(tg), _bits(tg2)), "target vs wan_prep"
    assert torch.equal(xin[:, :, C:C + Cm], _patchify_conv(mask).view(B, S, Cm, 4)), "mask channels"


def test_wan_i2v_prep_golden(ops):
    """Against the reference's own prologue (tests/golden/make_wan_i2v_golden.py runs its
    WanImageConditioningLatentEncodeProcessor and WanModelSpecification.forward on the CPU): its mask and condition
    channels of the 36-channel cat([x_t, mask, condition]) bit for bit; its x_t and target bit for bit wherever the CPU's
    and CUDA's exp round exp(0.5 clamp(logvar)) to the same bf16 value (as test_gpu_posterior.py's golden check), and,
    everywhere, bit for bit against the same reference arithmetic run on the GPU."""
    import os
    from oracle import wan_oracle as O
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "wan_i2v_golden.pt"), weights_only=False)
    B, C, F, H, W = g["noise"].shape
    Cm = g["mask"].shape[1]
    assert not g["mask"].is_contiguous()  # the reference builds it as a transposed view
    dev = {k: v.cuda().contiguous() for k, v in g.items()}
    mean = dev["latents_mean"].expand(B, C).contiguous()
    std = dev["latents_std"].expand(B, C).contiguous()
    S = F * (H // 2) * (W // 2)
    x_in = torch.empty(B, S, 4 * (2 * C + Cm), dtype=torch.bfloat16, device="cuda")
    tg = torch.empty(B, S, 4 * C, dtype=torch.bfloat16, device="cuda")
    ops.wan_i2v_prep(dev["moments"], dev["cond_moments"], dev["mask"], dev["eps"], dev["noise"], mean, std,
                     dev["sigmas"], x_in, tg, B, C, Cm, F, H, W)
    torch.cuda.synchronize()
    got5 = x_in.view(B, F, H // 2, W // 2, 2 * C + Cm, 2, 2).permute(0, 4, 1, 2, 5, 3, 6).reshape(B, 2 * C + Cm, F, H, W)
    got_t = tg.view(B, F, H // 2, W // 2, 2, 2, C).permute(0, 6, 1, 2, 4, 3, 5).reshape(B, C, F, H, W)
    want = dev["hidden_states"]
    assert torch.equal(_bits(got5[:, C:]), _bits(want[:, C:])), "mask and condition channels"
    lv = O.normalize_latents(g["moments"][:, C:], g["latents_mean"], g["latents_std"]).clamp(-30.0, 20.0)
    apart = (_bits(torch.exp(0.5 * lv)) != _bits(torch.exp(0.5 * lv.cuda()).cpu())).cuda()
    for got, ref, what in ((got5[:, :C], want[:, :C], "x_t"), (got_t, dev["target"], "target")):
        differ = _bits(got) != _bits(ref)
        assert not (differ & ~apart).any(), f"{what}: differs from the golden where CPU and CUDA exp agree"
        print(f"wan_i2v_prep golden {what}: {int(differ.sum())} of {ref.numel()} apart, exp apart at {int(apart.sum())}")
    x_t, target = O.prologue(dev["moments"], dev["latents_mean"], dev["latents_std"], dev["eps"], dev["noise"],
                             dev["sigmas"])
    assert torch.equal(_bits(got5[:, :C]), _bits(x_t)) and torch.equal(_bits(got_t), _bits(target)), "vs GPU oracle"


def test_wan_i2v_prep_refusals(ops):
    from finetrainers_b200.lib import B2DError
    t = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    f = torch.zeros(4, device="cuda")
    for kw, code in ((dict(Cm=17), -1), (dict(Cm=0), -1), (dict(H=3), -1), (dict(F=0), -1)):
        a = dict(B=1, C=16, Cm=4, F=1, H=2, W=2)
        a.update(kw)
        with pytest.raises(B2DError, match=rf"\(code {code}\)"):
            ops.wan_i2v_prep(t, t, t, t, t, f, f, f, t, t, *a.values())
    with pytest.raises(B2DError, match=r"\(code -5\)"):
        ops.wan_i2v_prep(t, None, t, t, t, f, f, f, t, t, 1, 16, 4, 1, 2, 2)


@pytest.mark.parametrize("n", [1, 257 * 1280, 1000003])
def test_gelu_erf(ops, n):
    g = torch.Generator(device="cuda").manual_seed(n)
    x = (torch.randn(n, device="cuda", generator=g) * 3).bfloat16()
    if n > 16:
        x[:8] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 10.0, -10.0, float("inf"), -float("inf")]).bfloat16()
    yb, y = _guarded(n, shift=1)
    ops.gelu_erf(x, y, n)
    torch.cuda.synchronize()
    check_sentinel(yb, [window(yb, PAD + 1, 1, n, n)], "gelu_erf")
    ref = F.gelu(x, approximate="none")
    diff = _bits(y) != _bits(ref)
    nd = int(diff.sum().item())
    print(f"gelu_erf n={n}: {nd} elements differ from F.gelu(approximate='none')")
    if nd:
        assert ((y[diff].double() - ref[diff].double()).abs() <= bf16_ulp(ref[diff].double())).all(), "more than 1 ulp"
    # in place
    z = x.clone()
    ops.gelu_erf(z, z, n)
    assert torch.equal(_bits(z), _bits(y))


@pytest.mark.parametrize("M,D", [(300, 1536), (8, 5120), (2 * 13 * 30 * 52, 5120)])
def test_patch_gemm_k144(ops, M, D):
    """The 36-channel patch embedding: x_in [M, 144] times patch_embedding.weight [D, 36, 1, 2, 2] viewed as [D, 144]."""
    g = torch.Generator(device="cuda").manual_seed(M)
    A = torch.randn(M, 144, device="cuda", generator=g).bfloat16()
    Wt = (torch.randn(D, 36, 1, 2, 2, device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn(D, device="cuda", generator=g).bfloat16()
    W2 = Wt.view(D, 144)
    out = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
    ops.gemm(A, W2, out, M=M, N=D, K=144, bias=bias)
    ref = mm64(A, W2) + bias.double()
    bound = bf16_ulp(ref) + 2.0 ** -16 * (absmm64(A, W2) + bias.double().abs())
    check_bound(out, ref, bound, f"patch GEMM M{M} D{D}")
