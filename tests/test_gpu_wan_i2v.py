"""GPU: Wan-2.1 image-to-video (I2V) LoRA training on the engine.

- The 14B width (40 heads x 128 = 5120, FFN 13824), 2 blocks, r = 32, image_dim 1280, against the fp32 oracle
  (tests/_wan_i2v_oracle.py): F = 2 latent frames of 30 x 52 (780 latent tokens, a ragged last query tile; the mask is
  1 on the first frame and 0 on the second), 512 text + 257 image keys.  Loss within 1e-3 relative, every LoRA
  gradient within 5 % of its own scale (attn2.to_q, whose dQ comes from both contexts, reported by name), the
  concatenated gradient at cosine > 0.999 and norm ratio within 1 %: the T2V-14B bars.
- attention_head_dim 64 against the oracle, and on that model: the public forward's autograd gradients equal to the
  fused step's and the no-grad inference prediction equal to the training forward's, bit for bit; CUDA-graph steps,
  "full" and "block_skip" checkpointing bit-identical to eager keep-all; graph-replayed gradient accumulation
  bit-identical to eager accumulation; two seeded 20-step runs bit-identical; the kept cross-attention output and both
  log-sum-exps left as they were by the backward (it re-runs the two-context forward for the branch outputs).
- The image embedder's exact GELU element by element against float64 (a tanh GELU would miss the bound).
- The specification's call surface with the real prologue kernel against what the reference's own forward passed
  (tests/golden/wan_i2v_call_golden.pt).
"""
import math
import os

import pytest
import torch

import _wan_i2v_oracle as I
from oracle import wan_oracle as O

pytestmark = pytest.mark.gpu

SMALL64 = dict(num_attention_heads=4, attention_head_dim=64, ffn_dim=512)


@pytest.fixture(scope="module", autouse=True)
def _device():
    from finetrainers_b200 import lib
    lib.check(lib.load().b2d_device_check(), "device")


def _same(a, b, what):
    a, b = a.reshape(-1).cpu(), b.reshape(-1).cpu()
    diff = int((a.view(torch.int16) != b.view(torch.int16)).sum())
    assert diff == 0, f"{what}: {diff} element(s) differ"


def _pair(nl, r=32, seed=0, image_dim=128, **geom):
    from finetrainers_b200.wan import B200WanTransformer, WanConfig
    om = I.WanI2VTransformerOracle(I.WanI2VOracleConfig(image_dim=image_dim, num_layers=nl, **geom))
    O.add_lora(om, r, r)
    O.synthetic_init_(om, seed=seed)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    d = geom["num_attention_heads"] * geom["attention_head_dim"]
    bm = B200WanTransformer(WanConfig(num_layers=nl, in_channels=36, image_dim=image_dim, added_kv_proj_dim=d, **geom),
                            torch.bfloat16, "cuda")
    bm.add_adapter(r, r)
    bm.load_state_dict(om.state_dict(), strict=True)
    bm.prepare()
    bm.skip_block0_dx = False
    return om, bm


def _batch(B=1, F=2, H=8, W=12, L=512, Li=257, image_dim=128, seed=1):
    g = torch.Generator().manual_seed(seed)
    mom = torch.cat([torch.randn(B, 16, F, H, W, generator=g), torch.rand(B, 16, F, H, W, generator=g) * 4 - 8], 1)
    cond = torch.cat([torch.randn(B, 16, F, H, W, generator=g), torch.rand(B, 16, F, H, W, generator=g) * 4 - 8], 1)
    mask = torch.zeros(B, F, 4, H, W).transpose(1, 2)  # the reference's mask is a transposed view
    mask[:, :, 0] = 1
    return dict(moments=mom.to(torch.bfloat16), cond=cond.to(torch.bfloat16), mask=mask.to(torch.bfloat16),
                mean=torch.randn(16, generator=g) * 0.2, std=1.0 / (torch.rand(16, generator=g) + 0.5),
                eps=torch.randn(B, 16, F, H, W, generator=g).to(torch.bfloat16),
                noise=torch.randn(B, 16, F, H, W, generator=g).to(torch.bfloat16),
                sigmas=torch.rand(B, generator=g) * 0.9 + 0.05,
                ehs=torch.randn(B, L, 4096, generator=g).to(torch.bfloat16),
                img=torch.randn(B, Li, image_dim, generator=g).to(torch.bfloat16))


def _lat(bt):
    B = bt["moments"].shape[0]
    return {"latents": bt["moments"].cuda(), "latents_mean": bt["mean"].expand(B, 16).cuda(),
            "latents_std": bt["std"].expand(B, 16).cuda(), "latent_condition": bt["cond"].cuda(),
            "latent_condition_mask": bt["mask"].cuda(), "encoder_hidden_states_image": bt["img"].cuda()}


def _micro(st, bt):
    return st.micro_step({"encoder_hidden_states": bt["ehs"].cuda()}, _lat(bt), sigmas=bt["sigmas"].cuda(),
                         noise=bt["noise"].cuda(), posterior_noise=bt["eps"].cuda())


def _oracle(om, bt):
    return I.oracle_step(om, bt["moments"], bt["cond"], bt["mask"], bt["mean"], bt["std"], bt["eps"], bt["noise"],
                         bt["sigmas"], bt["ehs"], bt["img"])


def _compare(om, bm, bt, what):
    """-> (loss rel err, {name: grad err}, cosine, norm ratio) of one fused step against the oracle's."""
    from finetrainers_b200.trainer import SFTTrainStep
    loss_o, _ = _oracle(om, bt)
    st = SFTTrainStep(bm, flow_weighting_scheme="none")
    loss_b = _micro(st, bt).item()
    rel = abs(loss_b - loss_o.item()) / abs(loss_o.item())
    og, bg = dict(om.named_parameters()), dict(bm.named_parameters())
    names = [n for n in bg if "lora_" in n]
    errs = {n: (bg[n].grad.float().cpu() - og[n].grad).abs().max().item() / og[n].grad.abs().max().item() for n in names}
    gb = torch.cat([bg[n].grad.double().cpu().flatten() for n in names])
    go = torch.cat([og[n].grad.double().flatten() for n in names])
    cos, ratio = (torch.dot(gb, go) / (gb.norm() * go.norm())).item(), (gb.norm() / go.norm()).item()
    worst = max(errs.items(), key=lambda t: t[1])
    q2 = max(v for n, v in errs.items() if ".attn2.to_q." in n)
    print(f"\n{what}: loss rel err {rel:.2e}, worst LoRA grad err {worst[1]:.3e} ({worst[0]}), attn2.to_q worst "
          f"{q2:.3e}, gradient cosine {cos:.6f}, norm ratio {ratio:.5f}")
    assert math.isfinite(loss_b) and rel < 1e-3, (loss_b, loss_o.item())
    assert len(errs) == 2 * 16
    for n, v in errs.items():
        assert v < 5e-2, (n, v)
    assert cos > 0.999 and abs(ratio - 1) < 1e-2, (cos, ratio)


@pytest.mark.timeout(1200)
def test_wan_i2v_14b_width_two_blocks_vs_oracle():
    from finetrainers_b200.wan import WanConfig
    c = WanConfig.wan_i2v_14b()
    om, bm = _pair(2, r=32, image_dim=c.image_dim, num_attention_heads=c.num_attention_heads,
                   attention_head_dim=c.attention_head_dim, ffn_dim=c.ffn_dim)
    _compare(om, bm, _batch(F=2, H=30, W=52, image_dim=c.image_dim), "Wan I2V 14B width, 2 blocks, 780 tokens")


def test_wan_i2v_head_dim_64_vs_oracle():
    om, bm = _pair(2, r=32, image_dim=128, **SMALL64)
    _compare(om, bm, _batch(), "Wan I2V head_dim 64, 2 blocks, 48 tokens")


def _run(steps, graph=False, ckpt=None, accum=1, seed=0):
    """Loss of every micro-step and the final fp32 adapter masters of ``steps`` train_step calls on one batch."""
    from finetrainers_b200.model import apply_activation_checkpointing
    from finetrainers_b200.trainer import SFTTrainStep
    torch.manual_seed(seed)
    _, bm = _pair(2, r=16, seed=seed, **SMALL64)
    if ckpt:
        apply_activation_checkpointing(bm, *((ckpt,) if isinstance(ckpt, str) else ckpt))
    st = SFTTrainStep(bm, flow_weighting_scheme="logit_normal", use_cuda_graph=graph, seed=seed, lr=1e-4,
                      gradient_accumulation_steps=accum)
    bt = _batch(seed=seed + 1)
    losses = []
    for _ in range(steps):
        st.train_step({"encoder_hidden_states": bt["ehs"].cuda()}, _lat(bt))
        losses.append(float(st.loss_buf))
    torch.cuda.synchronize()
    assert st.opt_step == steps // accum
    return losses, bm.lora_flat.detach().clone()


def test_wan_i2v_graph_checkpointing_and_accumulation_bit_identical():
    base_l, base_p = _run(4)
    assert all(math.isfinite(x) for x in base_l)
    for kw in (dict(graph=True), dict(ckpt="full"), dict(ckpt=("block_skip", 2)), dict(graph=True, ckpt="full")):
        l, p = _run(4, **kw)
        assert l == base_l, (kw, l, base_l)
        assert torch.equal(p, base_p), kw
    acc_l, acc_p = _run(6, accum=2)
    assert not torch.equal(acc_p, base_p)
    l, p = _run(6, accum=2, graph=True)
    assert l == acc_l and torch.equal(p, acc_p)


def test_wan_i2v_seeded_runs_20_steps_bit_identical():
    a_l, a_p = _run(20, graph=True)
    b_l, b_p = _run(20, graph=True)
    assert all(math.isfinite(x) for x in a_l)
    assert a_l == b_l and torch.equal(a_p, b_p)


def test_wan_i2v_public_forward_matches_step_and_backward_keeps_attention_rows():
    """spec.forward through the public forward: the fused step's target and loss, its autograd backward the fused
    step's adapter gradients bit for bit, the no-grad inference plan the same prediction; the backward leaves the kept
    ao2 / lse2 / lse3 bytes as the forward wrote them."""
    from finetrainers_b200.trainer import SFTTrainStep
    from finetrainers_b200.wan import WanModelSpecification
    bt = _batch(seed=5)
    _, fused = _pair(2, r=16, **SMALL64)
    loss_f = _micro(SFTTrainStep(fused, flow_weighting_scheme="none"), bt).item()
    _, bm = _pair(2, r=16, **SMALL64)
    lat = _lat(bt)
    pred, target, _ = WanModelSpecification(bm.cfg).forward(bm, {"encoder_hidden_states": bt["ehs"].cuda()}, lat,
                                                            bt["sigmas"].cuda(), noise=bt["noise"].cuda(),
                                                            posterior_noise=bt["eps"].cuda())
    assert set(lat) == {"hidden_states", "encoder_hidden_states_image"}
    assert pred.shape == target.shape == (1, 16, 2, 8, 12) and lat["hidden_states"].shape == (1, 36, 2, 8, 12)
    hidden, tg = I.i2v_prologue(bt["moments"].cuda(), bt["cond"].cuda(), bt["mask"].cuda(), bt["mean"].cuda(),
                                bt["std"].cuda(), bt["eps"].cuda(), bt["noise"].cuda(), bt["sigmas"].cuda())
    _same(target, tg, "target")
    _same(lat["hidden_states"], hidden, "36-channel input")
    (ws,) = bm._ws.values()
    kept = {k: ws[k].clone() for k in ("ao2", "lse2", "lse3")}
    assert torch.isfinite(kept["lse3"]).all() and (kept["lse3"] != kept["lse2"]).any()
    loss = (pred.float() - target.float()).pow(2).mean()
    loss.backward()
    for k, v in kept.items():
        assert torch.equal(ws[k].view(torch.int32 if v.dtype == torch.float32 else torch.int16),
                           v.view(torch.int32 if v.dtype == torch.float32 else torch.int16)), k
    assert abs(loss.item() - loss_f) / loss_f < 1e-5, (loss.item(), loss_f)
    gf = dict(fused.named_parameters())
    for n, p in bm.named_parameters():
        if "lora_" in n:
            assert torch.equal(p.grad, gf[n].grad), n
    with torch.no_grad():
        pred2 = bm(hidden, (bt["sigmas"].cuda() * 1000.0).long(), bt["ehs"].cuda(),
                   encoder_hidden_states_image=bt["img"].cuda())[0]
    _same(pred2, pred.detach(), "no-grad inference plan vs training plan")


def test_wan_i2v_spec_call_surface_against_the_reference():
    """The specification with the real prologue kernel hands the transformer what the reference's own forward did: the
    same keyword arguments, shapes and dtypes, timestep, and 36-channel hidden_states (the mask and condition channels
    bit for bit; x_t and the target bit for bit against the reference's torch ops run on this GPU)."""
    from finetrainers_b200.wan import WanConfig, WanModelSpecification
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "wan_i2v_call_golden.pt"), weights_only=False)
    calls = []

    class Stub:
        cfg = WanConfig(in_channels=36, image_dim=16, added_kv_proj_dim=1536, text_dim=8)

        def __call__(self, **kw):
            calls.append(kw)
            return (torch.zeros(2, 16, 2, 4, 6, device="cuda"),)

    cu = {k: v.cuda() for k, v in g.items() if isinstance(v, torch.Tensor)}
    lat = {"latents": cu["moments"], "latents_mean": cu["latents_mean"], "latents_std": cu["latents_std"],
           "latent_condition": cu["cond_moments"], "latent_condition_mask": cu["mask"],
           "encoder_hidden_states_image": cu["encoder_hidden_states_image"]}
    _, target, _ = WanModelSpecification(Stub.cfg).forward(Stub(), {"encoder_hidden_states": cu["encoder_hidden_states"]},
                                                           lat, cu["sigmas"], noise=cu["noise"],
                                                           posterior_noise=cu["eps"])
    (kw,) = calls
    assert {k: (tuple(v.shape), str(v.dtype)) if isinstance(v, torch.Tensor) else v for k, v in kw.items()} == g["args"]
    assert sorted(lat) == g["left"] and torch.equal(kw["timestep"].cpu(), g["timestep"])
    _same(kw["hidden_states"][:, 16:], g["hidden_states"][:, 16:], "mask and condition channels")
    hidden, tg = I.i2v_prologue(cu["moments"], cu["cond_moments"], cu["mask"], cu["latents_mean"], cu["latents_std"],
                                cu["eps"], cu["noise"], cu["sigmas"])
    _same(kw["hidden_states"], hidden, "36-channel input")
    _same(target, tg, "target")


def _ulp(x):
    return 2.0 ** (torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 7)


def test_wan_i2v_image_embedder_gelu_is_exact():
    """The image embedder's activation (diffusers FeedForward with activation_fn="gelu": exact erf GELU) on the rounded
    Linear output, against float64 from the engine's own bf16 input of that Linear: |gelu - GELU64(pre)| within half a
    bf16 ulp of the output plus what half an ulp of the rounded pre-activation moves it (2 % slack and the fp32
    accumulation).  On the same data the tanh approximation misses that bound."""
    import torch.nn.functional as Fn
    _, bm = _pair(1, r=16, **SMALL64)
    bt = _batch(seed=9)
    with torch.no_grad():
        bm(torch.zeros(1, 36, 2, 8, 12, device="cuda"), torch.full((1,), 500, device="cuda"), bt["ehs"].cuda(),
           encoder_hidden_states_image=bt["img"].cuda())
    ws = bm._iws[1]
    rv = bm._root_views
    a, w, b = ws["imn"].double(), rv["img_ff1.w"].double(), rv["img_ff1.b"].double()
    pre = a @ w.T + b
    g64 = Fn.gelu(pre)
    dg = 0.5 * (1 + torch.erf(pre / math.sqrt(2))) + pre * torch.exp(-pre ** 2 / 2) / math.sqrt(2 * math.pi)
    acc = (a.abs() @ w.abs().T + b.abs()) * 2.0 ** -20
    bound = 1.02 * (dg.abs() * 0.5 * _ulp(pre) + 0.5 * _ulp(g64)) + dg.abs() * acc
    got = ws["imf"].double()
    ratio = ((got - g64).abs() / bound).max().item()
    tanh = Fn.gelu(pre.to(torch.bfloat16).float(), approximate="tanh").to(torch.bfloat16).double()
    miss = int(((tanh - g64).abs() > bound).sum())
    print(f"\nimage embedder GELU: worst error / bound {ratio:.3f}; a tanh GELU misses the bound at {miss} of "
          f"{got.numel()} elements")
    assert ratio <= 1.0 and miss > 0
