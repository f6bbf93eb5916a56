"""Host: the Wan-2.1 image-to-video model — module tree and FQNs, adapter targets, refusals, workspace plan (and the
text-to-video plan left as it was), the oracle's prologue against the reference's fixtures, and the specification's call
surface against what the reference's own ``WanModelSpecification.forward`` hands the transformer."""
import os

import pytest
import torch

import _wan_i2v_oracle as I
from finetrainers_b200.wan import B200WanTransformer, WanConfig, WanModelSpecification

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


class _Lora:
    def __init__(self, r=32, lora_alpha=32, target_modules="blocks.*(to_q|to_k|to_v|to_out.0)"):
        self.r, self.lora_alpha, self.target_modules, self.init_lora_weights = r, lora_alpha, target_modules, True


def _cfg(nl=2, **kw):
    return WanConfig(**dict(dict(num_attention_heads=2, attention_head_dim=128, ffn_dim=512, text_dim=64, num_layers=nl,
                                 in_channels=36, image_dim=64, added_kv_proj_dim=256), **kw))


# diffusers WanTransformer3DModel with image_dim / added_kv_proj_dim: what it adds to the T2V tree (WanImageEmbedding,
# the added K/V projections of every block's attn2 and their across-heads k-norm), restated
I2V_FQNS = ["condition_embedder.image_embedder.norm1.weight", "condition_embedder.image_embedder.norm1.bias",
            "condition_embedder.image_embedder.ff.net.0.proj.weight", "condition_embedder.image_embedder.ff.net.0.proj.bias",
            "condition_embedder.image_embedder.ff.net.2.weight", "condition_embedder.image_embedder.ff.net.2.bias",
            "condition_embedder.image_embedder.norm2.weight", "condition_embedder.image_embedder.norm2.bias"] + [
    f"blocks.{i}.attn2.{n}" for i in range(2) for n in ("add_k_proj.weight", "add_k_proj.bias", "add_v_proj.weight",
                                                         "add_v_proj.bias", "norm_added_k.weight")]


def test_i2v_14b_config():
    c = WanConfig.wan_i2v_14b()
    assert (c.inner_dim, c.ffn_dim, c.num_layers, c.in_channels, c.out_channels) == (5120, 13824, 40, 36, 16)
    assert (c.image_dim, c.added_kv_proj_dim, c.pos_embed_seq_len) == (1280, 5120, None)
    m = B200WanTransformer(WanConfig.wan_i2v_14b(), device="meta")
    assert m.desc.image_dim == 1280 and m.desc.in_features == 144 and m.desc.out_features == 64


def test_fqns_and_shapes_match_restated_diffusers_tree():
    bm = B200WanTransformer(_cfg(), device="cpu")
    t2v = B200WanTransformer(_cfg(in_channels=16, image_dim=None, added_kv_proj_dim=None), device="cpu")
    got = {k: tuple(v.shape) for k, v in bm.state_dict().items()}
    assert sorted(set(got) - set(t2v.state_dict())) == sorted(I2V_FQNS)
    assert got["patch_embedding.weight"] == (256, 36, 1, 2, 2) and got["proj_out.weight"] == (64, 256)
    assert got["condition_embedder.image_embedder.norm1.weight"] == (64,)
    assert got["condition_embedder.image_embedder.ff.net.0.proj.weight"] == (64, 64)
    assert got["condition_embedder.image_embedder.ff.net.2.weight"] == (256, 64)
    assert got["blocks.1.attn2.add_k_proj.weight"] == (256, 256) and got["blocks.1.attn2.norm_added_k.weight"] == (256,)
    om = I.WanI2VTransformerOracle(I.WanI2VOracleConfig(image_dim=64, num_attention_heads=2, attention_head_dim=128,
                                                        ffn_dim=512, text_dim=64, num_layers=2))
    assert got == {k: tuple(v.shape) for k, v in om.state_dict().items()}
    I.O.add_lora(om, 8, 8)
    I.O.synthetic_init_(om)
    bm.add_adapter(8, 8)
    bm.load_state_dict(om.state_dict(), strict=True)
    bm.prepare()
    # the image side sits in the root unit, every block's [Wk3; Wv3] stacked as the text side's [Wk2; Wv2]
    rv, d = bm._root_views, 256
    for i, blk in enumerate(bm.blocks):
        assert blk.attn2.add_k_proj.weight.data_ptr() == rv["Wkv3_all"][i, :d].data_ptr()
        assert blk.attn2.add_v_proj.weight.data_ptr() == rv["Wkv3_all"][i, d:].data_ptr()
        assert blk.attn2.add_v_proj.bias.data_ptr() == rv["bkv3_all"][i, d:].data_ptr()
        assert blk.attn2.norm_added_k.weight.data_ptr() == rv["nk3_all"][i].data_ptr()
        assert torch.equal(blk.attn2.add_k_proj.weight.float(), om.blocks[i].attn2.add_k_proj.weight.bfloat16().float())
    ie = bm.condition_embedder.image_embedder
    assert ie.ff.net[2].weight.data_ptr() == rv["img_ff2.w"].data_ptr()
    assert ie.norm2.bias.data_ptr() == rv["img_n2.b"].data_ptr()


@pytest.mark.parametrize("tm", ["blocks.*(to_q|to_k|to_v|to_out.0)", ["to_q", "to_k", "to_v", "to_out.0"]])
def test_lora_targets_resolve_without_the_image_projections(tm):
    bm = B200WanTransformer(_cfg(), device="cpu")
    bm.add_adapter(_Lora(target_modules=tm))
    names = [n for n, _ in bm.named_parameters() if "lora_A" in n]
    assert len(names) == 2 * 8
    assert not any("add_" in n or "image_embedder" in n for n in names)
    assert all(p.requires_grad == ("lora_" in n) for n, p in bm.named_parameters())


@pytest.mark.parametrize("tm", [["to_q", "to_k", "to_v", "to_out.0", "add_k_proj", "add_v_proj"],
                                ["to_q", "to_k", "to_v", "to_out.0", "add_k_proj"],
                                "blocks.*(to_q|to_k|to_v|to_out.0|add_v_proj)"])
def test_lora_on_the_image_projections_refused(tm):
    bm = B200WanTransformer(_cfg(), device="cpu")
    with pytest.raises(NotImplementedError, match="add_"):
        bm.add_adapter(_Lora(target_modules=tm))


def test_config_refusals():
    with pytest.raises(NotImplementedError):  # image_dim without the added K/V projections (an inconsistent config)
        B200WanTransformer(WanConfig(image_dim=1280, num_layers=1), device="cpu")
    with pytest.raises(NotImplementedError):  # added K/V from a width other than the embedded image's
        B200WanTransformer(_cfg(added_kv_proj_dim=128), device="cpu")
    with pytest.raises(NotImplementedError):
        B200WanTransformer(_cfg(added_kv_proj_dim=None), device="cpu")
    with pytest.raises(NotImplementedError, match="pos_embed_seq_len"):  # FLF2V / use_last_frame
        B200WanTransformer(_cfg(pos_embed_seq_len=514), device="cpu")
    with pytest.raises(ValueError, match="multiple of 8"):
        B200WanTransformer(_cfg(image_dim=60), device="cpu")
    bm = B200WanTransformer(_cfg(), device="cpu")
    with pytest.raises(NotImplementedError):
        bm.enable_layerwise_casting(torch.float8_e4m3fn, skip_modules_pattern=("norm",))
    from finetrainers_b200.fsdp import FSDPState
    with pytest.raises(NotImplementedError):
        FSDPState(bm)


def test_input_refusals():
    """Refused before anything is launched, so on the CPU too."""
    bm = B200WanTransformer(_cfg(), device="cpu")
    bm.add_adapter(_Lora())
    x, t = torch.zeros(1, 36, 1, 2, 2), torch.zeros(1)
    txt, img = torch.zeros(1, 512, 64), torch.zeros(1, 257, 64)
    with pytest.raises(ValueError, match="needs encoder_hidden_states_image"):
        bm(x, t, txt)
    with pytest.raises(ValueError, match="512 text tokens"):
        bm(x, t, torch.zeros(1, 511, 64), encoder_hidden_states_image=img)
    with pytest.raises(ValueError, match=r"\[1, Li, 64\]"):
        bm(x, t, txt, encoder_hidden_states_image=torch.zeros(1, 257, 32))
    with pytest.raises(ValueError, match=r"\[1, Li, 64\]"):
        bm(x, t, txt, encoder_hidden_states_image=torch.zeros(2, 257, 64))
    # the trainer's path (the engine's forward) checks the same
    with pytest.raises(ValueError, match="512 text tokens"):
        bm._forward_impl(torch.zeros(1, 1, 144), torch.zeros(1, 64, 64), torch.zeros(1), None, 1, 1, 1, (), img)
    with pytest.raises(ValueError, match="needs encoder_hidden_states_image"):
        bm._forward_impl(torch.zeros(1, 1, 144), txt, torch.zeros(1), None, 1, 1, 1, ())
    # a text-to-video model still refuses an image context (tests/test_host_wan.py's refusal)
    t2v = B200WanTransformer(_cfg(in_channels=16, image_dim=None, added_kv_proj_dim=None), device="cpu")
    with pytest.raises(NotImplementedError):
        t2v(torch.zeros(1, 16, 1, 2, 2), t, txt, encoder_hidden_states_image=img)
    # the specification: an image-to-video batch needs its condition, mask and image embeddings
    spec = WanModelSpecification(bm.cfg)
    lat = {"latents": torch.zeros(1, 32, 2, 2, 2), "latents_mean": torch.zeros(16), "latents_std": torch.ones(16),
           "encoder_hidden_states_image": img}
    with pytest.raises(ValueError, match="latent_condition"):
        spec.forward(bm, {"encoder_hidden_states": txt}, dict(lat), torch.ones(1))
    with pytest.raises(ValueError, match="latent_condition_mask"):
        spec.forward(bm, {"encoder_hidden_states": txt}, dict(lat, latent_condition=torch.zeros(1, 32, 2, 2, 2),
                                                                latent_condition_mask=torch.zeros(1, 3, 2, 2, 2)),
                     torch.ones(1))


I2V_ENTRIES = ("imn", "imf", "imh", "img", "kv3", "k3h", "v3h", "lse3", "o2t", "o2i")


def _planner(cfg):
    bm = B200WanTransformer(cfg, device="meta")
    bm.lora_rank, bm.rpad, bm.lora_ffn = 32, 64, False
    bm._groups = bm._lora_groups()
    return bm


def test_workspace_plan_i2v_14b():
    from finetrainers_b200 import ops
    from finetrainers_b200.model import checkpointed_blocks
    cfg = WanConfig.wan_i2v_14b()
    cfg.num_layers = 3
    bm = _planner(cfg)
    d, H, hd, di, nl = 5120, 40, 128, 1280, 3
    B, S, L, Li = 1, 20280, 512, 257
    bf, f32 = torch.bfloat16, torch.float32
    plan = bm.workspace_plan(B, S, L, sm_count=132, Li=Li)
    want = {"imn": ((Li, di), bf), "imf": ((Li, di), bf), "imh": ((Li, d), bf), "img": ((Li, d), bf),
            "kv3": ((nl, Li, 2 * d), bf), "k3h": ((nl, B, H, Li, hd), bf), "v3h": ((nl, B, H, Li, hd), bf),
            "lse3": ((nl, B, H, S), f32), "o2t": ((S, d), bf), "o2i": ((S, d), bf)}
    assert {k: plan[k] for k in want} == want
    assert plan["delta"] == ((ops.attn_dual_bwd_ws_floats(B, H, S, L, head_dim=hd),), f32)
    assert plan["pred"] == ((S, 64), bf) and plan["kv2"] == ((nl, L, 2 * d), bf)
    # the same tensors as the text-to-video plan otherwise
    t2v = WanConfig.wan_14b()
    t2v.num_layers = 3
    base = _planner(t2v).workspace_plan(B, S, L, sm_count=132)
    assert {k: v for k, v in plan.items() if k not in I2V_ENTRIES and k != "delta"} == \
        {k: v for k, v in base.items() if k != "delta"}
    extra = sum(torch.Size(s).numel() * dt.itemsize for k, (s, dt) in plan.items() if k in I2V_ENTRIES)
    assert bm.workspace_bytes(B, S, L, sm_count=132, Li=Li) - _planner(t2v).workspace_bytes(B, S, L, sm_count=132) == \
        extra + 4 * (plan["delta"][0][0] - base["delta"][0][0])
    # checkpointing keeps the per-block image k|v and lse3; inference keeps one lse3 row and no backward scratch
    full = bm.workspace_plan(B, S, L, ckpt=checkpointed_blocks(3, "full"), sm_count=132, Li=Li)
    assert full["k3h"] == want["k3h"] and full["lse3"] == want["lse3"] and full["o2t"] == want["o2t"]
    inf = bm.workspace_plan(B, S, L, sm_count=132, inference=True, Li=Li)
    assert inf["lse3"] == ((1, B, H, S), f32) and inf["k3h"] == want["k3h"] and inf["imn"] == want["imn"]
    assert "o2t" not in inf and "o2i" not in inf and "delta" not in inf
    # an image-to-video plan needs its image token count, and a text-to-video plan takes none
    with pytest.raises(ValueError):
        bm.workspace_plan(B, S, L, sm_count=132)
    with pytest.raises(ValueError):
        _planner(t2v).workspace_plan(B, S, L, sm_count=132, Li=Li)


def test_t2v_plan_and_root_layout_unchanged():
    """The text-to-video plan has none of the image entries and the delta of the two single-context backwards; its
    root unit is the image-to-video one's prefix (but for the patch projection's K)."""
    from finetrainers_b200 import ops
    t2v = WanConfig.wan_14b()
    t2v.num_layers = 3
    bm = _planner(t2v)
    B, S, L, H, hd = 1, 20280, 512, 40, 128
    plan = bm.workspace_plan(B, S, L, sm_count=132)
    assert not set(plan) & set(I2V_ENTRIES)
    assert plan["delta"][0] == (max(ops.attn_bwd_ws_floats(B, H, S, S, head_dim=hd),
                                    ops.attn_bwd_ws_floats(B, H, S, L, head_dim=hd)),)
    assert [k for k, _ in bm._root_specs()] == ["proj_in.w", "proj_in.b", "t1.w", "t1.b", "t2.w", "t2.b", "ada.w",
                                                  "ada.b", "c1.w", "c1.b", "c2.w", "c2.b", "sst", "proj_out.w",
                                                  "proj_out.b", "Wkv2_all", "bkv2_all", "nk2_all"]
    i2v = _planner(WanConfig.wan_i2v_14b())._root_specs()
    t2v_specs = _planner(WanConfig.wan_14b())._root_specs()
    assert i2v[1:len(t2v_specs)] == t2v_specs[1:] and i2v[0] == ("proj_in.w", (5120, 144))
    assert [k for k, _ in i2v[len(t2v_specs):]] == ["img_n1.w", "img_n1.b", "img_ff1.w", "img_ff1.b", "img_ff2.w",
                                                      "img_ff2.b", "img_n2.w", "img_n2.b", "Wkv3_all", "bkv3_all",
                                                      "nk3_all"]


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_oracle_i2v_prologue_matches_the_reference_goldens():
    """The oracle's I2V prologue (the transformer input cat([x_t, mask, condition]) and the target) against the tensors
    the reference's own code produced, bit for bit in bf16 on the CPU: wan_i2v_golden.pt (stub transformer returning
    its input) and wan_i2v_call_golden.pt (stub transformer recording its arguments)."""
    for name in ("wan_i2v_golden.pt", "wan_i2v_call_golden.pt"):
        g = _load(name)
        hidden, target = I.i2v_prologue(g["moments"], g["cond_moments"], g["mask"], g["latents_mean"],
                                        g["latents_std"], g["eps"], g["noise"], g["sigmas"])
        assert hidden.shape[1] == 36
        assert torch.equal(hidden.view(torch.int16), g["hidden_states"].view(torch.int16)), name
        assert torch.equal(target.view(torch.int16), g["target"].view(torch.int16)), name


def _patch(x, order):
    B, C, F, H, W = x.shape
    t = x.reshape(B, C, F, H // 2, 2, W // 2, 2)
    t = t.permute(0, 2, 3, 5, 4, 6, 1) if order else t.permute(0, 2, 3, 5, 1, 4, 6)
    return t.reshape(B, F * (H // 2) * (W // 2), 4 * C)


def test_spec_call_surface_matches_the_reference(monkeypatch):
    """The engine's ``WanModelSpecification.forward`` calls the transformer with the keyword arguments, shapes, dtypes,
    timestep and 36-channel hidden_states the reference's own forward passed (wan_i2v_call_golden.pt), and leaves the
    same keys in latent_model_conditions.  The two libb2d launches it makes are replaced by torch restatements here
    (tests/test_gpu_wan_i2v.py runs the kernels)."""
    from finetrainers_b200 import ops

    def fake_prep(moments, cond, mask, eps, noise, mean, std, sig, x_in, target, B, C, Cm, F, H, W):
        assert all(t.is_contiguous() for t in (moments, cond, mask, eps, noise, mean, std, sig))
        assert torch.equal(mean, mean[:1].expand_as(mean)) and torch.equal(std, std[:1].expand_as(std))
        hidden, tg = I.i2v_prologue(moments, cond, mask, mean[0], std[0], eps, noise, sig)
        x_in.copy_(_patch(hidden, 0))
        target.copy_(_patch(tg, 1))

    def fake_permute(src, dst, B, C, F, H, W, order, unpatchify):
        assert unpatchify
        idx = _patch(torch.arange(dst.numel()).view(dst.shape), order)
        dst.view(-1)[idx.reshape(-1)] = src.reshape(-1)
        return dst

    monkeypatch.setattr(ops, "wan_i2v_prep", fake_prep)
    monkeypatch.setattr(ops, "patch_permute", fake_permute)
    g = _load("wan_i2v_call_golden.pt")
    calls = []

    class Stub:
        cfg = WanConfig(in_channels=36, image_dim=16, added_kv_proj_dim=1536, text_dim=8)

        def __call__(self, **kw):
            calls.append(kw)
            return (torch.zeros(2, 16, 2, 4, 6),)

    lat = {"latents": g["moments"], "latents_mean": g["latents_mean"], "latents_std": g["latents_std"],
           "latent_condition": g["cond_moments"], "latent_condition_mask": g["mask"],
           "encoder_hidden_states_image": g["encoder_hidden_states_image"]}
    _, target, _ = WanModelSpecification(Stub.cfg).forward(
        Stub(), {"encoder_hidden_states": g["encoder_hidden_states"]}, lat, g["sigmas"], noise=g["noise"],
        posterior_noise=g["eps"])
    (kw,) = calls
    assert {k: (tuple(v.shape), str(v.dtype)) if isinstance(v, torch.Tensor) else v for k, v in kw.items()} == g["args"]
    assert sorted(lat) == g["left"]
    assert torch.equal(kw["timestep"], g["timestep"])
    assert kw["encoder_hidden_states_image"] is g["encoder_hidden_states_image"]
    assert kw["encoder_hidden_states"] is g["encoder_hidden_states"]
    assert torch.equal(kw["hidden_states"].view(torch.int16), g["hidden_states"].view(torch.int16))
    assert torch.equal(target.view(torch.int16), g["target"].view(torch.int16))
