import torch


def rnd(*shape, scale=1.0, dtype=torch.bfloat16, device="cuda"):
    return (torch.randn(*shape, device=device) * scale).to(dtype)


def rel_err(got, ref, floor=1e-6):
    """max |got - ref| relative to the reference's max magnitude (floored so exact-zero references compare absolutely)."""
    got, ref = got.float(), ref.float()
    return ((got - ref).abs().max() / max(ref.abs().max().item(), floor)).item()


def build_pair(cfg_kwargs, rank, seed=0, lora_b_std=0.02, device="cuda"):
    """oracle (CPU, fp32 math, bf16-valued base weights) + H100 model with identical parameters."""
    from oracle import ltx_oracle as O
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    om = O.LTXTransformerOracle(O.LTXConfig(**cfg_kwargs))
    O.add_lora(om, rank, rank)
    O.synthetic_init_(om, seed=seed, lora_b_std=lora_b_std)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    bm = B200LTXTransformer(LTXConfig(**cfg_kwargs), torch.bfloat16, device)
    bm.add_adapter(rank, rank)
    bm.load_state_dict(om.state_dict(), strict=True)
    bm.prepare()
    return O, om, bm


def run_b200_micro(bm, batch, scheme="none"):
    from finetrainers_b200.trainer import SFTTrainStep
    st = SFTTrainStep(bm, flow_weighting_scheme=scheme)
    st.spec.first_frame_conditioning_p = 0.0
    cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(),
            "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
    lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(),
           "latents_std": batch["latents_std"].cuda()}
    st.micro_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda())
    torch.cuda.synchronize()
    B = batch["latents"].shape[0]
    S = batch["latents"].shape[2] * batch["latents"].shape[3] * batch["latents"].shape[4]
    ws = bm._workspace(B, S, batch["encoder_hidden_states"].shape[1])
    return st, st.loss_buf.item(), ws["pred"].view(B, S, -1).float().cpu()


SMALL = dict(in_channels=32, out_channels=32, num_attention_heads=4, attention_head_dim=64, cross_attention_dim=256,
             num_layers=2, caption_channels=128)
