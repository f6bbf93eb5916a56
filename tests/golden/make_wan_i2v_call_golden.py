"""Writes wan_i2v_call_golden.pt: what the reference's OWN WanModelSpecification.forward hands the transformer in an
image-to-video training step, recorded by a stub transformer.

Run from the repository root with the finetrainers reference checkout given as the first argument:
    python tests/golden/make_wan_i2v_call_golden.py /path/to/finetrainers
As make_wan_i2v_golden.py (whose AST extraction it reuses), it imports nothing from the reference package.  It runs the
reference's WanImageConditioningLatentEncodeProcessor.forward (stub VAE) for the condition and its mask, then
WanModelSpecification.forward with latent_model_conditions holding the moments, the condition, the mask and
encoder_hidden_states_image (as the reference's latent processors deliver them) and condition_model_conditions holding
encoder_hidden_states.  The stub transformer records every keyword argument.  Stored: the recorded argument names,
shapes and dtypes, the 36-channel hidden_states and timestep it was given, the inputs, and the keys left in
latent_model_conditions.  This fixes the call surface and the prologue; the transformer's arithmetic is not pinned by
it (DESIGN §2).
"""
import ast
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_wan_i2v_golden as G  # noqa: E402


def main(ref):
    typing = __import__("typing")
    ns = {"torch": torch, "np": None, **{k: getattr(typing, k) for k in ("Optional", "Tuple", "Dict", "List", "Any",
                                                                          "Union")}}
    spec_py = os.path.join(ref, "finetrainers/models/wan/base_specification.py")
    nodes = (G._extract(os.path.join(ref, "finetrainers/models/utils.py"), ["DiagonalGaussianDistribution"])
             + G._extract(os.path.join(ref, "finetrainers/functional/diffusion.py"), ["flow_match_xt",
                                                                                     "flow_match_target"])
             + G._extract(spec_py, ["_normalize_latents"])
             + [G._method(spec_py, "WanImageConditioningLatentEncodeProcessor", "forward"),
                G._method(spec_py, "WanModelSpecification", "forward")])
    for n in nodes:
        n.decorator_list = []
    ns["AutoencoderKLWan"] = ns["WanTransformer3DModel"] = object
    exec(compile(ast.Module(body=nodes, type_ignores=[]), "reference", "exec"), ns)
    ns["DiagonalGaussianDistribution"].mode = lambda self: self.mean  # diffusers' mode()
    ns["FF"] = types.SimpleNamespace(flow_match_xt=ns["flow_match_xt"], flow_match_target=ns["flow_match_target"])

    g = torch.Generator().manual_seed(31337)
    B, C, num_frames, H, W, L, Li, text_dim, image_dim = 2, 16, 5, 4, 6, 512, 257, 8, 16
    F = (num_frames - 1) // 4 + 1
    moments = torch.cat([torch.randn(B, C, F, H, W, generator=g),
                         torch.rand(B, C, F, H, W, generator=g) * 8 - 6], 1).to(torch.bfloat16)
    cond_moments = torch.cat([torch.randn(B, C, F, H, W, generator=g) * 2,
                              torch.rand(B, C, F, H, W, generator=g) * 8 - 6], 1).to(torch.bfloat16)
    vae_mean = (torch.randn(C, generator=g) * 0.3).tolist()
    vae_std = (torch.rand(C, generator=g) + 0.5).tolist()
    eps = torch.randn(B, C, F, H, W, generator=g).to(torch.bfloat16)
    sigmas = torch.rand(B, generator=g)
    ehs = torch.randn(B, L, text_dim, generator=g).to(torch.bfloat16)
    ehs_img = torch.randn(B, Li, image_dim, generator=g).to(torch.bfloat16)

    vae = types.SimpleNamespace(device=torch.device("cpu"), dtype=torch.bfloat16, _encode=lambda video: cond_moments,
                                config=types.SimpleNamespace(latents_mean=vae_mean, latents_std=vae_std))
    proc = types.SimpleNamespace(output_names=["latent_condition", "latents_mean", "latents_std",
                                               "latent_condition_mask"], use_last_frame=False)
    cond = ns["WanImageConditioningLatentEncodeProcessor_forward"](
        proc, vae, video=torch.zeros(B, num_frames, 3, 8 * H, 8 * W), compute_posterior=False)

    ns["randn_tensor"] = lambda shape, generator=None, device=None, dtype=None: eps.clone()
    spec = types.SimpleNamespace(transformer_config={"image_dim": image_dim}, _normalize_latents=ns["_normalize_latents"])
    calls = []

    def transformer(**kw):
        calls.append(kw)
        return (torch.zeros(B, C, F, H, W),)

    latent_conditions = {"latents": moments, "latents_mean": cond["latents_mean"], "latents_std": cond["latents_std"],
                         "latent_condition": cond["latent_condition"],
                         "latent_condition_mask": cond["latent_condition_mask"], "encoder_hidden_states_image": ehs_img}
    noise_seed = 11
    _, target, _ = ns["WanModelSpecification_forward"](
        spec, transformer, {"encoder_hidden_states": ehs}, latent_conditions, sigmas.view(B, 1, 1, 1, 1),
        generator=torch.Generator().manual_seed(noise_seed))
    (kw,) = calls
    noise = torch.zeros(B, C, F, H, W, dtype=torch.bfloat16).normal_(generator=torch.Generator().manual_seed(noise_seed))
    out = dict(args={k: (tuple(v.shape), str(v.dtype)) if isinstance(v, torch.Tensor) else v for k, v in kw.items()},
               left=sorted(latent_conditions), hidden_states=kw["hidden_states"], timestep=kw["timestep"],
               target=target, moments=moments, cond_moments=cond_moments, mask=cond["latent_condition_mask"],
               latents_mean=cond["latents_mean"], latents_std=cond["latents_std"], eps=eps, noise=noise,
               sigmas=sigmas, encoder_hidden_states=ehs, encoder_hidden_states_image=ehs_img)
    torch.save(out, os.path.join(os.path.dirname(os.path.abspath(__file__)), "wan_i2v_call_golden.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
