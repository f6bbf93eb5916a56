"""Writes wan_i2v_golden.pt: the Wan image-to-video training prologue computed by the reference's OWN torch code, run on
the CPU in bf16.

Run from the repository root with the finetrainers reference checkout given as the first argument:
    python tests/golden/make_wan_i2v_golden.py /path/to/finetrainers
As make_wan_golden.py, it imports nothing from the reference package; it extracts by name, from the reference's
sources, and runs:
  * WanImageConditioningLatentEncodeProcessor.forward (models/wan/base_specification.py) with a stub VAE whose _encode
    returns the stored condition moments: it builds the reference's own condition mask;
  * WanModelSpecification.forward (same file) with a stub self (transformer_config={"image_dim": 1280}, the extracted
    _normalize_latents) and a stub transformer that returns its hidden_states: that is the reference's own 36-channel
    input cat([x_t, mask, condition]);
  * DiagonalGaussianDistribution (models/utils.py; its randn_tensor call is answered with the stored eps draw) and
    flow_match_xt / flow_match_target (functional/diffusion.py).
The specification imports diffusers' DiagonalGaussianDistribution, which is models/utils.py's class (copied from
diffusers, plus its _dim argument) together with diffusers' mode(), `return self.mean`; that one method is added here.
Only the resulting tensors are committed.
"""
import ast
import os
import sys
import types

import torch


def _extract(path, names):
    tree = ast.parse(open(path).read())
    found = {}
    for node in ast.walk(tree):
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names and node.name not in found:
            found[node.name] = node
    missing = set(names) - set(found)
    assert not missing, (path, missing)
    return [found[n] for n in names]


def _method(path, cls, name):
    """The FunctionDef `name` of class `cls`, renamed cls_name."""
    tree = ast.parse(open(path).read())
    for node in ast.walk(tree):
        if isinstance(node, ast.ClassDef) and node.name == cls:
            for f in node.body:
                if isinstance(f, ast.FunctionDef) and f.name == name:
                    f.name = f"{cls}_{name}"
                    f.decorator_list = []
                    return f
    raise AssertionError((path, cls, name))


def main(ref):
    typing = __import__("typing")
    ns = {"torch": torch, "np": None, **{k: getattr(typing, k) for k in ("Optional", "Tuple", "Dict", "List", "Any",
                                                                          "Union")}}
    spec_py = os.path.join(ref, "finetrainers/models/wan/base_specification.py")
    nodes = (_extract(os.path.join(ref, "finetrainers/models/utils.py"), ["DiagonalGaussianDistribution"])
             + _extract(os.path.join(ref, "finetrainers/functional/diffusion.py"), ["flow_match_xt", "flow_match_target"])
             + _extract(spec_py, ["_normalize_latents"])
             + [_method(spec_py, "WanImageConditioningLatentEncodeProcessor", "forward"),
                _method(spec_py, "WanModelSpecification", "forward")])
    for n in nodes:
        n.decorator_list = []
    ns["AutoencoderKLWan"] = ns["WanTransformer3DModel"] = object
    exec(compile(ast.Module(body=nodes, type_ignores=[]), "reference", "exec"), ns)
    ns["DiagonalGaussianDistribution"].mode = lambda self: self.mean  # diffusers' mode()
    ns["FF"] = types.SimpleNamespace(flow_match_xt=ns["flow_match_xt"], flow_match_target=ns["flow_match_target"])

    g = torch.Generator().manual_seed(20241)
    B, C, num_frames, H, W = 2, 16, 5, 4, 6  # 5 video frames -> 2 latent frames: the mask has ones and zeros
    F = (num_frames - 1) // 4 + 1
    moments = torch.cat([torch.randn(B, C, F, H, W, generator=g),
                         torch.rand(B, C, F, H, W, generator=g) * 20 - 10], 1).to(torch.bfloat16)
    cond_moments = torch.cat([torch.randn(B, C, F, H, W, generator=g) * 2,
                              torch.rand(B, C, F, H, W, generator=g) * 20 - 10], 1).to(torch.bfloat16)
    vae_mean = (torch.randn(C, generator=g) * 0.3).tolist()
    vae_std = (torch.rand(C, generator=g) + 0.5).tolist()
    eps = torch.randn(B, C, F, H, W, generator=g).to(torch.bfloat16)
    sigmas = torch.rand(B, generator=g)

    vae = types.SimpleNamespace(device=torch.device("cpu"), dtype=torch.bfloat16, _encode=lambda video: cond_moments,
                                config=types.SimpleNamespace(latents_mean=vae_mean, latents_std=vae_std))
    proc = types.SimpleNamespace(output_names=["latent_condition", "latents_mean", "latents_std",
                                               "latent_condition_mask"], use_last_frame=False)
    video = torch.zeros(B, num_frames, 3, 8 * H, 8 * W)
    cond = ns["WanImageConditioningLatentEncodeProcessor_forward"](proc, vae, video=video, compute_posterior=False)

    ns["randn_tensor"] = lambda shape, generator=None, device=None, dtype=None: eps.clone()
    spec = types.SimpleNamespace(transformer_config={"image_dim": 1280}, _normalize_latents=ns["_normalize_latents"])
    transformer = lambda hidden_states, **kw: (hidden_states,)  # noqa: E731
    latent_conditions = {"latents": moments, "latents_mean": cond["latents_mean"], "latents_std": cond["latents_std"],
                         "latent_condition": cond["latent_condition"],
                         "latent_condition_mask": cond["latent_condition_mask"]}
    noise_seed = 7
    hidden, target, _ = ns["WanModelSpecification_forward"](
        spec, transformer, {}, latent_conditions, sigmas.view(B, 1, 1, 1, 1),
        generator=torch.Generator().manual_seed(noise_seed))
    # the spec's noise draw: zeros_like(latents).normal_(generator) on the bf16 latents, the only draw from `generator`
    noise = torch.zeros(B, C, F, H, W, dtype=torch.bfloat16).normal_(generator=torch.Generator().manual_seed(noise_seed))
    out = dict(moments=moments, cond_moments=cond_moments, mask=cond["latent_condition_mask"],
               latents_mean=cond["latents_mean"], latents_std=cond["latents_std"], eps=eps, noise=noise, sigmas=sigmas,
               hidden_states=hidden, target=target)
    torch.save(out, os.path.join(os.path.dirname(os.path.abspath(__file__)), "wan_i2v_golden.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
