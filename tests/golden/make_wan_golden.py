"""Writes wan_golden.pt: the Wan training prologue computed by the reference's OWN torch code, run on the CPU in bf16.

Run from the repository root with the finetrainers reference checkout given as the first argument:
    python tests/golden/make_wan_golden.py /path/to/finetrainers
The generator imports nothing from the reference package (its modules import diffusers, which this project does not
need); it extracts, by name, the torch-only definitions the Wan prologue calls from the reference's sources and runs
them: WanModelSpecification._normalize_latents (models/wan/base_specification.py), DiagonalGaussianDistribution
(models/utils.py; its randn_tensor call is answered with the stored eps draw) and flow_match_xt / flow_match_target
(functional/diffusion.py).  Only the resulting tensors are committed.
"""
import ast
import os
import sys

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


def main(ref):
    ns = {"torch": torch, "Optional": __import__("typing").Optional, "Tuple": __import__("typing").Tuple, "np": None}
    nodes = (_extract(os.path.join(ref, "finetrainers/models/utils.py"), ["DiagonalGaussianDistribution"])
             + _extract(os.path.join(ref, "finetrainers/functional/diffusion.py"), ["flow_match_xt", "flow_match_target"])
             + _extract(os.path.join(ref, "finetrainers/models/wan/base_specification.py"), ["_normalize_latents"]))
    for n in nodes:
        n.decorator_list = []
    exec(compile(ast.Module(body=nodes, type_ignores=[]), "reference", "exec"), ns)
    g = torch.Generator().manual_seed(20240)
    B, C, F, H, W = 2, 16, 2, 4, 6
    moments = torch.cat([torch.randn(B, C, F, H, W, generator=g),
                         torch.rand(B, C, F, H, W, generator=g) * 60 - 35], 1).to(torch.bfloat16)
    latents_mean = torch.randn(C, generator=g) * 0.3
    latents_std = 1.0 / (torch.rand(C, generator=g) + 0.5)
    eps = torch.randn(B, C, F, H, W, generator=g).to(torch.bfloat16)
    noise = torch.randn(B, C, F, H, W, generator=g).to(torch.bfloat16)
    sigmas = torch.rand(B, generator=g)
    ns["randn_tensor"] = lambda shape, generator=None, device=None, dtype=None: eps.clone()
    norm = ns["_normalize_latents"]
    mu, logvar = torch.chunk(moments, 2, dim=1)
    latents = torch.cat([norm(mu, latents_mean, latents_std), norm(logvar, latents_mean, latents_std)], dim=1)
    x0 = ns["DiagonalGaussianDistribution"](latents).sample(generator=None)
    t = sigmas.view(B, 1, 1, 1, 1)
    x_t = ns["flow_match_xt"](x0, noise, t).to(x0)
    target = ns["flow_match_target"](noise, x0)
    out = dict(moments=moments, latents_mean=latents_mean, latents_std=latents_std, eps=eps, noise=noise,
               sigmas=sigmas, x_t=x_t, target=target)
    torch.save(out, os.path.join(os.path.dirname(os.path.abspath(__file__)), "wan_golden.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
