"""Generates tests/golden/ltx_golden.pt from the REAL reference sources (FINETRAINERS_SRC = a checkout of
a-r-r-o-w/finetrainers @ f476c37; the outputs are committed, so the tests never need the reference).

The reference package cannot be imported (diffusers/peft are not installed), so the torch-only functions on the hot
path are pulled out of their files with ``ast`` and executed unmodified:

  finetrainers/functional/diffusion.py ............ flow_match_xt, flow_match_target        (imported as a module)
  finetrainers/models/ltx_video/base_specification.py  _normalize_latents, _pack_latents    (static methods, source-extracted)
  finetrainers/patches/models/ltx_video/patch.py ....... apply_rotary_emb                   (nested function, source-extracted)
  finetrainers/patches/dependencies/diffusers/rms_norm.py  _patched_rms_norm_forward        (diffusers.utils helpers stubbed)
  finetrainers/utils/diffusion.py ...................... compute_density_for_timestep_sampling, prepare_sigmas
                                                         (scheduler classes stubbed: only isinstance() is used)
Usage: python tests/golden/make_golden.py
"""
import ast
import importlib.util
import math
import os
import textwrap
from typing import Optional, Union  # noqa: F401 (names used by the extracted sources)

import torch

REF = os.environ.get("FINETRAINERS_SRC", ".")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ltx_golden.pt")


def extract(path, name):
    src = open(os.path.join(REF, path)).read()
    tree = ast.parse(src)
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name == name:
            seg = ast.get_source_segment(src, node)
            lines = src.splitlines()[node.lineno - 1:node.end_lineno]
            code = textwrap.dedent("\n".join(lines))
            code = "\n".join(l for l in code.splitlines() if not l.strip().startswith("@staticmethod"))
            return code
    raise KeyError(name)


def main():
    g = {}
    torch.manual_seed(0)
    # ---- functional/diffusion.py (imports torch only)
    spec = importlib.util.spec_from_file_location("ref_functional_diffusion", os.path.join(REF, "finetrainers/functional/diffusion.py"))
    FF = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(FF)
    x0 = torch.randn(2, 8, 3, 4, 5).bfloat16()
    n = torch.randn(2, 8, 3, 4, 5).bfloat16()
    t = torch.tensor([0.3, 0.811]).view(2, 1, 1, 1, 1)
    g["fm_x0"], g["fm_n"], g["fm_t"] = x0, n, t
    g["fm_xt"] = FF.flow_match_xt(x0, n, t)
    g["fm_target"] = FF.flow_match_target(n, x0)

    ns = {"torch": torch, "math": math, "Optional": Optional, "Union": Union}
    # ---- _normalize_latents / _pack_latents
    exec(extract("finetrainers/models/ltx_video/base_specification.py", "_normalize_latents"), ns)
    exec(extract("finetrainers/models/ltx_video/base_specification.py", "_pack_latents"), ns)
    lat = torch.randn(2, 8, 3, 4, 5).bfloat16()
    mean = torch.randn(2, 8) * 0.1
    std = 1 + 0.1 * torch.rand(2, 8)
    g["nl_lat"], g["nl_mean"], g["nl_std"] = lat, mean, std
    g["nl_out"] = ns["_normalize_latents"](lat, mean, std)
    g["pack_out"] = ns["_pack_latents"](lat, 1, 1)

    # ---- apply_rotary_emb (TP-safe variant of the patch)
    exec(extract("finetrainers/patches/models/ltx_video/patch.py", "apply_rotary_emb"), ns)
    x = torch.randn(2, 6, 32).bfloat16()
    ang = torch.randn(2, 6, 16)
    cos = ang.cos().repeat_interleave(2, -1)
    sin = ang.sin().repeat_interleave(2, -1)
    g["rope_x"], g["rope_cos"], g["rope_sin"] = x, cos, sin
    g["rope_out"] = ns["apply_rotary_emb"](x, (cos, sin))

    # ---- patched RMSNorm forward
    ns["is_torch_npu_available"] = lambda: False
    ns["is_torch_version"] = lambda op, v: True  # torch >= 2.4 here
    ns["nn"] = torch.nn
    exec(extract("finetrainers/patches/dependencies/diffusers/rms_norm.py", "_patched_rms_norm_forward"), ns)

    class _M:  # the attributes the patched forward reads
        pass

    for tag, w in (("affine", (1 + 0.1 * torch.randn(32)).bfloat16()), ("noaffine", None)):
        m = _M()
        m.weight, m.bias, m.eps = w, None, 1e-5 if w is not None else 1e-6
        xin = torch.randn(3, 5, 32).bfloat16()
        g[f"rms_{tag}_x"], g[f"rms_{tag}_w"], g[f"rms_{tag}_eps"] = xin, w, m.eps
        g[f"rms_{tag}_out"] = ns["_patched_rms_norm_forward"](m, xin)

    # ---- sigma sampling
    class FlowMatchEulerDiscreteScheduler:  # stub: only isinstance() is exercised
        pass

    class CogVideoXDDIMScheduler:
        pass

    ns["FlowMatchEulerDiscreteScheduler"] = FlowMatchEulerDiscreteScheduler
    ns["CogVideoXDDIMScheduler"] = CogVideoXDDIMScheduler
    exec(extract("finetrainers/utils/diffusion.py", "compute_density_for_timestep_sampling"), ns)
    exec(extract("finetrainers/utils/diffusion.py", "prepare_sigmas"), ns)
    sig_table = torch.cat([torch.linspace(1, 1000, 1000).flip(0) / 1000.0, torch.zeros(1)])
    for scheme in ("none", "logit_normal", "mode"):
        gen = torch.Generator().manual_seed(1234)
        g[f"sig_{scheme}"] = ns["prepare_sigmas"](FlowMatchEulerDiscreteScheduler(), sig_table, 16, 1000, scheme, 0.0, 1.0,
                                                  1.29, torch.device("cpu"), gen)
    g["sig_table"] = sig_table
    torch.save(g, OUT)
    print("wrote", OUT, {k: (tuple(v.shape) if torch.is_tensor(v) else v) for k, v in g.items()})


if __name__ == "__main__":
    main()
