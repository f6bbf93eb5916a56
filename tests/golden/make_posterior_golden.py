"""Generates tests/golden/posterior_golden.pt from the REAL reference source (FINETRAINERS_SRC = a checkout of
a-r-r-o-w/finetrainers @ f476c37; the output is committed, so the tests never need the reference).

``DiagonalGaussianDistribution`` is pulled out of finetrainers/models/utils.py with ``ast`` and executed unmodified.  Its
one outside dependency, diffusers' ``randn_tensor``, is stubbed with its published same-device behaviour
(``torch.randn(shape, generator=generator, device=device, dtype=dtype)``); the stub also records the draw, so the golden
holds eps next to the sample.

Each case: bf16 moments [B, 2C, F, H, W] (mean | logvar, the training dtype the reference casts precomputed moments to),
a CPU generator seed, the eps the reference drew and the sample it returned.  logvar spans the clamp range and carries
values below -30, above 20, exactly at both bounds, +-inf and NaN.
Usage: FINETRAINERS_SRC=<checkout> python tests/golden/make_posterior_golden.py
"""
import ast
import os
import textwrap
from typing import Optional, Tuple  # noqa: F401 (names used by the extracted source)

import numpy as np
import torch

REF = os.environ.get("FINETRAINERS_SRC", ".")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "posterior_golden.pt")

# (B, C, F, H, W): C = 128 is LTX's latent width; F*H*W odd in the first, third and fourth
SHAPES = [(1, 8, 1, 3, 5), (2, 128, 2, 3, 3), (2, 16, 3, 1, 7), (1, 128, 3, 5, 7)]
EDGES = [-1e4, -31.0, -30.5, -30.0, -29.875, 19.875, 20.0, 20.5, 25.0, 1e4, float("inf"), float("-inf"), float("nan")]


def extract_class(path, name):
    src = open(os.path.join(REF, path)).read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.ClassDef) and node.name == name:
            return textwrap.dedent("\n".join(src.splitlines()[node.lineno - 1:node.end_lineno]))
    raise KeyError(name)


def main():
    drawn = []

    def randn_tensor(shape, generator=None, device=None, dtype=None, layout=None):
        t = torch.randn(shape, generator=generator, device=device, dtype=dtype)
        drawn.append(t.clone())
        return t

    ns = {"torch": torch, "np": np, "Optional": Optional, "Tuple": Tuple, "randn_tensor": randn_tensor}
    exec(extract_class("finetrainers/models/utils.py", "DiagonalGaussianDistribution"), ns)
    DGD = ns["DiagonalGaussianDistribution"]
    cases = []
    for i, (B, C, F, H, W) in enumerate(SHAPES):
        g = torch.Generator().manual_seed(100 + i)
        mean = torch.randn(B, C, F, H, W, generator=g) * 0.8
        logvar = torch.rand(B, C, F, H, W, generator=g) * 56.0 - 33.0   # [-33, 23): both clamp bounds crossed
        flat = logvar.view(-1)
        pos = torch.randperm(flat.numel(), generator=g)[:len(EDGES)]
        flat[pos] = torch.tensor(EDGES)
        moments = torch.cat([mean, logvar], dim=1).to(torch.bfloat16)
        seed = 1000 + i
        drawn.clear()
        sample = DGD(moments).sample(generator=torch.Generator().manual_seed(seed))
        assert len(drawn) == 1
        cases.append({"shape": (B, C, F, H, W), "moments": moments, "seed": seed, "eps": drawn[0], "sample": sample})
    torch.save({"cases": cases}, OUT)
    print("wrote", OUT, [(c["shape"], int(torch.isnan(c["sample"]).sum())) for c in cases])


if __name__ == "__main__":
    main()
