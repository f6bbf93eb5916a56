"""Generates tests/golden/clip_golden.pt from the REAL reference gradient-clipping code
(finetrainers/utils/torch.py: clip_grad_norm_ :99-161, _get_total_norm :299-340,
_clip_grads_with_norm_ :343-...), pulled out of the file with ``ast`` and executed unmodified (the package cannot be
imported here: finetrainers.logging pulls in diffusers).  The output is committed.
Usage: python tests/golden/make_clip_golden.py"""
import ast
import math
import os
import textwrap
from typing import Dict, List, Optional, Tuple, Union  # noqa: F401 (used by the extracted sources)

import torch
import torch.distributed as dist
import torch.distributed.tensor  # noqa: F401

REF = os.path.join(os.environ.get("FINETRAINERS_SRC", "."), "finetrainers/utils/torch.py")  # a-r-r-o-w/finetrainers @ f476c37
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "clip_golden.pt")


def main():
    src = open(REF).read()
    ns = {"torch": torch, "math": math, "dist": dist, "Dict": Dict, "List": List, "Optional": Optional, "Tuple": Tuple,
          "Union": Union}
    want = {"_get_total_norm", "_clip_grads_with_norm_", "clip_grad_norm_", "_get_foreach_kernels_supported_devices",
            "_group_tensors_by_device_and_dtype", "_device_has_foreach_support", "_has_foreach_support"}
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name in want:
            first = min([node.lineno] + [d.lineno for d in node.decorator_list])
            exec(textwrap.dedent("\n".join(src.splitlines()[first - 1:node.end_lineno])), ns)
    g = {}
    torch.manual_seed(0)
    for tag, scale in (("big", 3.0), ("small", 1e-3)):   # one case that clips, one that does not
        params = [torch.nn.Parameter(torch.randn(s)) for s in ((16, 256), (256, 16), (17,), (3, 5, 7))]
        for p in params:
            p.grad = torch.randn_like(p) * scale
        # (plain Parameters: the reference takes its foreach path for them, torch._foreach_norm / _foreach_mul_)
        g[f"{tag}_grads_in"] = [p.grad.clone() for p in params]
        total = ns["clip_grad_norm_"](params, 1.0)
        g[f"{tag}_total_norm"] = total.clone()
        g[f"{tag}_grads_out"] = [p.grad.clone() for p in params]
    torch.save(g, OUT)
    print("wrote", OUT, {k: (v.item() if torch.is_tensor(v) and v.ndim == 0 else len(v)) for k, v in g.items()})


if __name__ == "__main__":
    main()
