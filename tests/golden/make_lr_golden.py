"""Generates tests/golden/lr_golden.json from the REAL reference learning-rate lambdas
(finetrainers/optimizer.py:250-432), pulled out of the file with ``ast`` and executed unmodified (the
package itself cannot be imported here: diffusers is absent).  The output is committed.
Usage: python tests/golden/make_lr_golden.py"""
import ast
import json
import math
import os
import textwrap
from typing import Callable  # noqa: F401 (used by the extracted sources)

REF = os.path.join(os.environ.get("FINETRAINERS_SRC", "."), "finetrainers/optimizer.py")  # a-r-r-o-w/finetrainers @ f476c37
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lr_golden.json")
NAMES = ["get_constant_schedule", "get_constant_schedule_with_warmup", "get_piecewise_constant_schedule",
         "get_linear_schedule_with_warmup", "get_cosine_schedule_with_warmup",
         "get_cosine_with_hard_restarts_schedule_with_warmup", "get_polynomial_decay_schedule_with_warmup"]


def main():
    src = open(REF).read()
    ns = {"math": math, "Callable": Callable}
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name in NAMES:
            exec(textwrap.dedent("\n".join(src.splitlines()[node.lineno - 1:node.end_lineno])), ns)
    steps = list(range(0, 64)) + [99, 100, 101, 499, 500, 999, 1000, 1001, 5000]
    cases = [
        ("constant", {}, ns["get_constant_schedule"]()),
        ("constant_with_warmup", {"num_warmup_steps": 1000}, ns["get_constant_schedule_with_warmup"](1000)),
        ("constant_with_warmup", {"num_warmup_steps": 0}, ns["get_constant_schedule_with_warmup"](0)),
        ("piecewise_constant", {"step_rules": "1:10,0.1:20,0.01:30,0.005"},
         ns["get_piecewise_constant_schedule"]("1:10,0.1:20,0.01:30,0.005")),
        ("linear", {"num_warmup_steps": 10, "num_training_steps": 1000}, ns["get_linear_schedule_with_warmup"](10, 1000)),
        ("cosine", {"num_warmup_steps": 10, "num_training_steps": 1000, "num_cycles": 1},
         ns["get_cosine_schedule_with_warmup"](10, 1000, 1)),
        ("cosine_with_restarts", {"num_warmup_steps": 0, "num_training_steps": 500, "num_cycles": 1},
         ns["get_cosine_with_hard_restarts_schedule_with_warmup"](0, 500, 1)),
        ("cosine_with_restarts", {"num_warmup_steps": 20, "num_training_steps": 1000, "num_cycles": 3},
         ns["get_cosine_with_hard_restarts_schedule_with_warmup"](20, 1000, 3)),
        ("polynomial", {"num_warmup_steps": 10, "num_training_steps": 1000, "lr_init": 5e-5, "lr_end": 1e-7, "power": 2.0},
         ns["get_polynomial_decay_schedule_with_warmup"](10, 1000, 5e-5, 1e-7, 2.0)),
    ]
    out = [{"name": n, "kwargs": kw, "steps": steps, "factors": [float(fn(s)) for s in steps]} for n, kw, fn in cases]
    json.dump(out, open(OUT, "w"), indent=1)
    print("wrote", OUT, len(out), "cases")


if __name__ == "__main__":
    main()
