"""CPU: the attention kernels of every head dimension compile without spills, and the Python workspace size agrees with
the formula include/b2d.h states."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuobjdump():
    return shutil.which("cuobjdump") or next(
        (p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


def test_attention_kernels_use_no_local_memory():
    """Every attention kernel instantiation (d = 64 and d = 128) keeps its working set in registers: a spill would put
    local-memory traffic into the inner loop."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    from finetrainers_b200 import lib
    path = lib.build()
    out = subprocess.run([tool, "--dump-resource-usage", path], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r"Function (\S*attn\S*):\s*(.*)", out))
    for d in (64, 128):
        for kern in ("attn_fwd_kernel", "attn_bwd_kernelILb1E", "attn_bwd_kernelILb0E", "attn_delta_kernel"):
            assert any(kern in name and f"Li{d}E" in name for name in usage), (kern, d, sorted(usage))
    assert "attn_dkv_reduce_kernel" in " ".join(usage)
    for name, res in usage.items():
        assert re.search(r"\bLOCAL:0\b", res) and re.search(r"\bSTACK:0\b", res), (name, res)


@pytest.mark.parametrize("head_dim", [64, 128])
def test_attn_bwd_workspace_matches_header(head_dim):
    from finetrainers_b200 import ops
    header = open(os.path.join(ROOT, "include", "b2d.h")).read()
    assert "2*B*H*Sq floats, plus 8*2*B*H*Sk*head_dim floats when Sk <= 512" in header
    for B, H, Sq, Sk in [(1, 12, 32760, 512), (1, 12, 32760, 32760), (2, 8, 256, 513), (3, 2, 1, 1), (1, 32, 2688, 128)]:
        want = 2 * B * H * Sq + (8 * 2 * B * H * Sk * head_dim if Sk <= 512 else 0)
        assert ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=head_dim) == want
    assert ops.attn_bwd_ws_floats(1, 4, 640, 512) == ops.attn_bwd_ws_floats(1, 4, 640, 512, head_dim=64)
