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


def test_mask_to_key_bias_on_cpu():
    """The provider's mask -> key-bias conversion: bool masks give -inf on the hidden keys, [1,1,1,Sk] and [Sk] masks
    broadcast over the batch, values at or below the floor (finfo.min of bf16 and fp32 included) become -inf, each
    sample is shifted so that its largest finite bias is 0, a mask repeated or expanded over heads is accepted and one
    that differs between heads is refused."""
    import torch
    from finetrainers_b200.attention import KEY_BIAS_FLOOR, mask_to_key_bias
    inf = float("-inf")
    keep = torch.tensor([[True, False, True], [False, False, True]])
    kb = mask_to_key_bias(keep[:, None, None, :], 2, 3)
    assert kb.dtype == torch.float32 and kb.is_contiguous()
    assert torch.equal(kb, torch.tensor([[0.0, inf, 0.0], [inf, inf, 0.0]]))
    for m in (torch.tensor([True, False, True]), torch.tensor([[[[True, False, True]]]])):
        assert torch.equal(mask_to_key_bias(m, 2, 3), torch.tensor([[0.0, inf, 0.0]] * 2))
    assert torch.equal(mask_to_key_bias(keep, 2, 3), kb)  # [B, Sk]
    assert torch.equal(mask_to_key_bias(~keep.any(-1, keepdim=True).expand(2, 3), 2, 3), torch.full((2, 3), inf))
    assert KEY_BIAS_FLOOR * 1.4426950408889634 > torch.finfo(torch.float32).min
    for dt in (torch.bfloat16, torch.float32):
        lo = torch.finfo(dt).min
        m = torch.tensor([[lo, -3.5, inf, 2.0], [lo, lo, lo, lo]], dtype=dt)[:, None, None, :]
        got = mask_to_key_bias(m, 2, 4)
        assert torch.equal(got, torch.tensor([[inf, -5.5, inf, 0.0], [inf] * 4]))
    # a common offset is removed: the kernel then sees the bias that gives the same softmax with a well-scaled lse
    m = torch.tensor([[-1e9] * 3, [-1e9, -1e9 - 64, 7.0]])
    assert torch.equal(mask_to_key_bias(m, 2, 3), torch.tensor([[0.0, 0.0, 0.0], [-1e9 - 7.0, -1e9 - 64 - 7.0, 0.0]]))
    assert torch.equal(mask_to_key_bias(torch.tensor([[1e38, -1e38]]), 1, 2), torch.tensor([[0.0, inf]]))
    same = keep[:, None, None, :].expand(2, 5, 1, 3)
    assert torch.equal(mask_to_key_bias(same, 2, 3), kb)
    assert torch.equal(mask_to_key_bias(same.contiguous(), 2, 3), kb)
    differ = same.clone()
    differ[1, 4, 0, 2] = False
    with pytest.raises(ValueError, match="every head"):
        mask_to_key_bias(differ, 2, 3)
    with pytest.raises(ValueError, match="key-only"):
        mask_to_key_bias(torch.zeros(2, 1, 4, 3), 2, 3)


@pytest.mark.parametrize("head_dim", [64, 128])
def test_attn_bwd_workspace_matches_header(head_dim):
    from finetrainers_b200 import ops
    header = open(os.path.join(ROOT, "include", "b2d.h")).read()
    assert "2*B*H*Sq floats, plus 8*2*B*H*Sk*head_dim floats when Sk <= 512" in header
    for B, H, Sq, Sk in [(1, 12, 32760, 512), (1, 12, 32760, 32760), (2, 8, 256, 513), (3, 2, 1, 1), (1, 32, 2688, 128)]:
        want = 2 * B * H * Sq + (8 * 2 * B * H * Sk * head_dim if Sk <= 512 else 0)
        assert ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=head_dim) == want
    assert ops.attn_bwd_ws_floats(1, 4, 640, 512) == ops.attn_bwd_ws_floats(1, 4, 640, 512, head_dim=64)
