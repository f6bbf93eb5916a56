"""Host-side checks of the Wan image-to-video kernel entry points: the two-context attention workspace formula of
include/b2d.h, and the wrapper refusing a short workspace before anything reaches the library."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("B,H,Sq,Sk1,d", [(1, 40, 20280, 512, 128), (2, 3, 1000, 383, 64), (1, 12, 300, 513, 128)])
def test_dual_bwd_workspace_is_the_single_one_plus_context_2_row_terms(B, H, Sq, Sk1, d):
    from finetrainers_b200 import ops
    single = 2 * B * H * Sq + (8 * 2 * B * H * Sk1 * d if Sk1 <= 512 else 0)
    assert ops.attn_bwd_ws_floats(B, H, Sq, Sk1, head_dim=d) == single
    assert ops.attn_dual_bwd_ws_floats(B, H, Sq, Sk1, head_dim=d) == single + 2 * B * H * Sq


def test_header_states_the_dual_workspace():
    header = open(os.path.join(ROOT, "include", "b2d.h")).read()
    decl = header[header.index("Its backward for a caller"):header.index("int b2d_attn_dual_bwd_hd")]
    assert re.search(r"W1 \+ 2\*B\*H\*Sq floats", decl) and "Sk1 <= 512" in decl


def test_short_dual_workspace_is_refused_before_the_library():
    from finetrainers_b200 import ops
    from finetrainers_b200.lib import B2DError
    B, H, Sq, Sk1, d = 1, 2, 130, 64, 128
    ws = torch.empty(ops.attn_dual_bwd_ws_floats(B, H, Sq, Sk1, head_dim=d) - 1)  # CPU tensor: never passed on
    with pytest.raises(B2DError, match="workspace too small"):
        ops.attn_dual_bwd(None, None, None, Sk1, None, None, 257, None, None, None, None, None, ws, None, None, None,
                          B, H, Sq, 0.1, head_dim=d)


def _golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "wan_i2v_golden.pt"), weights_only=False)


def test_oracle_i2v_prologue_matches_the_reference_golden():
    """The restatement the GPU prologue test uses (oracle.wan_oracle.prologue and normalize_latents, the condition mode
    taken as the normalised mean, cat([x_t, mask, condition], dim=1), a first-latent-frame mask) against the tensors
    the reference's own WanImageConditioningLatentEncodeProcessor / WanModelSpecification.forward produced, bit for bit
    in bf16 on the CPU."""
    from oracle import wan_oracle as O
    g = _golden()
    B, C = g["noise"].shape[:2]
    x_t, target = O.prologue(g["moments"], g["latents_mean"], g["latents_std"], g["eps"], g["noise"], g["sigmas"])
    cond = O.normalize_latents(g["cond_moments"][:, :C], g["latents_mean"], g["latents_std"])
    mask = torch.zeros_like(g["mask"])
    mask[:, :, 0] = 1
    assert torch.equal(mask, g["mask"]), "the reference's mask is 1 on the first latent frame only, on all 4 channels"
    ref = g["hidden_states"]
    assert ref.shape[1] == 2 * C + 4
    for got, want, what in ((x_t, ref[:, :C], "x_t"), (mask, ref[:, C:C + 4], "mask"), (cond, ref[:, C + 4:], "cond"),
                            (target, g["target"], "target")):
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), what


def test_non_contiguous_prologue_operand_is_refused_before_the_library():
    """The reference's condition mask is a transposed view; the kernel reads dense arrays, so a strided operand is
    refused rather than misread."""
    from finetrainers_b200 import ops
    from finetrainers_b200.lib import B2DError
    mask = _golden()["mask"]
    assert not mask.is_contiguous()
    t = torch.zeros(8, dtype=torch.bfloat16)
    with pytest.raises(B2DError, match="cond_mask must be contiguous"):
        ops.wan_i2v_prep(t, t, mask, t, t, t, t, t, t, t, 2, 16, 4, 2, 4, 6)
