"""GPU: the attention backward with 128-row streamed tiles at head_dim 64.  Its results are pinned bit for bit by
tests/golden/attn_bwd_bits.json (LTX self- and cross-attention, the 13B self-attention at head_dim 128, ragged and split
shapes), and every streamed-tile edge of the dK/dV and dQ passes is checked against fp64, with and without a key bias,
inside NaN-filled output and workspace buffers."""
import importlib.util
import json
import os

import pytest
import torch

from _util import rel_err
from test_gpu_attention_conformance import _run
from test_gpu_attention_hd128 import _ref64

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_spec = importlib.util.spec_from_file_location("make_attn_bwd_bits", os.path.join(GOLDEN, "make_attn_bwd_bits.py"))
bits = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(bits)

# streamed rows around every multiple of 64 and 128 up to three tiles, plus a long ragged range
EDGES = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 1000]


@pytest.mark.parametrize("case", sorted(bits.CASES))
def test_attn_bwd_reproduces_golden_bits(case):
    with open(os.path.join(GOLDEN, "attn_bwd_bits.json")) as f:
        want = json.load(f)[case]
    assert bits.hashes(case) == want


def _key_bias(B, Sk, seed):
    """uniform in [-4, 4) on the kept keys, -10000 on the last fifth"""
    gen = torch.Generator().manual_seed(seed)
    kb = torch.rand(B, Sk, generator=gen) * 8 - 4
    kb[:, Sk - Sk // 5:] = -10000.0
    return kb.cuda()


def _check(B, H, Sq, Sk, bias, seed):
    d = 64
    gen = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, H, S, d, generator=gen).bfloat16().cuda() for S in (Sq, Sk, Sk))
    g = torch.randn(B, H, Sq, d, generator=gen).bfloat16().cuda()
    kb = _key_bias(B, Sk, seed) if bias else None
    out, lse, dq, dk, dv = _run(q, k, v, kb, 0.125, g.transpose(1, 2).reshape(B, Sq, H * d).contiguous(), head_dim=d)
    for t in (out, lse, dq, dk, dv):
        assert torch.isfinite(t).all()
    ro, rl, rdq, rdk, rdv = _ref64(q, k, v, kb, 0.125, g)
    assert rel_err(out, ro.transpose(1, 2).flatten(2)) < 1e-2
    assert (lse.double() - rl).abs().max().item() < 1e-3
    assert rel_err(dq, rdq, 1e-2) < 2e-2 and rel_err(dk, rdk, 1e-2) < 2e-2 and rel_err(dv, rdv, 1e-2) < 2e-2


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("Sq", EDGES)
def test_dkv_pass_streamed_query_tiles(Sq, bias):
    """dK/dV pass over Sq streamed queries; Sk = 640 is above 512, so the pass is never split over query ranges."""
    _check(1, 2, Sq, 640, bias, seed=Sq)


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("Sk", EDGES)
def test_dq_pass_streamed_key_tiles(Sk, bias):
    """dQ pass over Sk streamed keys; Sq = 300 (five 64-row query ranges) keeps the dK/dV pass unsplit."""
    _check(1, 40, 300, Sk, bias, seed=Sk)
