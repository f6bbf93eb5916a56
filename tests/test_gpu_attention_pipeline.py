"""GPU: the attention kernels' software pipeline at head_dim 64 and 128: one, two and three key tiles, ragged last key
tiles (Sk mod 128 = 1, 64, 127) and ragged streamed tiles of the backward, with and without a key bias, against fp64;
outputs inside NaN-patterned buffers whose outside must survive; and run-to-run bit identity, with the dK/dV query
range split (short keys, few heads) and without it."""
import pytest
import torch

from _util import check_sentinel, rel_err, rnd, sentinel_buffer, window
from test_gpu_attention_hd128 import _key_bias, _ref64, _run

pytestmark = pytest.mark.gpu

# (B, H, Sq, Sk): Sk = 128 / 256 / 384 are 1 / 2 / 3 full key tiles; 1, 129, 320, 383 end in a ragged tile of 1, 1, 64
# and 127 keys.  H = 2 at Sq = 1000 takes the split dK/dV path for Sk <= 512; H = 40 at Sq = 300 does not.
SHAPES = [(1, 2, 1000, 128), (1, 2, 1000, 256), (2, 2, 333, 384), (1, 2, 1000, 1), (1, 2, 1000, 129),
          (1, 40, 300, 320), (2, 3, 577, 383), (1, 2, 700, 1023)]


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("B,H,Sq,Sk", SHAPES)
def test_attention_key_tiles_against_fp64(B, H, Sq, Sk, bias, d):
    torch.manual_seed(11)
    q, k, v = rnd(B, H, Sq, d), rnd(B, H, Sk, d), rnd(B, H, Sk, d)
    kb = _key_bias(B, Sk) if bias else None
    dout = rnd(B, Sq, H * d)
    out, lse, dq, dk, dv = _run(q, k, v, kb, 0.125, dout, head_dim=d)
    ro, rl, rdq, rdk, rdv = _ref64(q, k, v, kb, 0.125, dout.unflatten(2, (H, d)).transpose(1, 2))
    assert rel_err(out, ro.transpose(1, 2).flatten(2)) < 1e-2
    assert (lse.double() - rl).abs().max().item() < 1e-3
    assert rel_err(dq, rdq, 1e-2) < 2e-2 and rel_err(dk, rdk, 1e-2) < 2e-2 and rel_err(dv, rdv, 1e-2) < 2e-2


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("B,H,Sq,Sk", [(1, 2, 1000, 129), (1, 40, 300, 383), (2, 3, 577, 700)],
                         ids=["split", "nosplit", "long"])
def test_attention_outputs_stay_inside_and_repeat_bitwise(B, H, Sq, Sk, d):
    """out, lse, dq, dk and dv inside NaN-patterned buffers: nothing outside them changes, and a second launch (its
    workspace NaN-filled) gives the same bits."""
    from finetrainers_b200 import ops
    torch.manual_seed(12)
    pad = 4096
    q, k, v = rnd(B, H, Sq, d), rnd(B, H, Sk, d), rnd(B, H, Sk, d)
    kb = _key_bias(B, Sk)
    dout = rnd(B, Sq, H * d)
    runs = []
    for ws_fill in (0.0, float("nan")):
        bufs, views = {}, {}
        for name, shape, dt in (("out", (B, Sq, H * d), torch.bfloat16), ("lse", (B, H, Sq), torch.float32),
                                ("dq", (B, H, Sq, d), torch.bfloat16), ("dk", (B, H, Sk, d), torch.bfloat16),
                                ("dv", (B, H, Sk, d), torch.bfloat16)):
            n = 1
            for s in shape:
                n *= s
            bufs[name] = sentinel_buffer(n + 2 * pad, dt)
            views[name] = bufs[name][pad:pad + n].view(shape)
        ops.attn_fwd(q, k, v, kb, views["out"], views["lse"], B, H, Sq, Sk, 0.125, head_dim=d)
        ws = torch.full((ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=d),), ws_fill, device="cuda")
        ops.attn_bwd(q, k, v, kb, views["out"], dout, views["lse"], ws, views["dq"], views["dk"], views["dv"], B, H, Sq,
                     Sk, 0.125, head_dim=d)
        torch.cuda.synchronize()
        for name, buf in bufs.items():
            n = views[name].numel()
            check_sentinel(buf, [window(buf, pad, 1, n, n)], name)
            assert torch.isfinite(views[name].float()).all(), name
        runs.append(views)
    for name in runs[0]:
        x, y = runs[0][name], runs[1][name]
        it = torch.int16 if x.dtype == torch.bfloat16 else torch.int32
        assert torch.equal(x.view(it), y.view(it)), name
    ro, rl, rdq, rdk, rdv = _ref64(q, k, v, kb, 0.125, dout.unflatten(2, (H, d)).transpose(1, 2))
    v0 = runs[0]
    assert rel_err(v0["out"], ro.transpose(1, 2).flatten(2)) < 1e-2
    assert rel_err(v0["dq"], rdq, 1e-2) < 2e-2
    assert rel_err(v0["dk"], rdk, 1e-2) < 2e-2 and rel_err(v0["dv"], rdv, 1e-2) < 2e-2
