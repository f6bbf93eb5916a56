"""Host-side checks of validation sampling: the sigma schedule against an independent float64 derivation, the inference
workspace plan, the sampler step's C ABI entry point, and the input checks of ``generate_latents`` (CPU only)."""
import math
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sigmas_f64(n, seq_len, base_len=1024, max_len=4096, base_shift=0.95, max_shift=2.05, terminal=0.1):
    """Scalar float64 restatement of LTXPipeline + FlowMatchEulerDiscreteScheduler.set_timesteps (no shared code)."""
    mu = base_shift + (seq_len - base_len) * (max_shift - base_shift) / (max_len - base_len)
    out = []
    for i in range(n):
        s = 1.0 - i * (1.0 - 1.0 / n) / (n - 1) if n > 1 else 1.0
        out.append(math.exp(mu) / (math.exp(mu) + (1.0 / s - 1.0)))
    if terminal:
        last = 1.0 - out[-1]
        out = [1.0 - (1.0 - s) * (1.0 - terminal) / last for s in out]
    return out + [0.0]


def _f32_ulp(x):
    return math.ldexp(1.0, math.frexp(abs(x))[1] - 24) if x else 2.0 ** -149


@pytest.mark.parametrize("n,seq_len", [(50, 2688), (4, 72), (2, 2688), (30, 6144), (7, 1024), (50, 24 * 16 * 13)])
def test_ltx_sigmas_match_an_independent_float64_derivation(n, seq_len):
    from finetrainers_b200.sampling import ltx_sigmas
    sig = ltx_sigmas(n, seq_len)
    assert sig.dtype == torch.float32 and sig.shape == (n + 1,)
    ref = _sigmas_f64(n, seq_len)
    for got, want in zip(sig.tolist(), ref):
        # the scheduler's float32 arithmetic holds both sigma and 1 - sigma (the terminal stretch), so it rounds at the
        # scale of the larger of the two: 2 fp32 ulps there
        assert abs(got - want) <= 2 * _f32_ulp(max(want, 1.0 - want)), (got, want)
    assert sig[-1].item() == 0.0
    # the last non-zero sigma is shift_terminal to fp32 rounding; strictly decreasing
    assert abs(sig[-2].item() - 0.1) <= 2 * _f32_ulp(0.9)
    assert bool((sig[1:] < sig[:-1]).all())
    # the transformer's timesteps: fp32(sigma) * 1000 in fp32, not truncated
    t = sig[:-1] * 1000.0
    assert t.dtype == torch.float32
    assert torch.equal(t, torch.from_numpy(sig[:-1].numpy() * np.float32(1000.0)))


def test_ltx_sigmas_arguments():
    from finetrainers_b200.sampling import ltx_sigmas
    a = ltx_sigmas(8, 2688, shift_terminal=None)
    ref = _sigmas_f64(8, 2688, terminal=None)
    assert all(abs(g - w) <= 2 * _f32_ulp(max(w, 1.0 - w)) for g, w in zip(a.tolist(), ref))
    assert abs(a[0].item() - 1.0) <= _f32_ulp(1.0)
    b = ltx_sigmas(0, 2688, sigmas=[1.0, 0.75, 0.5, 0.25])  # a custom base schedule sets N
    assert b.shape == (5,)
    c = ltx_sigmas(4, 2688)
    assert torch.equal(b, c)
    with pytest.raises(ValueError, match="num_inference_steps"):
        ltx_sigmas(0, 2688)
    with pytest.raises(ValueError, match="shift_terminal"):  # one step: the stretch would divide 0 by 0
        ltx_sigmas(1, 2688)
    assert ltx_sigmas(1, 2688, shift_terminal=None).tolist() == [1.0, 0.0]


def _model(ffn=False, **cfg):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, LORA_FFN_TARGETS
    kw = dict(in_channels=32, out_channels=32, num_attention_heads=4, attention_head_dim=64, cross_attention_dim=256,
              num_layers=6, caption_channels=128)
    kw.update(cfg)
    m = B200LTXTransformer(LTXConfig(**kw), torch.bfloat16, "cpu")
    if ffn:
        m.add_adapter(64, 64, target_modules=list(LORA_FFN_TARGETS))
    else:
        m.add_adapter(64, 64)
    m.prepare()
    return m


@pytest.mark.parametrize("ffn", [False, True], ids=["attn", "ffn"])
@pytest.mark.parametrize("hd", [64, 128])
def test_inference_plan_keeps_nothing_per_block_but_the_text_side_kv(ffn, hd):
    m = _model(ffn=ffn, num_attention_heads=256 // hd, attention_head_dim=hd)
    nl = m.cfg.num_layers
    B, S, L = 2, 72, 24
    train = m.workspace_plan(B, S, L, sm_count=132)
    inf = m.workspace_plan(B, S, L, sm_count=132, inference=True)
    per_block = {k for k, (s, _) in inf.items() if len(s) > 1 and s[0] == nl}
    assert per_block == {"kv2", "k2h", "v2h", "u_kv2"}, per_block
    for k in per_block:
        assert inf[k] == train[k], k
    assert inf["h"][0] == (2, B * S, m.cfg.inner_dim)
    for k in ("ao", "lse", "ao2", "lse2"):
        assert inf[k][0][0] == 1 and inf[k][0][1:] == train[k][0][1:], k
    for k in ("n1", "qkv", "qh", "kh", "vh", "h1", "q2", "q2h", "h2", "ffpre"):
        assert inf[k][0][0] == 1 and inf[k][0][1:] == train[k][0][1:], k
    gone = {"dh", "g", "dwide", "dn", "da", "dqh", "dkh", "dvh", "dk2h", "dv2h", "delta"}
    gone |= {k for k in train if k.startswith(("dy_", "du_"))}
    assert not gone & set(inf), gone & set(inf)
    assert set(inf) <= set(train)
    assert ("splitk" in inf) == ("splitk" in train)
    # the checkpointing policy sizes only the training plans
    m.set_activation_checkpointing(range(nl))
    assert m.workspace_plan(B, S, L, sm_count=132, inference=True) == inf
    ib = m.workspace_bytes(B, S, L, sm_count=132, inference=True)
    assert ib == sum(math.prod(s) * torch.empty((), dtype=dt).element_size() for s, dt in inf.values())
    assert ib < m.workspace_bytes(B, S, L, sm_count=132) / 2


def test_kept_rows_of_the_three_plans():
    from finetrainers_b200.model import B200LTXTransformer
    assert [B200LTXTransformer._kept_rows(l) for l in range(3)] == [(0, 1, 0), (1, 2, 1), (2, 3, 2)]
    assert [B200LTXTransformer._kept_rows(l, True) for l in range(3)] == [(0, 1, 0), (1, 0, 0), (0, 1, 0)]


def test_cfg_euler_step_entry_point_is_declared_bound_and_wrapped():
    from finetrainers_b200 import lib, ops
    hdr = open(os.path.join(ROOT, "include", "b2d.h")).read()
    assert re.search(r"int b2d_cfg_euler_step\(const void\* pred, float\* latents, void\* x_next, int32_t B, int64_t n,"
                     r"\s*int32_t guided,\s*float guidance, const float\* dt, void\* stream\);", hdr)
    assert "b2d_cfg_euler_step" in lib.EXPORTS
    assert callable(ops.cfg_euler_step)
    src = open(os.path.join(ROOT, "finetrainers_b200", "csrc", "b2d_elem.cu")).read()
    assert "launch_k(cfg_euler_step_kernel<true>" in src and "launch_k(cfg_euler_step_kernel<false>" in src
    x = torch.zeros(2, 8)
    with pytest.raises(lib.B2DError):  # no CPU fallback
        ops.cfg_euler_step(x.bfloat16(), x[:1], x.bfloat16(), 1, 8, True, 3.0, torch.zeros(1))


class _NoLaunch(torch.nn.Module):
    """A transformer stand-in whose forward must never run: the checks come first."""

    def __init__(self):
        super().__init__()
        from finetrainers_b200.model import LTXConfig
        self.cfg = LTXConfig(in_channels=32)
        self.proj_in = torch.nn.Linear(1, 1)

    def forward(self, *a, **k):
        raise AssertionError("forward ran before the input checks")


def test_generate_latents_rejects_bad_input_before_launching():
    from finetrainers_b200.specification import LTXVideoModelSpecification
    spec = LTXVideoModelSpecification()
    tr = _NoLaunch()
    pe, pm = torch.zeros(1, 16, 4096), torch.ones(1, 16)
    ne, nm = torch.zeros(1, 16, 4096), torch.ones(1, 16)
    ok = dict(num_frames=9, height=64, width=96)
    with pytest.raises(ValueError, match="num_inference_steps"):
        spec.generate_latents(tr, pe, pm, ne, nm, num_inference_steps=0, **ok)
    with pytest.raises(ValueError, match="negative_prompt_embeds"):
        spec.generate_latents(tr, pe, pm, **ok)
    with pytest.raises(ValueError, match="negative_prompt_embeds"):
        spec.generate_latents(tr, pe, pm, ne, None, **ok)
    with pytest.raises(ValueError, match="share L"):
        spec.generate_latents(tr, pe, pm, torch.zeros(1, 12, 4096), torch.ones(1, 12), **ok)
    with pytest.raises(ValueError, match="share L"):
        spec.generate_latents(tr, pe, pm, ne, torch.ones(1, 12), **ok)
    for bad in (dict(num_frames=10, height=64, width=96), dict(num_frames=9, height=48, width=96),
                dict(num_frames=9, height=64, width=100), dict(num_frames=9, height=0, width=96)):
        with pytest.raises(ValueError, match="multiple"):
            spec.generate_latents(tr, pe, pm, ne, nm, **bad)
    with pytest.raises(ValueError, match="latents must be packed"):
        spec.generate_latents(tr, pe, pm, ne, nm, latents=torch.zeros(1, 5, 32), **ok)
