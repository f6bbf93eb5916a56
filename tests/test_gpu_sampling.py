"""GPU: validation sampling.  The guided Euler step kernel bit for bit against the pipeline's torch op sequence, the
inference forward bit for bit against the training forward, training unaffected by a sample between steps, the
pending-backward guard, the sampler against a plain-torch fp32 restatement of the pipeline loop on the oracle, graph
replay equal to eager steps, and a 13B sample between training steps."""
import gc
import random

import pytest
import torch

from _util import SMALL, build_pair, check_sentinel, rel_err, sentinel_buffer, window

pytestmark = pytest.mark.gpu

SMALL128 = dict(SMALL, num_attention_heads=2, attention_head_dim=128)
CLI_SKIP = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]


# ---- the step kernel -------------------------------------------------------------------------------------------------
def _torch_step(pred, x, g, dt):
    """LTXPipeline's guidance + FlowMatchEulerDiscreteScheduler.step + the next step's input, as torch ops on the GPU."""
    noise_pred = pred.float()
    if g > 1.0:
        u, c = noise_pred.chunk(2)
        noise_pred = u + g * (c - u)
    x_new = x + dt * noise_pred          # sample + (sigma_next - sigma) * model_output; dt a 0-dim fp32 tensor
    rows = pred.shape[0] // x.shape[0]
    return x_new, torch.cat([x_new] * rows).to(torch.bfloat16)


def _same(got, want, what):
    """Equal bits, except that a NaN only has to be a NaN (torch and the CUDA intrinsics pick different NaN codes)."""
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), f"{what}: NaN positions differ"
    ints = {torch.float32: torch.int32, torch.bfloat16: torch.int16}[want.dtype]
    assert torch.equal(got.view(ints)[~nan], want.view(ints)[~nan]), f"{what}: bits differ"


@pytest.mark.parametrize("B", [1, 2])
# 1 + 2^-30: guided (the pipeline decides g > 1 in double precision) with g rounded to 1.0f in the arithmetic
@pytest.mark.parametrize("g", [3.0, 4.7, 1.0 + 2 ** -30, 1.0], ids=["cfg3", "cfg4.7", "cfg_g1", "nocfg"])
@pytest.mark.parametrize("n", [2688 * 128, 1003, 5], ids=["n2688x128", "ragged1003", "tiny5"])
@pytest.mark.parametrize("dt", [-0.0213, 0.37])
def test_cfg_euler_step_is_the_torch_op_sequence(B, g, n, dt):
    from finetrainers_b200 import ops
    torch.manual_seed(B * 1000 + n)
    rows = 2 * B if g > 1 else B
    pred = (torch.randn(rows, n, device="cuda") * 2).bfloat16()
    x0 = torch.randn(B, n, device="cuda")
    if n > 64:  # special values propagate as in the torch ops
        pred[0, 3] = float("nan")
        pred[rows - 1, 7] = float("inf")
        pred[0, 11] = float("-inf")
        x0[0, 13] = float("nan")
        x0[B - 1, 17] = float("inf")
    dt_t = torch.tensor(dt, dtype=torch.float32, device="cuda")
    want_x, want_next = _torch_step(pred, x0, g, dt_t)
    # outputs inside sentinel-filled buffers, 16-byte aligned windows
    off = 16
    xbuf = sentinel_buffer(off + B * n + 64, torch.float32)
    nbuf = sentinel_buffer(off + rows * n + 64, torch.bfloat16)
    xw, nw = window(xbuf, off, B, n, n), window(nbuf, off, rows, n, n)
    xw.copy_(x0)
    ops.cfg_euler_step(pred, xw, nw, B, n, g > 1.0, g, dt_t.reshape(1))
    torch.cuda.synchronize()
    _same(xw, want_x, "latents")
    _same(nw, want_next, "x_next")
    check_sentinel(xbuf, [xw], "latents buffer")
    check_sentinel(nbuf, [nw], "x_next buffer")


# ---- models ----------------------------------------------------------------------------------------------------------
def _model(cfgk, ffn=False, layerwise=False, ckpt=False, seed=0, std=0.05):
    from finetrainers_b200.model import (B200LTXTransformer, LTXConfig, LORA_FFN_TARGETS,
                                         apply_activation_checkpointing)
    torch.manual_seed(seed)
    m = B200LTXTransformer(LTXConfig(**cfgk), torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "scale_shift_table" in n:
                p.normal_(0, 1.0 / p.shape[-1] ** 0.5)
            elif "norm_q" in n or "norm_k" in n:
                p.fill_(1.0)
            else:
                p.normal_(0, std)
    if layerwise:
        m.enable_layerwise_casting(torch.float8_e4m3fn, torch.bfloat16, CLI_SKIP)
    m.add_adapter(64, 64, target_modules=list(LORA_FFN_TARGETS) if ffn else None)
    if ckpt:
        apply_activation_checkpointing(m, "full")
    m.prepare()
    with torch.no_grad():
        m.lora_flat.normal_(0, 0.02)  # non-zero B: every adapter contributes
    return m


def _inputs(m, B, F, H, W, L, seed=3):
    g = torch.Generator().manual_seed(seed)
    cfg = m.cfg
    x = torch.randn(B, F * H * W, cfg.in_channels, generator=g).bfloat16().cuda()
    ehs = torch.randn(B, L, cfg.caption_channels, generator=g).bfloat16().cuda()
    mask = torch.ones(B, L)
    mask[0, 1:] = 0                  # one valid key
    mask[B - 1, L // 2:] = 0
    t = torch.tensor([437.25, 912.625][:B])  # not integers: the pipeline's sigma * 1000
    return dict(hidden_states=x, encoder_hidden_states=ehs, timestep=t.cuda(), encoder_attention_mask=mask.cuda(),
                num_frames=F, height=H, width=W, rope_interpolation_scale=[8 / 25, 32, 32])


INFER_CASES = {
    "full_width": (dict(num_layers=2), {}, (7, 16, 24, 128)),
    "fp8": (dict(SMALL, num_layers=3), dict(layerwise=True), (2, 4, 9, 24)),
    "ckpt_full": (dict(SMALL, num_layers=3), dict(ckpt=True), (2, 4, 9, 24)),
    "ffn": (dict(SMALL, num_layers=3), dict(ffn=True), (2, 4, 9, 24)),
    "hd128": (dict(SMALL128, num_layers=3), {}, (2, 4, 9, 24)),
}


@pytest.mark.timeout(600)
@pytest.mark.parametrize("case", list(INFER_CASES))
def test_inference_forward_is_the_training_forward(case):
    """B = 2 with two masks (one with a single valid key) and non-integer timesteps: the no-grad forward (inference plan)
    gives the training forward's bits, adds no training workspace, and grows the peak by at most its own workspace."""
    cfgk, kw, (F, H, W, L) = INFER_CASES[case]
    m = _model(cfgk, **kw)
    args = _inputs(m, 2, F, H, W, L)
    out = m(**args)[0]                       # autograd forward: the training plan
    assert out.requires_grad
    want = out.detach().clone()
    keys = set(m._ws)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        got = m(**args)[0].clone()
    torch.cuda.synchronize()
    grow = torch.cuda.max_memory_allocated() - base
    assert torch.equal(got, want)
    assert set(m._ws) == keys
    S = F * H * W
    iws = m.workspace_bytes(2, S, L, inference=True)
    assert m._iws is not None and m._iws[0] == (2, S, L)
    assert grow <= iws + 64 * 2 ** 20, (grow, iws)
    with torch.no_grad():                     # again, into the same inference workspace
        again = m(**args)[0]
    assert torch.equal(again, want)
    print(f"\n{case}: inference workspace {iws / 1e6:.1f} MB (training {m.workspace_bytes(2, S, L) / 1e6:.1f} MB), "
          f"peak growth {grow / 1e6:.1f} MB")


def _sinusoid64(t):
    """[cos | sin](t f_i), f_i = exp(-ln(1e4) i / 128), in float64 (diffusers Timesteps(256, flip_sin_to_cos=True))."""
    f = torch.exp(-torch.log(torch.tensor(1e4, dtype=torch.float64)) * torch.arange(128, dtype=torch.float64) / 128)
    a = t.double()[:, None] * f[None]
    return torch.cat([a.cos(), a.sin()], 1)


def test_non_integer_timestep_reaches_the_embedding():
    """The pipeline's timesteps are fp32 sigma * 1000, not integers: both plans embed them unrounded."""
    m = _model(dict(SMALL, num_layers=2))
    args = _inputs(m, 2, 2, 4, 9, 24)
    t = args["timestep"]
    assert not torch.equal(t, t.floor())
    ref, ref_floor = _sinusoid64(t.cpu()), _sinusoid64(t.floor().cpu())
    assert (ref - ref_floor).abs().max() > 0.1
    out = m(**args)[0]                        # training plan
    with torch.no_grad():
        got = m(**args)[0].clone()            # inference plan
    # bf16 rounding of values in [-1, 1] plus the fp32 argument t * f: far below the 0.1 a truncated t would give
    for tsin in (m._ws[(2, 72, 24)]["tsin"], m._iws[1]["tsin"]):
        assert (tsin.double().cpu() - ref).abs().max() < 4e-3
    with torch.no_grad():
        at_floor = m(**dict(args, timestep=t.floor()))[0].clone()
    assert not torch.equal(got, at_floor)
    assert torch.equal(got, out.detach())


def test_inference_workspace_is_replaced_at_another_shape():
    m = _model(dict(SMALL, num_layers=2))
    with torch.no_grad():
        m(**_inputs(m, 2, 2, 4, 9, 24))
        first = m._iws[1]["h"]
        m(**_inputs(m, 1, 2, 4, 8, 16))
    assert m._iws[0] == (1, 64, 16) and m._iws[1]["h"] is not first
    assert not m._ws


def test_no_grad_forward_between_forward_and_backward_raises():
    m = _model(dict(SMALL, num_layers=2))
    args = _inputs(m, 2, 2, 4, 9, 24)
    out = m(**args)[0]
    with torch.no_grad():
        m(**args)
    with pytest.raises(RuntimeError, match="ONE set of saved activations"):
        out.backward(torch.ones_like(out))


# ---- training around a sample ----------------------------------------------------------------------------------------
def _prompts(m, B, L, seed=9):
    g = torch.Generator().manual_seed(seed)
    pe = torch.randn(B, L, m.cfg.caption_channels, generator=g).bfloat16().cuda()
    ne = torch.randn(B, L, m.cfg.caption_channels, generator=g).bfloat16().cuda()
    pm = torch.ones(B, L, device="cuda")
    pm[0, L // 3:] = 0
    nm = torch.ones(B, L, device="cuda")
    nm[B - 1, 1:] = 0
    return pe, pm, ne, nm


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("layerwise", [False, True], ids=["resident", "fp8"])
def test_sample_between_training_steps_changes_nothing(graph, layerwise):
    from finetrainers_b200.specification import LTXVideoModelSpecification
    from finetrainers_b200.trainer import SFTTrainStep

    def run(with_sample):
        random.seed(0)
        m = _model(dict(SMALL, num_layers=3), layerwise=layerwise)
        st = SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=graph)
        st.spec.first_frame_conditioning_p = 0.0
        g = torch.Generator().manual_seed(77)
        out = []
        for i in range(3):
            lat = torch.randn(2, 32, 2, 4, 9, generator=g).bfloat16().cuda()
            ehs = torch.randn(2, 24, 128, generator=g).bfloat16().cuda()
            mask = (torch.arange(24)[None] < torch.tensor([[24], [7]])).float().cuda()
            st.micro_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                          {"latents": lat, "latents_mean": torch.zeros(2, 32, device="cuda"),
                           "latents_std": torch.ones(2, 32, device="cuda")})
            torch.cuda.synchronize()
            loss, grad = st.loss_buf.clone(), m.lora_grad_flat.clone()
            st.optimizer_step()
            out.append((loss, grad, m.lora_flat.clone()))
            if with_sample and i == 0:
                spec = LTXVideoModelSpecification(m.cfg)
                pe, pm, ne, nm = _prompts(m, 1, 16)
                lat_s = spec.generate_latents(m, pe, pm, ne, nm, num_frames=9, height=96, width=256,
                                              num_inference_steps=3, generator=torch.Generator().manual_seed(1))
                assert torch.isfinite(lat_s).all()
        return out

    a, b = run(False), run(True)
    for i, (x, y) in enumerate(zip(a, b)):
        for what, u, v in zip(("loss", "lora_grad_flat", "lora_flat"), x, y):
            assert torch.equal(u, v), (i, what)


# ---- the sampler -----------------------------------------------------------------------------------------------------
def _oracle_sample(om, pe, pm, ne, nm, lat, sig, F, H, W, g, rope):
    """Plain-torch fp32 restatement of LTXPipeline.__call__'s denoising loop (CPU): cat([negative, positive]),
    cat([latents] * 2) cast to the embeddings' dtype (bf16), guidance on noise_pred.float(), scheduler.step.
    -> (final latents, the first step's guided velocity)."""
    ehs, mask = torch.cat([ne, pe]).float(), torch.cat([nm, pm]).float()
    x, v0 = lat.clone(), None
    for i in range(sig.numel() - 1):
        inp = torch.cat([x] * 2).to(torch.bfloat16).float()
        t = (sig[i] * 1000.0).expand(inp.shape[0])
        pred = om(inp, ehs, t, mask, F, H, W, rope)[0].float()
        u, c = pred.chunk(2)
        v = u + g * (c - u)
        v0 = v if v0 is None else v0
        x = x + (sig[i + 1] - sig[i]) * v
    return x, v0


@pytest.mark.timeout(600)
def test_sampler_matches_the_oracle_pipeline_loop():
    """SMALL, 4 steps, guidance 3, B = 2.  Measured on an H100 80GB HBM3: final latents rel_err 3.0e-3, first guided
    velocity rel_err 1.6e-2 (guidance triples the difference of the two predictions, and with it their rounding)."""
    from finetrainers_b200.sampling import ltx_sigmas
    from finetrainers_b200.specification import LTXVideoModelSpecification
    O, om, bm = build_pair(SMALL, 64)
    spec = LTXVideoModelSpecification(bm.cfg)
    pe, pm, ne, nm = _prompts(bm, 2, 24)
    F, H, W = 2, 4, 9
    lat0 = torch.randn(2, F * H * W, 32, generator=torch.Generator().manual_seed(4))
    got = spec.generate_latents(bm, pe, pm, ne, nm, num_frames=9, height=128, width=288, num_inference_steps=4,
                                guidance_scale=3.0, latents=lat0)
    sig = ltx_sigmas(4, F * H * W)
    rope = (8 / 25, 32, 32)
    with torch.no_grad():
        want, v0 = _oracle_sample(om, pe.cpu(), pm.cpu(), ne.cpu(), nm.cpu(), lat0, sig, F, H, W, 3.0, rope)
        pred = bm(torch.cat([lat0] * 2).bfloat16().cuda(), torch.cat([ne, pe]), (sig[0] * 1000).expand(4).cuda(),
                  torch.cat([nm, pm]), F, H, W, rope)[0].float().cpu()
    u, c = pred.chunk(2)
    e_v, e_x = rel_err(u + 3.0 * (c - u), v0), rel_err(got.cpu(), want)
    print(f"\nsampler vs oracle: first velocity rel_err {e_v:.2e}, final latents rel_err {e_x:.2e}")
    assert e_v < 3e-2
    assert e_x < 2e-2


@pytest.mark.parametrize("g", [3.0, 1.0 + 2 ** -30, 1.0], ids=["cfg", "cfg_g1", "nocfg"])
@pytest.mark.parametrize("case", ["resident", "fp8", "hd128"])
def test_graph_replay_equals_eager_steps(g, case):
    from finetrainers_b200.specification import LTXVideoModelSpecification
    cfgk = dict(SMALL128 if case == "hd128" else SMALL, num_layers=3)
    m = _model(cfgk, layerwise=case == "fp8")
    spec = LTXVideoModelSpecification(m.cfg)
    pe, pm, ne, nm = _prompts(m, 2, 24)
    kw = dict(num_frames=9, height=128, width=288, num_inference_steps=6, guidance_scale=g)
    a = spec.generate_latents(m, pe, pm, ne, nm, generator=torch.Generator().manual_seed(2), cuda_graph=True, **kw)
    b = spec.generate_latents(m, pe, pm, ne, nm, generator=torch.Generator().manual_seed(2), cuda_graph=False, **kw)
    assert a.shape == (2, 72, 32) and a.dtype == torch.float32
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)


@pytest.mark.timeout(1800)
def test_13b_sample_between_graph_training_steps():
    """The 13B geometry (48 blocks, r = 64): 3 training steps with CUDA graphs (the third a replay), a 3-step guided
    sample at 2688 tokens, one more training step.  Peak below 70 GB; every training step bit-identical to the same run
    without the sample."""
    from finetrainers_b200.model import LTXConfig
    from finetrainers_b200.specification import LTXVideoModelSpecification
    from finetrainers_b200.trainer import SFTTrainStep
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 70e9:
        pytest.skip(f"needs 70 GB of free device memory, {free / 1e9:.1f} GB are free")
    cfgk = LTXConfig.ltx_13b().to_dict()

    def run(with_sample):
        random.seed(0)
        m = _model(cfgk, std=0.02)
        st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)
        g = torch.Generator().manual_seed(1234)
        lat = torch.randn(1, 128, 7, 16, 24, generator=g).bfloat16().cuda()
        ehs = (torch.randn(1, 128, 4096, generator=g) * 0.1).bfloat16().cuda()
        mask = (torch.arange(128)[None] < 100).cuda()
        mean, std = torch.zeros(1, 128, device="cuda"), torch.ones(1, 128, device="cuda")
        out = []
        for i in range(4):
            if with_sample and i == 3:
                pe, pm, ne, nm = _prompts(m, 1, 128)
                s = LTXVideoModelSpecification(m.cfg).generate_latents(
                    m, pe, pm, ne, nm, num_frames=49, height=512, width=768, num_inference_steps=3,
                    generator=torch.Generator().manual_seed(1))
                assert s.shape == (1, 2688, 128) and torch.isfinite(s).all()
            st.train_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                          {"latents": lat, "latents_mean": mean, "latents_std": std})
            torch.cuda.synchronize()
            out.append((st.metrics[1].item(), st.metrics[0].item()))
        return out, m.lora_flat.clone()

    torch.cuda.reset_peak_memory_stats()
    m1, p1 = run(True)
    peak = torch.cuda.max_memory_allocated()
    gc.collect()
    torch.cuda.empty_cache()
    m0, p0 = run(False)
    print(f"\n13B: (loss, grad norm) per step {m1}; max_memory_allocated with the sample {peak / 1e9:.2f} GB")
    assert peak < 70e9
    assert m0 == m1
    assert torch.equal(p0, p1)
