"""GPU: image-to-video.  The per-frame timestep plan against the oracle and bit for bit against the per-sample plan, its
training / inference / checkpointed / block-range backward consistency, input errors, the conditioned Euler step kernel
bit for bit against the pipeline's torch op sequence, the I2V sampler against a plain-torch fp32 restatement of
LTXImageToVideoPipeline's loop on the oracle, graph replay, training around a sample, and a 13B sample."""
import gc
import random

import pytest
import torch

from _util import SMALL, build_pair, check_sentinel, rel_err, sentinel_buffer, window

pytestmark = pytest.mark.gpu

SMALL128 = dict(SMALL, num_attention_heads=2, attention_head_dim=128)
CLI_SKIP = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]
ROPE = (8 / 25, 32.0, 32.0)


def _model(cfgk, ffn=False, layerwise=False, ckpt=None, seed=0, std=0.05):
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
        apply_activation_checkpointing(m, *ckpt)
    m.prepare()
    with torch.no_grad():
        m.lora_flat.normal_(0, 0.02)  # non-zero B: every adapter contributes
    return m


def _inputs(cfg, B, F, H, W, L, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, F * H * W, cfg.in_channels, generator=g).bfloat16()
    ehs = torch.randn(B, L, cfg.caption_channels, generator=g).bfloat16()
    mask = torch.ones(B, L)
    mask[0, 1:] = 0                  # one valid key
    mask[B - 1, L // 2:] = 0
    dpred = torch.randn(B, F * H * W, cfg.out_channels, generator=g).bfloat16()
    return x, ehs, mask, dpred


# per-frame timesteps: frame 0 is the conditioning frame (t = 0), the others distinct and not integers
FRAME_T = torch.tensor([[0.0, 437.25, 912.625], [0.0, 101.5, 655.875]])


def _tokens(tf, HW):
    """[B, F] per-frame values -> the [B, F HW] per-token timesteps (frame-major tokens)."""
    return tf.repeat_interleave(HW, 1).contiguous()


def _public(m, x, ehs, mask, t, F, H, W, dpred=None):
    """Public forward (+ backward when dpred is given) -> (pred, flat LoRA gradient or None)."""
    if dpred is not None:
        m.lora_grad_flat.zero_()
    out = m(hidden_states=x.cuda(), encoder_hidden_states=ehs.cuda(), timestep=t.cuda(),
            encoder_attention_mask=mask.cuda(), num_frames=F, height=H, width=W, rope_interpolation_scale=ROPE)[0]
    if dpred is None:
        return out.detach().clone(), None
    out.backward(dpred.cuda())
    torch.cuda.synchronize()
    return out.detach().clone(), m.lora_grad_flat.clone()


def _per_frame(m, x, ehs, mask, tvals, F, H, W, dpred):
    """The per-frame plan on [B F] timesteps through the model's forward and backward -> (pred, flat LoRA gradient)."""
    m.lora_grad_flat.zero_()
    key_bias = ((1.0 - mask.cuda().float()) * -10000.0).contiguous()
    pred = m._forward_impl(x.cuda(), ehs.cuda(), tvals.cuda().float().contiguous(), key_bias, F, H, W, ROPE).clone()
    m._backward_impl(dpred.cuda())
    torch.cuda.synchronize()
    return pred, m.lora_grad_flat.clone()


# ---- the model -------------------------------------------------------------------------------------------------------
def test_per_frame_forward_backward_matches_oracle():
    """B = 2, F = 3, frame 0 at t = 0: pred and every LoRA gradient against the oracle fed the same per-token timesteps,
    within test_gpu_model's bounds (a forward that embeds frame 0's t = 0 for every token is far outside them)."""
    O, om, bm = build_pair(SMALL, 64)
    B, F, H, W, L = 2, 3, 4, 9, 24
    x, ehs, mask, dpred = _inputs(bm.cfg, B, F, H, W, L)
    t = _tokens(FRAME_T, H * W)
    pred, _ = _public(bm, x, ehs, mask, t, F, H, W, dpred)
    pred_o = om(x.float(), ehs.float(), t, mask.float(), F, H, W, ROPE)[0]
    (pred_o * dpred.float()).sum().backward()
    e_pred = rel_err(pred.cpu(), pred_o.detach())
    assert e_pred < 3e-2
    og = dict(om.named_parameters())
    gmax = max(p.grad.abs().max().item() for n, p in om.named_parameters() if "lora_" in n)
    errs = {}
    for n, p in bm.named_parameters():
        if "lora_" in n:
            go = og[n].grad
            assert go.abs().max().item() > gmax / 300, n   # nothing is rounding noise
            errs[n] = (p.grad.float().cpu() - go).abs().max().item() / go.abs().max().item()
    assert len(errs) == 2 * 8 * SMALL["num_layers"]
    assert max(errs.values()) < 5e-2, max(errs.items(), key=lambda kv: kv[1])
    # the per-sample embedding of frame 0's timestep is not what the oracle computes
    with torch.no_grad():
        frame0, _ = _public(bm, x, ehs, mask, FRAME_T[:, 0].contiguous(), F, H, W)
    assert rel_err(frame0.cpu(), pred_o.detach()) > 3e-2
    print(f"\nper-frame vs oracle: pred rel_err {e_pred:.2e}, worst LoRA grad {max(errs.values()):.2e}")


PLANS = {"keep_all": ({}, {}), "full": ({}, dict(ckpt=("full",))), "block_skip": ({}, dict(ckpt=("block_skip", 2))),
         "fp8": ({}, dict(layerwise=True)), "ffn": ({}, dict(ffn=True)),
         "hd128": (dict(num_attention_heads=2, attention_head_dim=128), {})}


@pytest.mark.parametrize("hw", [(4, 9), (16, 24)], ids=["hw36", "hw384"])
@pytest.mark.parametrize("plan", list(PLANS))
def test_per_sample_values_in_the_per_frame_plan_are_the_per_sample_plan(plan, hw):
    """One timestep per sample, repeated per frame, through the per-frame plan: pred and the LoRA gradients equal the
    1-D [B] call's bits, at H W = 36 (cooperative gate epilogue) and 384 (ping-pong), and the per-token [B, S, 1] call
    (constant per sample) takes the per-sample plan."""
    base, kw = PLANS[plan]
    m = _model(dict(SMALL, **base, num_layers=3), **kw)
    B, F, (H, W), L = 2, 3, hw, 24
    x, ehs, mask, dpred = _inputs(m.cfg, B, F, H, W, L)
    t = torch.tensor([437.25, 912.625])
    want, gwant = _public(m, x, ehs, mask, t, F, H, W, dpred)
    assert gwant.abs().max().item() > 0
    got, ggot = _per_frame(m, x, ehs, mask, t.repeat_interleave(F), F, H, W, dpred)
    assert B * F in m._tws
    assert torch.equal(got, want)
    assert torch.equal(ggot, gwant)
    tok, gtok = _public(m, x, ehs, mask, t.view(B, 1, 1).expand(B, F * H * W, 1), F, H, W, dpred)
    assert torch.equal(tok, want) and torch.equal(gtok, gwant)


def test_public_forward_under_capture_takes_the_per_frame_plan():
    """Under CUDA-graph capture nothing is read back: per-token timesteps run the per-frame plan, whose replay gives the
    per-sample call's bits for per-sample values and the eager per-frame call's bits for per-frame values."""
    m = _model(dict(SMALL, num_layers=3))
    B, F, H, W, L = 2, 3, 4, 9, 24
    x, ehs, mask = (v.cuda() for v in _inputs(m.cfg, B, F, H, W, L)[:3])  # no host copies inside the capture
    t = torch.tensor([437.25, 912.625])
    t_buf = _tokens(t.view(B, 1).expand(B, F), H * W).cuda()
    with torch.no_grad():
        want, _ = _public(m, x, ehs, mask, t, F, H, W)
        frames, _ = _public(m, x, ehs, mask, _tokens(FRAME_T, H * W), F, H, W)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m(hidden_states=x, encoder_hidden_states=ehs, timestep=t_buf,
                    encoder_attention_mask=mask, num_frames=F, height=H, width=W,
                    rope_interpolation_scale=ROPE)[0]
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want)
        t_buf.copy_(_tokens(FRAME_T, H * W))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, frames)
        assert not torch.equal(frames, want)
    del graph


def test_per_frame_plans_agree():
    """Per-frame timesteps that differ by frame: the inference plan gives the training plan's pred; checkpointing
    ("full", "block_skip") gives keep-all's pred and gradients; the DDP segments' block-range backward gives the whole
    backward's gradients, range by range."""
    B, F, H, W, L = 2, 3, 4, 9, 24
    from finetrainers_b200.model import LTXConfig
    cfgk = dict(SMALL, num_layers=4)
    x, ehs, mask, dpred = _inputs(LTXConfig(**cfgk), B, F, H, W, L)
    t = _tokens(FRAME_T, H * W)
    ref = None
    for ckpt in (None, ("full",), ("block_skip", 3)):
        m = _model(cfgk, ffn=True, ckpt=ckpt)
        pred, grad = _public(m, x, ehs, mask, t, F, H, W, dpred)
        with torch.no_grad():
            inf, _ = _public(m, x, ehs, mask, t, F, H, W)
        assert torch.equal(inf, pred), ckpt
        if ref is None:
            ref = (pred, grad)
            assert grad.abs().max().item() > 0
        assert torch.equal(pred, ref[0]) and torch.equal(grad, ref[1]), ckpt
        # block ranges, top first, each range's slice final when its tail returns
        m.lora_grad_flat.zero_()
        key_bias = ((1.0 - mask.cuda().float()) * -10000.0).contiguous()
        m._forward_impl(x.cuda(), ehs.cuda(), FRAME_T.reshape(-1).cuda(), key_bias, F, H, W, ROPE)
        m._backward_head(dpred.cuda())
        pb = m._per_blk
        for lo, hi in [(2, 4), (0, 2)]:
            m._backward_blocks(hi - 1, lo)
            m._backward_tail(lo, hi)
            torch.cuda.synchronize()
            assert torch.equal(m.lora_grad_flat[lo * pb:hi * pb], grad[lo * pb:hi * pb]), (ckpt, lo, hi)
        m._schedule.end_backward()


def test_bad_timesteps_raise_before_any_launch():
    from finetrainers_b200 import ops
    m = _model(dict(SMALL, num_layers=2))
    B, F, H, W, L = 2, 3, 4, 9, 24
    x, ehs, mask, _ = _inputs(m.cfg, B, F, H, W, L)
    t = _tokens(FRAME_T, H * W)
    t[1, 2 * H * W + 5] += 0.5                 # sample 1, frame 2: one token differs
    n0 = ops.LAUNCH_COUNT
    for grad in (True, False):
        with torch.set_grad_enabled(grad):
            with pytest.raises(ValueError, match="frame 2 of sample 1"):
                _public(m, x, ehs, mask, t, F, H, W)
            for bad in (torch.zeros(B, F), torch.zeros(B * F * H * W - 1), torch.zeros(B + 1)):
                with pytest.raises(ValueError, match="elements"):
                    _public(m, x, ehs, mask, bad, F, H, W)
    torch.cuda.synchronize()
    assert ops.LAUNCH_COUNT == n0


# ---- the conditioned step kernel -------------------------------------------------------------------------------------
def _torch_cond_step(pred, x, n_cond, g, dt):
    """LTXImageToVideoPipeline after the transformer: guidance on noise_pred.float(), scheduler.step on the frames after
    the first, torch.cat with the first frame, the next step's input, as torch ops on the GPU."""
    noise_pred = pred.float()
    if g > 1.0:
        u, c = noise_pred.chunk(2)
        noise_pred = u + g * (c - u)
    pred_latents = x[:, n_cond:] + dt * noise_pred[:, n_cond:]
    x_new = torch.cat([x[:, :n_cond], pred_latents], 1)
    rows = pred.shape[0] // x.shape[0]
    return x_new, torch.cat([x_new] * rows).to(torch.bfloat16)


def _same(got, want, what):
    """Equal bits, except that a NaN only has to be a NaN (torch and the CUDA intrinsics pick different NaN codes)."""
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), f"{what}: NaN positions differ"
    ints = {torch.float32: torch.int32, torch.bfloat16: torch.int16}[want.dtype]
    assert torch.equal(got.view(ints)[~nan], want.view(ints)[~nan]), f"{what}: bits differ"


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("g", [3.0, 1.0 + 2 ** -30, 1.0], ids=["cfg3", "cfg_g1", "nocfg"])
@pytest.mark.parametrize("n,n_cond", [(2688 * 128, 384 * 128), (2688 * 128, 49151), (2688 * 128, 0), (1003, 328),
                                      (1003, 335), (2304, 1), (64, 63)],
                         ids=["vec_a8", "vec_odd", "vec_0", "ragged_a8", "ragged_odd", "short_head", "last_one"])
def test_cfg_euler_step_cond_is_the_pipeline_op_sequence(B, g, n, n_cond):
    from finetrainers_b200 import ops
    torch.manual_seed(B * 1000 + n + n_cond)
    rows = 2 * B if g > 1 else B
    dt = torch.tensor(-0.0213, dtype=torch.float32, device="cuda")
    pred = (torch.randn(rows, n, device="cuda") * 2).bfloat16()
    x0 = torch.randn(B, n, device="cuda")
    if n - n_cond > 64:  # special values propagate as in the torch ops
        pred[0, n_cond + 3] = float("nan")
        pred[rows - 1, n_cond + 7] = float("inf")
        x0[B - 1, n_cond + 13] = float("nan")
    want_x, want_next = _torch_cond_step(pred, x0, n_cond, g, dt)
    off = 16
    xbuf = sentinel_buffer(off + B * n + 64, torch.float32)
    nbuf = sentinel_buffer(off + rows * n + 64, torch.bfloat16)
    xw, nw = window(xbuf, off, B, n, n), window(nbuf, off, rows, n, n)
    xw[:, n_cond:] = x0[:, n_cond:]             # the frozen elements hold the sentinel: they must not be written
    ops.cfg_euler_step_cond(pred, xw, nw, B, n, n_cond, g > 1.0, g, dt.reshape(1))
    torch.cuda.synchronize()
    _same(xw[:, n_cond:], want_x[:, n_cond:], "latents")
    _same(nw[:, n_cond:], want_next[:, n_cond:], "x_next")
    check_sentinel(xbuf, [xw[:, n_cond:]], "latents buffer")
    check_sentinel(nbuf, [nw[:, n_cond:]], "x_next buffer")
    if n_cond == 0:                             # nothing frozen: the unconditioned step's bits
        xo, no = x0.clone(), torch.empty_like(nw)
        ops.cfg_euler_step(pred, xo, no, B, n, g > 1.0, g, dt.reshape(1))
        torch.cuda.synchronize()
        _same(xw, xo, "latents vs cfg_euler_step")
        _same(nw, no, "x_next vs cfg_euler_step")


def test_cfg_euler_step_cond_rejects_bad_arguments():
    from finetrainers_b200 import lib, ops
    x = torch.zeros(2, 64, device="cuda")
    p, nx, dt = x.bfloat16(), x.bfloat16(), torch.zeros(1, device="cuda")
    for n_cond in (-1, 64, 65):
        with pytest.raises(lib.B2DError, match="n_cond"):
            ops.cfg_euler_step_cond(p, x[:1], nx, 1, 64, n_cond, True, 3.0, dt)
    with pytest.raises(lib.B2DError, match="aligned"):
        ops.cfg_euler_step_cond(p, x.view(-1)[1:65], nx, 1, 64, 8, True, 3.0, dt)
    with pytest.raises(lib.B2DError, match="positive"):
        ops.cfg_euler_step_cond(p, x[:1], nx, 0, 64, 8, True, 3.0, dt)


# ---- the sampler -----------------------------------------------------------------------------------------------------
def _prompts(m, B, L, seed=9):
    g = torch.Generator().manual_seed(seed)
    pe = torch.randn(B, L, m.cfg.caption_channels, generator=g).bfloat16().cuda()
    ne = torch.randn(B, L, m.cfg.caption_channels, generator=g).bfloat16().cuda()
    pm = torch.ones(B, L, device="cuda")
    pm[0, L // 3:] = 0
    nm = torch.ones(B, L, device="cuda")
    nm[B - 1, 1:] = 0
    return pe, pm, ne, nm


def _image(m, B, H, W, seed=6):
    g = torch.Generator().manual_seed(seed)
    C = m.cfg.in_channels
    img = torch.randn(B, C, 1, H, W, generator=g) * 1.5 + 0.3
    mean, std = torch.randn(C, generator=g) * 0.2, torch.rand(C, generator=g) + 0.5
    return img, mean, std


def _oracle_i2v(om, pe, pm, ne, nm, img, mean, std, noise, sig, F, H, W, g, rope):
    """Plain-torch fp32 restatement of LTXImageToVideoPipeline (CPU): prepare_latents (normalise, repeat, blend with
    the noise under the frame-0 mask, pack), then per step cat([latents] * 2) cast to bf16, timestep
    t.expand(2B).unsqueeze(-1) * (1 - mask), guidance on noise_pred.float(), scheduler.step on the frames after the
    first and cat with the first frame (on the packed layout: frame 0 is the first H W tokens)."""
    B, C = img.shape[:2]
    init = ((img - mean.view(1, -1, 1, 1, 1)) * 1.0 / std.view(1, -1, 1, 1, 1)).repeat(1, 1, F, 1, 1)
    mask = torch.zeros(B, 1, F, H, W)
    mask[:, :, 0] = 1.0
    x = (init * mask + noise * (1 - mask)).reshape(B, C, -1).transpose(1, 2)
    cmask = torch.cat([mask.reshape(B, -1)] * 2)
    ehs, emask = torch.cat([ne, pe]).float(), torch.cat([nm, pm]).float()
    hw = H * W
    for i in range(sig.numel() - 1):
        inp = torch.cat([x] * 2).to(torch.bfloat16).float()
        t = (sig[i] * 1000.0).expand(inp.shape[0]).unsqueeze(-1) * (1 - cmask)
        pred = om(inp, ehs, t, emask, F, H, W, rope)[0].float()
        u, c = pred.chunk(2)
        v = u + g * (c - u)
        x = torch.cat([x[:, :hw], x[:, hw:] + (sig[i + 1] - sig[i]) * v[:, hw:]], 1)
    return x, init[:, :, :1].reshape(B, C, -1).transpose(1, 2)


@pytest.mark.timeout(600)
def test_i2v_sampler_matches_the_oracle_pipeline_loop():
    """SMALL, B = 2, F = 3 latent frames, 4 steps, guidance 3.  Frame 0 of the result is the normalised image latents bit
    for bit.  Measured on an H100 80GB HBM3: final latents rel_err 1.5e-3."""
    from finetrainers_b200.sampling import ltx_sigmas
    from finetrainers_b200.specification import LTXVideoModelSpecification
    O, om, bm = build_pair(SMALL, 64)
    spec = LTXVideoModelSpecification(bm.cfg)
    B, F, H, W = 2, 3, 4, 9
    pe, pm, ne, nm = _prompts(bm, B, 24)
    img, mean, std = _image(bm, B, H, W)
    noise = torch.randn(B, 32, F, H, W, generator=torch.Generator().manual_seed(4))
    packed_noise = noise.reshape(B, 32, -1).transpose(1, 2).contiguous()
    got = spec.generate_latents(bm, pe, pm, ne, nm, num_frames=17, height=128, width=288, num_inference_steps=4,
                                guidance_scale=3.0, latents=packed_noise, image_latents=img, latents_mean=mean,
                                latents_std=std)
    sig = ltx_sigmas(4, F * H * W)
    with torch.no_grad():
        want, frame0 = _oracle_i2v(om, pe.cpu(), pm.cpu(), ne.cpu(), nm.cpu(), img, mean, std, noise, sig, F, H, W, 3.0,
                                   ROPE)
    assert torch.equal(got[:, :H * W].cpu(), frame0)
    e_x = rel_err(got.cpu(), want)
    print(f"\ni2v sampler vs oracle: final latents rel_err {e_x:.2e}")
    assert e_x < 2e-2


@pytest.mark.parametrize("case", ["resident", "fp8", "hd128"])
def test_i2v_graph_replay_equals_eager_steps(case):
    from finetrainers_b200.specification import LTXVideoModelSpecification
    cfgk = dict(SMALL128 if case == "hd128" else SMALL, num_layers=3)
    m = _model(cfgk, layerwise=case == "fp8")
    spec = LTXVideoModelSpecification(m.cfg)
    pe, pm, ne, nm = _prompts(m, 2, 24)
    img, mean, std = _image(m, 2, 4, 9)
    kw = dict(num_frames=17, height=128, width=288, num_inference_steps=6, image_latents=img, latents_mean=mean,
              latents_std=std)
    a = spec.generate_latents(m, pe, pm, ne, nm, generator=torch.Generator().manual_seed(2), cuda_graph=True, **kw)
    b = spec.generate_latents(m, pe, pm, ne, nm, generator=torch.Generator().manual_seed(2), cuda_graph=False, **kw)
    assert a.shape == (2, 108, 32) and a.dtype == torch.float32
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)
    assert not torch.equal(a[:, 36:72], a[:, :36])   # later frames moved away from the image


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_i2v_sample_between_training_steps_changes_nothing(graph):
    from finetrainers_b200.specification import LTXVideoModelSpecification
    from finetrainers_b200.trainer import SFTTrainStep

    def run(with_sample):
        random.seed(0)
        m = _model(dict(SMALL, num_layers=3))
        st = SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=graph)
        st.spec.first_frame_conditioning_p = 0.0
        g = torch.Generator().manual_seed(77)
        out = []
        for i in range(3):
            lat = torch.randn(2, 32, 3, 4, 9, generator=g).bfloat16().cuda()
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
                pe, pm, ne, nm = _prompts(m, 2, 24)
                img, mean, std = _image(m, 2, 4, 9)
                s = spec.generate_latents(m, pe, pm, ne, nm, num_frames=17, height=128, width=288,
                                          num_inference_steps=3, generator=torch.Generator().manual_seed(1),
                                          image_latents=img, latents_mean=mean, latents_std=std)
                assert torch.isfinite(s).all()
        return out

    a, b = run(False), run(True)
    for i, (x, y) in enumerate(zip(a, b)):
        for what, u, v in zip(("loss", "lora_grad_flat", "lora_flat"), x, y):
            assert torch.equal(u, v), (i, what)


@pytest.mark.timeout(1800)
def test_13b_i2v_sample_between_graph_training_steps():
    """The 13B geometry (48 blocks, r = 64): 2 training steps with CUDA graphs, a 3-step guided I2V sample at 2688
    tokens, one more training step.  Peak below 70 GB."""
    from finetrainers_b200.model import LTXConfig
    from finetrainers_b200.specification import LTXVideoModelSpecification
    from finetrainers_b200.trainer import SFTTrainStep
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 70e9:
        pytest.skip(f"needs 70 GB of free device memory, {free / 1e9:.1f} GB are free")
    torch.cuda.reset_peak_memory_stats()
    random.seed(0)
    m = _model(LTXConfig.ltx_13b().to_dict(), std=0.02)
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)
    g = torch.Generator().manual_seed(1234)
    lat = torch.randn(1, 128, 7, 16, 24, generator=g).bfloat16().cuda()
    ehs = (torch.randn(1, 128, 4096, generator=g) * 0.1).bfloat16().cuda()
    mask = (torch.arange(128)[None] < 100).cuda()
    mean, std = torch.zeros(1, 128, device="cuda"), torch.ones(1, 128, device="cuda")
    for i in range(3):
        if i == 2:
            pe, pm, ne, nm = _prompts(m, 1, 128)
            img, imean, istd = _image(m, 1, 16, 24)
            s = LTXVideoModelSpecification(m.cfg).generate_latents(
                m, pe, pm, ne, nm, num_frames=49, height=512, width=768, num_inference_steps=3,
                generator=torch.Generator().manual_seed(1), image_latents=img, latents_mean=imean, latents_std=istd)
            assert s.shape == (1, 2688, 128) and torch.isfinite(s).all()
        st.train_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                      {"latents": lat, "latents_mean": mean, "latents_std": std})
        torch.cuda.synchronize()
        assert torch.isfinite(st.metrics).all()
    peak = torch.cuda.max_memory_allocated()
    print(f"\n13B I2V: max_memory_allocated {peak / 1e9:.2f} GB")
    assert peak < 70e9
