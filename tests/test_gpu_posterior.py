"""GPU: training from precomputed VAE moments (``compute_posterior=False``).

- Kernel: b2d_prep_posterior_noise_pack against the torch restatement (_posterior.py on top of the oracle) run on the
  GPU from the same bf16 moments, eps, noise and sigmas: latents_out, x_t and target bit-identical (NaN in, NaN out),
  outputs inside sentinel buffers; against the CPU golden of the reference's own class within one bf16 ulp, only where
  CPU and CUDA exp round apart.
- Equivalence: a step fed moments is bit-identical to a step fed the latent _posterior.py samples from the same
  generator state (eager, CUDA graphs, gradient accumulation).
- Parity: spec.forward and the train step on the posterior path against the fp32 oracle.
- Feed: moments items on disk through the reader, sampler and collate into train_step.
"""
import os

import pytest
import torch

from _posterior import posterior_sample, spec_forward_moments
from _util import bf16_ulp, build_pair, check_sentinel, rel_err, sentinel_buffer, window, SMALL

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAD = 64
EDGES = [-1e4, -31.0, -30.0, 20.0, 20.5, 1e4, float("inf"), float("-inf"), float("nan")]


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


class Guarded:
    """n bf16 elements inside a sentinel-filled buffer with PAD elements of margin on each side."""

    def __init__(self, n):
        self.n = n
        self.buf = sentinel_buffer(n + 2 * PAD, torch.bfloat16)
        self.t = self.buf[PAD:PAD + n]

    def check(self, what):
        check_sentinel(self.buf, [window(self.buf, PAD, 1, self.n, self.n)], what)


def _same(a, b, what):
    """Bit-identical, NaN matching NaN."""
    a, b = a.reshape(-1).cpu(), b.reshape(-1).cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), f"{what}: NaN positions differ"
    diff = int((a.view(torch.int16)[~na] != b.view(torch.int16)[~nb]).sum())
    assert diff == 0, f"{what}: {diff} element(s) differ"


def _moments(g, B, C, F, HW, edges=True):
    mean = torch.randn(B, C, F, 1, HW, generator=g) * 0.8
    logvar = torch.rand(B, C, F, 1, HW, generator=g) * 10.0 - 7.0
    if edges:
        flat = logvar.view(-1)
        pos = torch.randperm(flat.numel(), generator=g)[:len(EDGES)]
        flat[pos] = torch.tensor(EDGES)[:pos.numel()]
    return torch.cat([mean, logvar], dim=1).bfloat16()


def _oracle_prologue(moments, eps, noise, mean, std, sig, sff):
    """The restated posterior sample (_posterior.py), then the oracle's normalise, flow-match x_t, pack and target, in
    torch on the tensors' device."""
    from oracle.ltx_oracle import flow_match_target, flow_match_xt, normalize_latents, pack_latents
    B = moments.shape[0]
    x = posterior_sample(moments, eps=eps)
    x0 = normalize_latents(x, mean, std)
    v = lambda s: s.view(B, 1, 1, 1, 1)
    if sff is not None:
        noisy = torch.cat([flow_match_xt(x0[:, :, :1], noise[:, :, :1], v(sff)),
                           flow_match_xt(x0[:, :, 1:], noise[:, :, 1:], v(sig))], dim=2)
    else:
        noisy = flow_match_xt(x0, noise, v(sig))
    return x, pack_latents(noisy).bfloat16(), pack_latents(flow_match_target(noise, x0)).bfloat16()


def _run_kernel(ops, moments, eps, noise, mean, std, sig, sff, B, C, F, HW):
    n = B * C * F * HW
    lo, xt, tg = Guarded(n), Guarded(n), Guarded(n)
    ops.prep_posterior_noise_pack(moments, eps, noise, mean, std, sig, sff, xt.t, tg.t, B, C, F, HW, latents_out=lo.t)
    torch.cuda.synchronize()
    for gd, name in ((lo, "latents_out"), (xt, "x_t"), (tg, "target")):
        gd.check(name)
    return lo.t.clone(), xt.t.clone(), tg.t.clone()


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("C", [8, 128])
@pytest.mark.parametrize("F,HW", [(1, 7), (3, 33)])
@pytest.mark.parametrize("first_frame", [False, True])
def test_prep_posterior_kernel_bit_identical_to_oracle(ops, B, C, F, HW, first_frame):
    g = torch.Generator().manual_seed(B * 1000 + C + F * 10 + HW)
    moments = _moments(g, B, C, F, HW).cuda()
    eps = torch.randn(B, C, F, 1, HW, generator=g).bfloat16().cuda()
    noise = torch.randn(B, C, F, 1, HW, generator=g).bfloat16().cuda()
    mean, std = (torch.randn(B, C, generator=g) * 0.1).cuda(), (torch.rand(B, C, generator=g) + 0.5).cuda()
    sig = torch.tensor([1.0, 0.37][:B]).cuda()
    sff = (torch.rand(B, generator=g) * 0.25).cuda() if first_frame else None
    lo, xt, tg = _run_kernel(ops, moments, eps, noise, mean, std, sig, sff, B, C, F, HW)
    x, xt_o, tg_o = _oracle_prologue(moments, eps, noise, mean, std, sig, sff)
    _same(lo, x, "latents_out")
    _same(xt, xt_o, "x_t")
    _same(tg, tg_o, "target")
    assert torch.isnan(lo).any() and torch.isfinite(lo).sum() > lo.numel() // 2
    # the kernel without latents_out computes the same
    n = B * C * F * HW
    xt2, tg2 = Guarded(n), Guarded(n)
    ops.prep_posterior_noise_pack(moments, eps, noise, mean, std, sig, sff, xt2.t, tg2.t, B, C, F, HW)
    xt2.check("x_t without latents_out")
    tg2.check("target without latents_out")
    _same(xt2.t, xt, "x_t without latents_out")
    _same(tg2.t, tg, "target without latents_out")


def test_prep_posterior_kernel_against_the_reference_golden(ops):
    """The reference's DiagonalGaussianDistribution run on the CPU (tests/golden/posterior_golden.pt): at most one bf16
    ulp apart, and only where CPU and CUDA exp round 0.5 * clamp(logvar) to different bf16 values."""
    cases = torch.load(os.path.join(ROOT, "tests", "golden", "posterior_golden.pt"), weights_only=False)["cases"]
    report = []
    for c in cases:
        B, C, F, H, W = c["shape"]
        mom, eps = c["moments"].cuda(), c["eps"].cuda()
        zeros = torch.zeros(B, C, F, H, W, dtype=torch.bfloat16, device="cuda")
        mean, std = torch.zeros(B, C, device="cuda"), torch.ones(B, C, device="cuda")
        lo, _, _ = _run_kernel(ops, mom, eps, zeros, mean, std, torch.zeros(B, device="cuda"), None, B, C, F, H * W)
        got, ref = lo.view(B, C, F, H, W).cpu(), c["sample"]
        nan = torch.isnan(ref)
        assert torch.equal(torch.isnan(got), nan), c["shape"]
        differ = (got.view(torch.int16) != ref.view(torch.int16)) & ~nan
        lv = torch.clamp(c["moments"][:, C:], -30.0, 20.0)
        std_cpu, std_gpu = torch.exp(0.5 * lv), torch.exp(0.5 * lv.cuda()).cpu()
        exp_apart = (std_cpu.view(torch.int16) != std_gpu.view(torch.int16)) & ~torch.isnan(std_cpu)
        assert not (differ & ~exp_apart).any(), f"{c['shape']}: differs where exp agrees"
        d = (got.double() - ref.double()).abs()[differ]
        assert (d <= bf16_ulp(ref.double()[differ])).all(), c["shape"]
        report.append((c["shape"], int(differ.sum()), int(exp_apart.sum()), ref.numel()))
    print("\nposterior golden: (shape, elements apart, exp apart, elements):", report)


def test_prep_posterior_empty_shape_is_refused(ops):
    from finetrainers_b200.lib import B2DError
    t = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    f = torch.zeros(4, device="cuda")
    for shape in ((0, 4, 1, 1), (1, 0, 1, 1), (1, 4, 0, 1), (1, 4, 1, 0)):
        with pytest.raises(B2DError, match=r"\(code -1\)"):
            ops.prep_posterior_noise_pack(t, t, t, f, f, f, None, t, t, *shape)


# ---------------------------------------------------------------------------------------------------------------------
# whole steps
# ---------------------------------------------------------------------------------------------------------------------
def _full_width_model(num_layers, seed=0):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    m = B200LTXTransformer(LTXConfig(num_layers=num_layers), torch.bfloat16, "cuda")
    m.add_adapter(64, 64)
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for n, p in sorted(m.named_parameters(), key=lambda kv: kv[0]):
            if "scale_shift_table" in n:
                p.copy_(torch.randn(p.shape, device="cuda", generator=g) / p.shape[-1] ** 0.5)
            elif "norm_q" in n or "norm_k" in n:
                p.fill_(1.0)
            elif "lora_A" in n:
                p.copy_((torch.rand(p.shape, device="cuda", generator=g) * 2 - 1) / p.shape[1] ** 0.5)
            else:
                p.copy_(torch.randn(p.shape, device="cuda", generator=g) * 0.02)
    m.prepare()
    return m


def _step_inputs(g, B, C, F, H, W, L=64):
    moments = torch.cat([torch.randn(B, C, F, H, W, generator=g) * 0.8,
                         torch.rand(B, C, F, H, W, generator=g) * 4.0 - 5.0], dim=1).bfloat16().cuda()
    cond = {"encoder_hidden_states": (torch.randn(B, L, 4096, generator=g)).bfloat16().cuda(),
            "encoder_attention_mask": (torch.arange(L)[None] < L - 9).expand(B, L).cuda()}
    mean, std = (torch.randn(B, C, generator=g) * 0.1).cuda(), (torch.rand(B, C, generator=g) + 0.5).cuda()
    return moments, cond, mean, std


@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", ["eager", "graph", "accum2"])
def test_moments_step_bit_identical_to_oracle_sampled_latents(mode):
    """Two steps seeded alike, full width (D = 2048), 2 blocks, r = 64.  A is fed moments; B is fed the latent the oracle
    samples from B's generator (sigmas then eps, the order of the step), and then draws the noise and first-frame sigma
    from the post-eps state itself.  After 3 optimizer steps: loss, grad norm and adapters bit-identical."""
    from finetrainers_b200.trainer import SFTTrainStep, prepare_sigmas
    accum = 2 if mode == "accum2" else 1
    steps = []
    for _ in range(2):
        m = _full_width_model(2)
        st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=7, use_cuda_graph=(mode == "graph"),
                          gradient_accumulation_steps=accum)
        st.spec.first_frame_conditioning_p = 1.0
        steps.append(st)
    a, b = steps
    g = torch.Generator().manual_seed(3)
    B, C, F, H, W = 1, 128, 3, 4, 8
    out = {"a": [], "b": []}
    for i in range(3 * accum):
        moments, cond, mean, std = _step_inputs(g, B, C, F, H, W)
        ma = a.train_step(cond, {"latents": moments, "latents_mean": mean, "latents_std": std}, sync_metrics=True,
                          compute_posterior=False)
        sig = prepare_sigmas(b.scheduler, b.scheduler_sigmas, B, 1000, b.scheme, b.flow_logit_mean, b.flow_logit_std,
                             b.flow_mode_scale, b.device, b.generator)
        x = posterior_sample(moments, generator=b.generator)
        mb = b.train_step(cond, {"latents": x, "latents_mean": mean, "latents_std": std}, sigmas=sig,
                          sync_metrics=True)
        if (i + 1) % accum == 0:
            out["a"].append((ma["train/global_avg_loss"], ma["train/grad_norm"]))
            out["b"].append((mb["train/global_avg_loss"], mb["train/grad_norm"]))
    torch.cuda.synchronize()
    assert out["a"] == out["b"], out
    assert all(l == l and l > 0 for l, _ in out["a"])
    assert torch.equal(a.transformer.lora_flat, b.transformer.lora_flat)
    sample = torch.randperm(a.transformer.lora_flat.numel(), device="cuda")[:100_000]
    assert torch.equal(a.transformer.lora_flat[sample], b.transformer.lora_flat[sample])
    if mode == "graph":
        assert len(a._graphs) == 1 and len(b._graphs) == 1
        (ka,), (kb,) = a._static.keys(), b._static.keys()
        assert ka[-1] is True and kb[-1] is False
    print(f"\n{mode}: (loss, grad norm) per optimizer step {out['a']}")


def _lora_grad_errors(bm, om):
    og = dict(om.named_parameters())
    errs = {}
    for n, p in bm.named_parameters():
        if "lora_" in n:
            go = og[n].grad
            errs[n] = (p.grad.float().cpu() - go).abs().max().item() / go.abs().max().item()
    return errs


@pytest.mark.timeout(900)
def test_posterior_path_matches_fp32_oracle():
    """Full width, 1 block, r = 64, with injected eps and noise: spec.forward(compute_posterior=False) with a torch loss,
    and one train step, against the fp32 oracle's moments path: loss within 1e-3 relative, every adapter gradient within
    5 % of its own scale."""
    from finetrainers_b200.specification import LTXVideoModelSpecification
    from finetrainers_b200.trainer import SFTTrainStep
    O, om, bm = build_pair(dict(num_layers=1), 64)
    batch = O.make_synthetic_batch(om.cfg, 1, 7, 16, 24, seed=1234, text_scale=1.0)
    g = torch.Generator().manual_seed(5)
    shp = batch["latents"].shape
    moments = torch.cat([batch["latents"].float(), torch.rand(shp, generator=g) * 4.0 - 5.0], dim=1).bfloat16()
    eps = torch.randn(shp, generator=g).bfloat16()
    mean, std = torch.randn(1, 128, generator=g) * 0.1, torch.rand(1, 128, generator=g) + 0.5
    pred_o, target_o, sig_o = spec_forward_moments(om, moments.float(), mean, std,
                                                   batch["encoder_hidden_states"].float(),
                                                   batch["encoder_attention_mask"], batch["sigmas"],
                                                   noise=batch["noise"].float(), posterior_eps=eps.float())
    loss_o = O.sft_loss(pred_o, target_o, sig_o)
    loss_o.backward()
    cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(),
            "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}

    def lat():
        return {"latents": moments.cuda(), "latents_mean": mean.cuda(), "latents_std": std.cuda()}

    # (a) the finetrainers-style path: spec.forward, loss in torch, autograd
    spec = LTXVideoModelSpecification(bm.cfg)
    spec.first_frame_conditioning_p = 0.0
    ld = lat()
    pred, target, sig = spec.forward(bm, cond, ld, batch["sigmas"].cuda(), compute_posterior=False,
                                     noise=batch["noise"].cuda(), posterior_noise=eps.cuda())
    assert "hidden_states" in ld and "latents" not in ld and "latents_mean" not in ld
    assert rel_err(target.float().cpu(), target_o.detach()) < 2e-2
    assert rel_err(pred.float().cpu(), pred_o.detach()) < 3e-2
    loss = (pred.float() - target.float()).pow(2).mean(list(range(1, 3))).mean()
    loss.backward()
    err_spec = abs(loss.item() - loss_o.item()) / loss_o.item()
    assert err_spec < 1e-3
    errs = _lora_grad_errors(bm, om)
    assert len(errs) == 16 and max(errs.values()) < 5e-2, errs
    # (b) the train step
    bm.lora_grad_flat.zero_()   # the adapters' .grad are views of this buffer
    st = SFTTrainStep(bm, flow_weighting_scheme="none")
    st.spec.first_frame_conditioning_p = 0.0
    st.micro_step(cond, lat(), sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda(),
                  compute_posterior=False, posterior_noise=eps.cuda())
    torch.cuda.synchronize()
    err_step = abs(st.loss_buf.item() - loss_o.item()) / loss_o.item()
    assert err_step < 1e-3
    errs = _lora_grad_errors(bm, om)
    assert len(errs) == 16 and max(errs.values()) < 5e-2, errs
    print(f"\nposterior parity: loss err spec.forward {err_spec:.2e}, step {err_step:.2e}; worst grad err "
          f"{max(errs.values()):.2e} ({max(errs, key=errs.get)})")


def test_precomputed_moments_feed_into_train_step(tmp_path):
    """Moments items on disk (the reference's layout, [1, 2C, F, H, W] per item, two resolutions) through the async
    reader, the resolution sampler and collate into train_step(compute_posterior=False): every step finite.  Batch
    size 1, as the LTX recipe trains: collate takes latents_mean / latents_std from the first item of a batch, so they
    describe one sample.  The step runs eagerly: a CUDA-graph capture is opened in torch's global capture mode, which
    forbids the reader thread's event waits and pinned allocations while it is open (the moments path under graphs is
    covered by test_moments_step_bit_identical_to_oracle_sampled_latents)."""
    from finetrainers_b200.data import PrecomputedOnceReader, ResolutionSampler, collate, save_item
    from finetrainers_b200.trainer import SFTTrainStep
    _, _, bm = build_pair(SMALL, 64, seed=2)
    C = SMALL["in_channels"]
    g = torch.Generator().manual_seed(11)
    for i in range(6):
        F, H, W = (2, 4, 8) if i % 2 == 0 else (3, 4, 6)
        mom = torch.cat([torch.randn(1, C, F, H, W, generator=g), torch.rand(1, C, F, H, W, generator=g) * 4 - 5], 1)
        save_item({"latents": mom.bfloat16(), "num_frames": F, "height": H, "width": W,
                   "latents_mean": torch.randn(1, C, generator=g) * 0.1, "latents_std": torch.rand(1, C, generator=g) + 0.5},
                  i, tmp_path / "latents", "latent")
        save_item({"encoder_hidden_states": torch.randn(1, 16, SMALL["caption_channels"], generator=g).bfloat16(),
                   "encoder_attention_mask": torch.ones(1, 16)}, i, tmp_path / "conditions", "condition")
    dev = torch.device("cuda", 0)
    lat_rd = iter(PrecomputedOnceReader(tmp_path / "latents", "latent", device=dev))
    cond_rd = iter(PrecomputedOnceReader(tmp_path / "conditions", "condition", device=dev))
    sampler = ResolutionSampler(batch_size=1, dim_keys={"latents": (2, 3, 4)})
    st = SFTTrainStep(bm, flow_weighting_scheme="logit_normal", seed=1)
    losses = []
    while len(losses) < 8:
        sampler.consume(next(cond_rd), next(lat_rd))
        while sampler.is_ready:
            conds, lats = sampler.get_batch()
            m = st.train_step(collate(list(conds)), collate(list(lats)), sync_metrics=True, compute_posterior=False)
            losses.append((m["train/global_avg_loss"], m["train/grad_norm"]))
    lat_rd.close()
    cond_rd.close()
    assert all(torch.isfinite(torch.tensor(v)).all() for v in losses), losses
    assert len(st._static) == 2 and all(k[-1] is True for k in st._static)
    print("\nfeed: (loss, grad norm) per step", losses)
