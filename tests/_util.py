import torch


def rnd(*shape, scale=1.0, dtype=torch.bfloat16, device="cuda"):
    return (torch.randn(*shape, device=device) * scale).to(dtype)


def rel_err(got, ref, floor=1e-6):
    """max |got - ref| relative to the reference's max magnitude (floored so exact-zero references compare absolutely)."""
    got, ref = got.float(), ref.float()
    return ((got - ref).abs().max() / max(ref.abs().max().item(), floor)).item()


def mm64(a, b):
    """fp64 product a @ b^T of bf16-valued operands (a [M, K], b [N, K]; any layout views), on their device."""
    return a.double() @ b.double().t()


def absmm64(a, b):
    """|a| @ |b|^T in fp64: the scale of the accumulation error of a @ b^T (bounds every partial sum)."""
    return a.double().abs() @ b.double().abs().t()


def bf16_ulp(x):
    """Spacing of bf16 numbers at |x| (fp64 in, fp64 out): 2^(e - 7) for |x| in [2^e, 2^(e+1)), the subnormal
    spacing 2^-133 below 2^-126."""
    x = x.double().abs().clamp_min(2.0 ** -126)
    _, e = torch.frexp(x)                      # x = m * 2^e, m in [0.5, 1)
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


def f32_ulp(x):
    """Spacing of fp32 numbers at |x| (fp64 in, fp64 out)."""
    x = x.double().abs().clamp_min(2.0 ** -126)
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e - 24).to(torch.int32))


def check_bound(got, ref, bound, what=""):
    """Element-wise |got - ref| <= bound (all compared in fp64).  Returns the worst error/bound ratio; raises
    AssertionError naming the worst element (index, got, ref, bound) when that ratio exceeds 1 or anything is NaN."""
    got, ref, bound = got.double(), ref.double(), bound.double().expand_as(ref)
    err = (got - ref).abs()
    ratio = err / bound
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    flat = int(ratio.argmax())
    worst = ratio.reshape(-1)[flat].item()
    if not worst <= 1.0:
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), ratio.shape))
        bad = int((ratio > 1).sum())
        raise AssertionError(f"{what}: {bad} element(s) out of bound, worst ratio {worst:.3g} at {idx}: "
                             f"got {got[idx].item()!r} ref {ref[idx].item()!r} bound {bound[idx].item():.3g}")
    return worst


# Bit patterns written around kernel outputs: negative NaNs with a payload no arithmetic produces (the fp32 one is the
# bf16 one twice), so a stray store of any computed value changes them.
SENTINEL_BF16 = 0xFFA5 - (1 << 16)
SENTINEL_F32 = 0xFFA5FFA5 - (1 << 32)


def _int_view(t):
    return t.view({torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float32: torch.int32}[t.dtype])


def sentinel_buffer(numel, dtype, device="cuda"):
    """A flat buffer of `numel` elements of `dtype` filled with the sentinel bit pattern."""
    buf = torch.empty(numel, dtype=dtype, device=device)
    _int_view(buf).fill_(SENTINEL_BF16 if buf.element_size() == 2 else SENTINEL_F32)
    return buf


def window(buf, offset, rows, cols, ld):
    """The [rows, cols] matrix with leading dimension ld starting `offset` elements into the flat buffer."""
    return buf.as_strided((rows, cols), (ld, 1), offset)


def check_sentinel(buf, windows, what=""):
    """Every element of the flat buffer outside the given windows still holds the sentinel bit pattern."""
    inside = torch.zeros(buf.numel(), dtype=torch.bool, device=buf.device)
    for w in windows:
        window(inside, w.storage_offset() - buf.storage_offset(), w.shape[0], w.shape[1], w.stride(0)).fill_(True)
    pat = SENTINEL_BF16 if buf.element_size() == 2 else SENTINEL_F32
    changed = (_int_view(buf) != pat) & ~inside
    n = int(changed.sum())
    if n:
        raise AssertionError(f"{what}: {n} element(s) outside the output windows were written, first at flat offset "
                             f"{int(changed.nonzero()[0])}")


def build_pair(cfg_kwargs, rank, seed=0, lora_b_std=0.02, device="cuda", alpha=None):
    """oracle (CPU, fp32 math, bf16-valued base weights) + H100 model with identical parameters; lora_alpha defaults to
    the rank (scaling 1)."""
    from oracle import ltx_oracle as O
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    alpha = rank if alpha is None else alpha
    om = O.LTXTransformerOracle(O.LTXConfig(**cfg_kwargs))
    O.add_lora(om, rank, alpha)
    O.synthetic_init_(om, seed=seed, lora_b_std=lora_b_std)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    bm = B200LTXTransformer(LTXConfig(**cfg_kwargs), torch.bfloat16, device)
    bm.add_adapter(rank, alpha)
    bm.load_state_dict(om.state_dict(), strict=True)
    bm.prepare()
    return O, om, bm


def run_b200_micro(bm, batch, scheme="none"):
    from finetrainers_b200.trainer import SFTTrainStep
    st = SFTTrainStep(bm, flow_weighting_scheme=scheme)
    st.spec.first_frame_conditioning_p = 0.0
    cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(),
            "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
    lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(),
           "latents_std": batch["latents_std"].cuda()}
    st.micro_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda())
    torch.cuda.synchronize()
    B = batch["latents"].shape[0]
    S = batch["latents"].shape[2] * batch["latents"].shape[3] * batch["latents"].shape[4]
    ws = bm._workspace(B, S, batch["encoder_hidden_states"].shape[1])
    return st, st.loss_buf.item(), ws["pred"].view(B, S, -1).float().cpu()


SMALL = dict(in_channels=32, out_channels=32, num_attention_heads=4, attention_head_dim=64, cross_attention_dim=256,
             num_layers=2, caption_channels=128)
