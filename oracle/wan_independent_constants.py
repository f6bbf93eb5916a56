"""Second, independent derivation of the UPSTREAM-ONLY constants the Wan-2.1 oracle restates — TEST INFRASTRUCTURE.

The companion of ``oracle/independent_constants.py`` (LTX-Video) for ``oracle/wan_oracle.py``: diffusers is neither
vendored in the reference nor installed here, so the Wan module arithmetic cannot be pinned against reference-held
vectors.  What can be done offline is to derive each upstream constant a second time, from the published definition,
in a different style (scalar float64 loops, no torch, no code shared with ``wan_oracle.py``), and check the two against
each other (tests/test_host_wan.py) and against the kernels (tests/test_gpu_wan.py).

Provenance (diffusers ``src/diffusers/models/transformers/transformer_wan.py`` and ``models/embeddings.py``, 0.33;
the 1.3B / 14B values from the published ``Wan-AI/Wan2.1-T2V-*-Diffusers`` transformer configs):

| constant | value | upstream symbol |
|---|---|---|
| RoPE split of a head | h = w = 2 (head_dim // 6), t = head_dim - h - w: 44 / 42 / 42 at 128 | ``WanRotaryPosEmbed.__init__``: ``h_dim = w_dim = 2 * (attention_head_dim // 6)``, ``t_dim = attention_head_dim - h_dim - w_dim`` |
| RoPE frequencies | pair i of a part of n dims: ``theta ** (-2 i / n)``, theta 10000, float64 | ``get_1d_rotary_pos_embed(dim, max_seq_len, theta, use_real=False, repeat_interleave_real=False, freqs_dtype=torch.float64)``: ``1 / theta ** (arange(0, dim, 2)[: dim // 2] / dim)`` |
| RoPE positions | integer grid index on the post-patch grid (f, h // 2, w // 2), table of ``rope_max_seq_len`` = 1024 rows | ``WanRotaryPosEmbed.forward``: ``freqs[0][:ppf]``, ``freqs[1][:pph]``, ``freqs[2][:ppw]``, concatenated t, h, w per token |
| RoPE pairs | channels (2 i, 2 i + 1) of a head form one complex number | ``WanAttnProcessor2_0.apply_rotary_emb``: ``view_as_complex(x.unflatten(3, (-1, 2)))`` |
| timestep sinusoid | ``freq_dim`` = 256, ``[cos | sin]``, ``exp(-ln(10000) i / 128)`` | ``WanTimeTextImageEmbedding.timesteps_proj = Timesteps(freq_dim, flip_sin_to_cos=True, downscale_freq_shift=0)`` |
| patch embedding | Conv3d(16, D, kernel = stride = (1, 2, 2)); its weight [D, 16, 1, 2, 2] flattened row-major: k = c 4 + kh 2 + kw | ``WanTransformer3DModel.patch_embedding`` |
| token order | tokens f-major, then h // 2, then w // 2 | ``patch_embedding(x).flatten(2).transpose(1, 2)`` |
| output channel order | proj_out column (kh 2 + kw) 16 + c | ``WanTransformer3DModel.forward`` unpatchify: ``reshape(B, F', H', W', p_t, p_h, p_w, -1).permute(0, 7, 1, 4, 2, 5, 3, 6)`` |
"""
import math


def wan_rope_split(head_dim: int):
    """(t, h, w) channel counts of one head."""
    hw = 2 * (head_dim // 6)
    return head_dim - 2 * hw, hw, hw


def wan_rope_entry(f: int, h: int, w: int, pair: int, head_dim: int = 128, theta: float = 10000.0):
    """(cos, sin) of rotary pair ``pair`` (0 .. head_dim / 2) of every head, for the token at post-patch grid position
    (f, h, w)."""
    t_dim, h_dim, _ = wan_rope_split(head_dim)
    if pair < t_dim // 2:
        i, n, p = pair, t_dim, f
    elif pair < t_dim // 2 + h_dim // 2:
        i, n, p = pair - t_dim // 2, h_dim, h
    else:
        i, n, p = pair - t_dim // 2 - h_dim // 2, h_dim, w
    ang = p * (1.0 / theta ** ((2 * i) / n))
    return math.cos(ang), math.sin(ang)


def wan_sinusoid(t: float, freq_dim: int = 256):
    """freq_dim numbers: cos(t f_i) for i < freq_dim / 2, then sin(t f_i)."""
    half = freq_dim // 2
    out = [0.0] * freq_dim
    for i in range(half):
        fr = math.exp(-math.log(10000.0) * i / half)
        out[i] = math.cos(t * fr)
        out[half + i] = math.sin(t * fr)
    return out


def conv_k(c: int, kh: int, kw: int) -> int:
    """Column of the Conv3d weight viewed as [D, 4 C] that multiplies latent channel c at patch offset (kh, kw)."""
    return c * 4 + kh * 2 + kw


def out_k(c: int, kh: int, kw: int, channels: int = 16) -> int:
    """proj_out column that unpatchifies to channel c at patch offset (kh, kw)."""
    return (kh * 2 + kw) * channels + c


def token(f: int, h: int, w: int, height: int, width: int) -> int:
    """Token index of latent position (f, h, w) of an [F, height, width] latent after the (1, 2, 2) patch."""
    return (f * (height // 2) + h // 2) * (width // 2) + w // 2
