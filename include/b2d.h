/* b2d.h — C ABI of libb2d.so: the sm_90a DiT-training-step kernels behind finetrainers' LTX hot path.
 *
 * The reference (a-r-r-o-w/finetrainers @ f476c37) is pure Python and has NO FFI; every entry point below replaces a
 * span of PyTorch/diffusers/peft calls on the hot path.  The citation after each declaration names that span
 * (paths relative to the reference repository; "diffusers:"/"peft:" = the un-vendored dependency the reference delegates to).
 *
 * Conventions: plain pointers + sizes, no torch types, no hidden allocation, no implicit synchronisation.  All device
 * pointers are 16-byte aligned, activations/weights bf16 row-major, statistics/gradients fp32.  The last argument is
 * the CUDA stream (cudaStream_t passed as void*).  Return 0 on success, negative b2d_status on error
 * (b2d_last_error() gives a thread-local message).  Callable from any host thread (autograd's backward thread too).
 */
#ifndef B2D_H
#define B2D_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  B2D_OK = 0,
  B2D_ERR_SHAPE = -1,   /* unsupported / inconsistent dims */
  B2D_ERR_ALIGN = -2,   /* pointer or leading dimension not 16-byte aligned */
  B2D_ERR_ARCH = -3,    /* device is not sm_90 */
  B2D_ERR_CUDA = -4,    /* CUDA runtime/driver error (see b2d_last_error) */
  B2D_ERR_ARG = -5
} b2d_status;

int b2d_version(void);                 /* ABI version (this header = 1) */
const char* b2d_last_error(void);      /* thread-local, never NULL */
int b2d_device_check(void);            /* B2D_OK iff current device is compute capability 9.x */

/* ---------------------------------------------------------------------------------------------------------------
 * GEMM on Hopper tensor cores (TMA -> 128B-swizzled smem -> wgmma -> register accumulators -> fused epilogue).
 *   C[M,N] = epilogue( alpha * ( opA(A)[M,K] * opB(B)[N,K]^T  +  A2[M,K2] * B2[N,K2]^T ) )
 * a_mn_major = 0: A is row-major [M, K] (lda);  1: A is given as its transpose, row-major [K, M] (lda)
 * b_mn_major = 0: B is row-major [N, K] (ldb) (an nn.Linear weight); 1: row-major [K, N] (ldb)
 * The optional (A2,B2) pair extends the contraction by K2 (LoRA low-rank update fused into the same accumulator):
 *   a2_group_n > 0 : the A2 column offset for output tile column n0 is (n0 / a2_group_n) * K2 (per-adapter slices of a
 *                    packed u = [u_q|u_k|u_v]); 0 : offset 0.
 * splits > 1 splits the main contraction over CTAs; only valid with the fp32 atomic epilogues.
 * batch > 1 repeats the problem with per-batch element offsets (a_boff, b_boff, c_boff... applied as coordinates).
 *   An offset along K (a_boff_col of a K-major A, a_boff_row of an MN-major A, likewise for B) needs K % 64 == 0:
 *   otherwise the last k-block would read the next batch's elements instead of zeros, and the call fails with
 *   B2D_ERR_SHAPE.  (With only one operand offset along K the other's zero tail keeps finite data correct, but
 *   Inf/NaN in the neighbouring batch would still leak in, so those launches are refused as well.)
 * Alignment: every pointer is 16-byte aligned; lda, ldb, ldc2, ldres, ldaux, temb_stride are multiples of 8 elements,
 *   ldc and c_boff multiples of 8 (bf16 output) or 4 (fp32 output) elements; else B2D_ERR_ALIGN.
 * gate2_table needs gate2_temb, rows_per_sample > 0 and out2 (else B2D_ERR_ARG).
 * Replaces: every nn.Linear on the path (diffusers: LTXVideoTransformerBlock / Attention / FeedForward;
 *   finetrainers/patches/models/ltx_video/patch.py:82-85,118-123), peft: lora.Linear.forward, and their autograd
 *   backward (dX; LoRA dA/dB).
 * ------------------------------------------------------------------------------------------------------------- */
typedef enum {
  B2D_EPI_STORE = 0,        /* out(bf16) = alpha*acc + bias */
  B2D_EPI_GELU = 1,         /* pre = acc + bias; out2 = pre (optional); out = gelu_tanh(pre) */
  B2D_EPI_SILU = 2,         /* pre = acc + bias; out2 = pre (optional); out = silu(pre) */
  B2D_EPI_GATE_RES = 3,     /* out = res + gate[b,col] * (acc + bias); gate = gate_table[col] + gate_temb[b,col] or 1;
                               optional out2 = out * (gate2_table[col] + gate2_temb[b,col]) */
  B2D_EPI_MUL_DGELU = 4,    /* out = acc * gelu_tanh'(aux) */
  B2D_EPI_F32_ATOMIC = 5,   /* out_f32[row, col]  += alpha*acc   (split-K) */
  B2D_EPI_F32_ATOMIC_T = 6, /* out_f32[col, row]  += alpha*acc   (transposed accumulate) */
  B2D_EPI_F32_STORE = 7     /* out_f32[row, col]   = alpha*acc + bias */
} b2d_epilogue;

typedef struct {
  const void* A; int64_t lda;
  const void* B; int64_t ldb;
  const void* A2; int64_t lda2;
  const void* B2; int64_t ldb2;
  int32_t M, N, K, K2;
  int32_t a_mn_major, b_mn_major;
  int32_t a2_group_n;
  int32_t splits, batch;
  int64_t a_boff_row, a_boff_col, b_boff_row, b_boff_col, c_boff;  /* per-batch offsets (elements / rows / cols) */
  int32_t epi;
  float alpha;               /* multiplies the accumulator; set it explicitly (1.0f for a plain product; 0 yields zeros) */
  void* out; int64_t ldc;
  void* out2; int64_t ldc2;
  const void* bias;                 /* bf16 [N] or NULL */
  const void* res; int64_t ldres;   /* bf16 [M, N] */
  const void* aux; int64_t ldaux;   /* bf16 [M, N] */
  const void* gate_table;           /* bf16 [N]          (row of scale_shift_table) or NULL */
  const void* gate_temb;            /* bf16 [nb, temb_stride] (already offset to the gate row) or NULL */
  const void* gate2_table;
  const void* gate2_temb;
  int64_t temb_stride;
  int32_t rows_per_sample;          /* b = row / rows_per_sample */
  int32_t block_n;                  /* 0 = auto; else 64/128/160/192/256 */
  int32_t max_ctas;                 /* 0 = #SMs */
  /* batch offsets of the extension operands and of the bias (batch z reads A2 rows + z*a2_boff_row, B2 rows
   * + z*b2_boff_row, bias + z*bias_boff elements): one launch covers the same projection of several DiT blocks */
  int64_t a2_boff_row, b2_boff_row, bias_boff;
  /* tile scheduling across CTAs: 0 = auto (one CTA per tile), 1 = one CTA per 128 x block_n tile, 2 = CTA pairs: a 2-CTA
   * cluster computes a 256 x block_n tile, each CTA loading half of B and multicasting it to both (needs K-major A, no
   * split-K, block_n in 128/160/192/256, M > 128) */
  int32_t cta_pair;
} b2d_gemm_desc;

int b2d_gemm(const b2d_gemm_desc* d, void* stream);

/* Deterministic split-K for skinny GEMMs (N small, K long: the feed-forward LoRA launches u = s f A^T and du = s dwide B
 * at K = 4 D, N = padded rank).  The caller splits K into `splits` slices with b2d_gemm's batch offsets along K, each
 * slice writing B2D_EPI_F32_STORE (alpha 1) into part[z] of an fp32 workspace [splits, M, N] (contiguous, row stride N).
 * This call then writes
 *   out[m * ldc + c] = bf16_rn( alpha * (part[0, m, c] + part[1, m, c] + ... + part[splits - 1, m, c]) )
 * for m < M, c < N, adding the slices in slice order, so the output is the same on every run.  Nothing outside that
 * window of out is written: out may point at a column slice of a wider packed matrix.  part and out must not overlap.
 * Checks: part, out non-NULL and 1 <= splits <= B2D_SPLITK_MAX (else B2D_ERR_ARG); M > 0, N > 0, N % 8 == 0 and
 * ldc >= N (else B2D_ERR_SHAPE); part and out 16-byte aligned and ldc a multiple of 8 (else B2D_ERR_ALIGN).
 * Replaces: the same peft lora.Linear matmuls as b2d_gemm, for the two launches that would otherwise run one CTA per
 *   128-row tile over the whole 4 D contraction. */
#define B2D_SPLITK_MAX 16
int b2d_splitk_reduce_bf16(const float* part, int32_t splits, int32_t M, int32_t N, float alpha, void* out, int64_t ldc,
                           void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Fused RMSNorm / LayerNorm (no affine) + AdaLN modulate.   y = norm(x) * (1 + scale[b]) + shift[b]
 *   scale[b,c] = table[scale_row, c] + temb[b, scale_row*D + c]  (likewise shift); layer_norm=1 subtracts the mean.
 * Replaces: diffusers LTXVideoTransformerBlock norm1/norm2 + ada_values (and patch.py:113-120 norm_out + modulate);
 *   RMSNorm numerics finetrainers/patches/dependencies/diffusers/rms_norm.py:17-30.
 * bwd: dx_accum += d norm/dx ( dy * (1+scale) )   (adds into the residual-stream gradient; optional second output
 *   dx_scaled = dx_accum * gate2[b] for the next GEMM's A operand)
 * Row kernels: one row per 256-thread CTA; D must be a multiple of 8 and <= 8192.
 * Alignment (these and b2d_colscale): every pointer passed (x, y, dy, dx_in, dx_out, out, out2, tables, emb rows)
 *   16-byte aligned and emb_stride a multiple of 8 elements, else B2D_ERR_ALIGN before any launch.
 * bwd may run in place (dx_in == dx_out): every element is read before the same thread writes it.
 * ------------------------------------------------------------------------------------------------------------- */
int b2d_norm_modulate_fwd(const void* x, void* y, const void* shift_tab, const void* shift_emb, const void* scale_tab,
                          const void* scale_emb, int64_t emb_stride, int32_t rows, int32_t D, int32_t rows_per_sample,
                          float eps, int32_t layer_norm, void* stream);
/* dx_out = (accumulate ? dx_accum_in : 0) + dnorm(dy * (1 + scale)); optional out2 = dx_out * (gate2_tab + gate2_emb[b]) */
int b2d_norm_modulate_bwd(const void* dy, const void* x, const void* dx_in, void* dx_out, const void* scale_tab,
                          const void* scale_emb, const void* gate2_tab, const void* gate2_emb, void* out2,
                          int64_t emb_stride, int32_t rows, int32_t D, int32_t rows_per_sample, float eps,
                          int32_t layer_norm, void* stream);

/* out = x * (tab[c] + emb[b, c]) per column (gate application on the gradient path). */
int b2d_colscale(const void* x, void* out, const void* tab, const void* emb, int64_t emb_stride, int32_t rows,
                 int32_t D, int32_t rows_per_sample, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * q/k RMSNorm-across-heads (affine) + 3-D RoPE + head split.
 *   src [rows, ld] bf16 (q, k, v at column offsets) -> q',k',v' in [B, H, S, head_dim]; head_dim is 64 unless the entry
 *   point takes it.
 * rope cos/sin: fp32 [S, D/2], one value per rotary pair (NULL = no RoPE: cross attention).
 * Replaces: diffusers LTXVideoAttentionProcessor2_0 (norm_q/norm_k, apply_rotary_emb patch.py:23-33, unflatten+transpose).
 * ------------------------------------------------------------------------------------------------------------- */
int b2d_qknorm_rope_fwd(const void* src, int64_t ld, int64_t col_off, const void* weight, const void* cos,
                        const void* sin, void* dst, int32_t B, int32_t S, int32_t H, int32_t norm, float eps,
                        void* stream);
int b2d_qknorm_rope_bwd(const void* dsrc_heads, const void* x, int64_t ld, int64_t col_off, const void* weight,
                        const void* cos, const void* sin, void* dx, int64_t ld_dx, int64_t dx_col_off, int32_t B,
                        int32_t S, int32_t H, int32_t norm, float eps, void* stream);
/* Same, for nseg (1..3) consecutive D-wide column segments of one packed row in ONE launch (q|k|v of the fused QKV
 * projection; k|v of cross attention): segment i lives at col_off + i*D, is RMS-normed iff w_i != NULL, rotated iff bit i of
 * rope_mask is set, and is written head-split to dst_i.  The (cos, sin) row is read once for all segments.  The backward
 * reads the head-split upstream gradients dy_i and writes dx[row, dx_col_off + i*D + c].
 * rows_per_w > 0: the rows are several DiT blocks stacked (B = blocks * batch); row r then uses the norm weights
 * w_i + (r / rows_per_w) * w_stride (elements) - the text-side k|v of all blocks in one launch.
 * Checks (all four q/k entry points): dst_i / dy_i non-NULL for every i < nseg and rope_mask < 2^nseg (else
 * B2D_ERR_ARG); src / x, dst_i / dy_i, w_i, dx, cos and sin 16-byte aligned, ld, col_off, ld_dx, dx_col_off and
 * w_stride multiples of 8 elements (else B2D_ERR_ALIGN). */
int b2d_qkv_norm_rope_fwd(const void* src, int64_t ld, int64_t col_off, int32_t nseg, const void* w0, const void* w1,
                          const void* w2, int32_t rope_mask, const void* cos, const void* sin, void* dst0, void* dst1,
                          void* dst2, int32_t B, int32_t S, int32_t H, float eps, int32_t rows_per_w, int64_t w_stride,
                          void* stream);
int b2d_qkv_norm_rope_bwd(const void* dy0, const void* dy1, const void* dy2, const void* x, int64_t ld, int64_t col_off,
                          int32_t nseg, const void* w0, const void* w1, const void* w2, int32_t rope_mask, const void* cos,
                          const void* sin, void* dx, int64_t ld_dx, int64_t dx_col_off, int32_t B, int32_t S, int32_t H,
                          float eps, int32_t rows_per_w, int64_t w_stride, void* stream);
/* The same two with the head dimension as an argument: head_dim 64 or 128 (else B2D_ERR_SHAPE), D = H * head_dim.  With
 * head_dim = 64 they are the two entry points above. */
int b2d_qkv_norm_rope_hd_fwd(const void* src, int64_t ld, int64_t col_off, int32_t nseg, const void* w0, const void* w1,
                             const void* w2, int32_t rope_mask, const void* cos, const void* sin, void* dst0, void* dst1,
                             void* dst2, int32_t B, int32_t S, int32_t H, int32_t head_dim, float eps, int32_t rows_per_w,
                             int64_t w_stride, void* stream);
int b2d_qkv_norm_rope_hd_bwd(const void* dy0, const void* dy1, const void* dy2, const void* x, int64_t ld,
                             int64_t col_off, int32_t nseg, const void* w0, const void* w1, const void* w2,
                             int32_t rope_mask, const void* cos, const void* sin, void* dx, int64_t ld_dx,
                             int64_t dx_col_off, int32_t B, int32_t S, int32_t H, int32_t head_dim, float eps,
                             int32_t rows_per_w, int64_t w_stride, void* stream);
/* The same two with per-head RoPE: the cos / sin tables are fp32 [S, head_dim/2], one value per rotary pair (2i, 2i+1)
 * of a head and the same for every head; column c of a segment reads pair (c mod head_dim) / 2.  Arguments, checks
 * and everything else as the _hd entry points, which keep their own instantiations.
 * Replaces (per head): diffusers WanAttnProcessor2_0's norm_q / norm_k, unflatten + transpose and apply_rotary_emb. */
int b2d_qkv_norm_rope_ph_fwd(const void* src, int64_t ld, int64_t col_off, int32_t nseg, const void* w0, const void* w1,
                             const void* w2, int32_t rope_mask, const void* cos, const void* sin, void* dst0, void* dst1,
                             void* dst2, int32_t B, int32_t S, int32_t H, int32_t head_dim, float eps, int32_t rows_per_w,
                             int64_t w_stride, void* stream);
int b2d_qkv_norm_rope_ph_bwd(const void* dy0, const void* dy1, const void* dy2, const void* x, int64_t ld,
                             int64_t col_off, int32_t nseg, const void* w0, const void* w1, const void* w2,
                             int32_t rope_mask, const void* cos, const void* sin, void* dx, int64_t ld_dx,
                             int64_t dx_col_off, int32_t B, int32_t S, int32_t H, int32_t head_dim, float eps,
                             int32_t rows_per_w, int64_t w_stride, void* stream);

/* RoPE table (diffusers LTXVideoRotaryPosEmbed.forward, called at patch.py:52): fp32 cos,sin [F*H*W, D/2]
 * (the reference's repeat_interleave(2) duplicates are not stored).  F, H, W must be positive (else B2D_ERR_SHAPE). */
int b2d_rope_table(float* cos, float* sin, int32_t F, int32_t H, int32_t W, int32_t D, float sf, float sh, float sw,
                   void* stream);

/* Wan RoPE table (diffusers WanRotaryPosEmbed, patch (1, 2, 2) already applied to the grid): fp32 cos, sin
 *   [F*H*W, head_dim/2].  The head splits into t / h / w parts of head_dim - 4*(head_dim/6), 2*(head_dim/6), 2*(head_dim/6)
 *   dims (44 / 42 / 42 at 128); pair i of a part of n dims at integer grid position p along its axis rotates by
 *   p * theta^(-2i/n), computed in float64 (freqs_dtype=torch.float64) and rounded once to fp32.  cos, sin non-NULL (else
 *   B2D_ERR_ARG); head_dim even and >= 6, F, H, W positive (else B2D_ERR_SHAPE).  The engine applies the rotation in fp32
 *   where diffusers applies it in float64. */
int b2d_rope_table_wan(float* cos, float* sin, int32_t F, int32_t H, int32_t W, int32_t head_dim, double theta,
                       void* stream);

/* Affine LayerNorm (diffusers FP32LayerNorm with weight and bias: Wan's cross-attention pre-norm norm2): fp32 statistics,
 *   weight and bias bf16 [D] upcast to fp32, y = bf16((x - mean) * rstd * weight + bias).
 * bwd: dx_out = (dx_in or 0) + d layer_norm / dx (dy), no weight or bias gradient (frozen under LoRA); optional
 *   out2 = bf16(dx_out) * (gate2_tab[c] + gate2_emb[b, c]) as b2d_norm_modulate_bwd (out2 needs both gate pointers, else
 *   B2D_ERR_ARG).  In place allowed (dx_in == dx_out).  Shapes and alignment as the norm + modulate row kernels; x, y,
 *   weight, bias, dy, dx_out non-NULL (else B2D_ERR_ARG).
 * Replaces: diffusers WanTransformerBlock norm2 (cross_attn_norm=True) and its autograd backward. */
int b2d_layer_norm_affine_fwd(const void* x, void* y, const void* weight, const void* bias, int32_t rows, int32_t D,
                              float eps, void* stream);
int b2d_layer_norm_affine_bwd(const void* dy, const void* x, const void* dx_in, void* dx_out, const void* weight,
                              const void* gate2_tab, const void* gate2_emb, void* out2, int64_t emb_stride, int32_t rows,
                              int32_t D, int32_t rows_per_sample, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Attention, head_dim 64 or 128, non-causal, optional additive key bias [B, Sk] (fp32; the -10000 mask bias of
 * patch.py:55-57).
 *   q [B,H,Sq,head_dim], k,v [B,H,Sk,head_dim] bf16 -> out [B,Sq,H*head_dim] bf16 (token-major, feeds to_out directly),
 *   lse [B,H,Sq] fp32.  Any other head_dim returns B2D_ERR_SHAPE.
 * Key-bias values are -inf (a masked key) or finite with |bias| * log2(e) < FLT_MAX.  A row whose keys are all -inf
 *   gets out = 0, lse = +inf and zero gradients.  The backward rebuilds P as exp(score + bias - lse), so lse must keep
 *   the scores: if a sample's largest bias is so negative that it absorbs them in fp32 (every key at -1e9, say), the
 *   forward is the mean of V but the gradients are wrong by orders of magnitude and can overflow.  Callers shift each
 *   sample's bias so that its largest finite value is 0 (softmax is unchanged), and mask a key with -inf, not with a
 *   huge finite value; the attention provider does both (attention.py, mask_to_key_bias).
 * Replaces: F.scaled_dot_product_attention == finetrainers/models/attention_dispatch.py:405-447 -> _native_attention
 *   :938-962, and its backward.
 * ------------------------------------------------------------------------------------------------------------- */
int b2d_attn_fwd_hd(const void* q, const void* k, const void* v, const float* key_bias, void* out, float* lse,
                    int32_t B, int32_t H, int32_t Sq, int32_t Sk, int32_t head_dim, float scale, void* stream);
/* dout [B,Sq,H*head_dim] bf16; out as produced by fwd; dq,dk,dv [B,H,S,head_dim] bf16; workspace delta_ws:
 * 2*B*H*Sq floats, plus 8*2*B*H*Sk*head_dim floats when Sk <= 512 (fp32 partial dV/dK of up to 8 query ranges, summed
 * in a fixed order so that the gradients are the same on every run; the caller only provides the space). */
int b2d_attn_bwd_hd(const void* q, const void* k, const void* v, const float* key_bias, const void* out,
                    const void* dout, const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int32_t B,
                    int32_t H, int32_t Sq, int32_t Sk, int32_t head_dim, float scale, void* stream);
/* Two-context attention: q attends to context 1 (k1, v1 [B,H,Sk1,head_dim]) and to context 2 (k2, v2 [B,H,Sk2,head_dim])
 *   with two independent softmaxes, no key bias, in ONE launch (one CTA per 128-query tile and (b, h), Q loaded once,
 *   context 1's key tiles then context 2's through one ring):
 *     out = bf16(float(bf16(O1)) + float(bf16(O2))) [B,Sq,H*head_dim],  lse1, lse2 [B,H,Sq] fp32.
 *   out1 / out2 (optional, NULL to skip) receive bf16(O1) and bf16(O2).  lse1 and bf16(O1) are bit-identical to
 *   b2d_attn_fwd_hd(q, k1, v1, NULL, ...), lse2 and bf16(O2) to b2d_attn_fwd_hd(q, k2, v2, NULL, ...).  head_dim 64 or 128
 *   and positive sizes (else B2D_ERR_SHAPE); q, k1, v1, k2, v2, out, lse1, lse2 non-NULL (else B2D_ERR_ARG); out, out1,
 *   out2 32-byte aligned (else B2D_ERR_ALIGN).
 * Replaces: diffusers WanAttnProcessor2_0 with add_k_proj (image-to-video cross attention): the text and image
 *   F.scaled_dot_product_attention calls and `hidden_states + hidden_states_img`. */
int b2d_attn_dual_fwd_hd(const void* q, const void* k1, const void* v1, int32_t Sk1, const void* k2, const void* v2,
                         int32_t Sk2, void* out, float* lse1, float* lse2, void* out1, void* out2, int32_t B, int32_t H,
                         int32_t Sq, int32_t head_dim, float scale, void* stream);
/* Its backward for a caller that trains context 1's keys and values but not context 2's: dq (both contexts, accumulated
 *   in one fp32 accumulator and rounded once) and dk1, dv1; no dK2 / dV2.  out1, out2 are the branch outputs the
 *   forward wrote, dout the gradient of out (it reaches both branches unchanged).  dk1 and dv1 are bit-identical to
 *   b2d_attn_bwd_hd(q, k1, v1, NULL, out1, dout, lse1, ...): the same delta and dK / dV launches.  dQ is one launch that
 *   streams context 1's key tiles, then context 2's, switching the row terms (-lse log2e, delta) at the boundary.
 *   Workspace ws: W1 + 2*B*H*Sq floats, W1 = b2d_attn_bwd_hd's for (Sq, Sk1) = 2*B*H*Sq plus 8*2*B*H*Sk1*head_dim when
 *   Sk1 <= 512; context 2's delta and -lse log2e sit after W1.  Checks as the forward; every pointer non-NULL.
 * Replaces: the autograd backward of the two scaled_dot_product_attention calls of WanAttnProcessor2_0 with add_k_proj
 *   when add_k_proj / add_v_proj are frozen (dQ summed over both contexts; no image key / value gradient). */
int b2d_attn_dual_bwd_hd(const void* q, const void* k1, const void* v1, int32_t Sk1, const void* k2, const void* v2,
                         int32_t Sk2, const void* out1, const void* out2, const void* dout, const float* lse1,
                         const float* lse2, float* ws, void* dq, void* dk1, void* dv1, int32_t B, int32_t H, int32_t Sq,
                         int32_t head_dim, float scale, void* stream);
/* head_dim = 64 forms of the two above (workspace 2*B*H*Sq floats, plus 8*2*B*H*Sk*64 when Sk <= 512). */
int b2d_attn_fwd(const void* q, const void* k, const void* v, const float* key_bias, void* out, float* lse, int32_t B,
                 int32_t H, int32_t Sq, int32_t Sk, float scale, void* stream);
int b2d_attn_bwd(const void* q, const void* k, const void* v, const float* key_bias, const void* out, const void* dout,
                 const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int32_t B, int32_t H, int32_t Sq,
                 int32_t Sk, float scale, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Step prologue / epilogue.
 * prep: normalise latents, x_t = (1-sigma) x0 + sigma n (first latent frame may use sigma_ff[b]), pack [B,C,F,H,W] ->
 *   [B, F*H*W, C]; target = n - x0 (packed).   finetrainers/models/ltx_video/base_specification.py:285-322,343,427-459;
 *   finetrainers/functional/diffusion.py:4-11.
 * loss: loss = mean_b( mean_{s,c}( w[b] * (pred - target)^2 ) ) * loss_scale  (fp32);  dpred = dloss/dpred (bf16).
 *   finetrainers/trainer/sft_trainer/trainer.py:463-481.
 *   weight NULL: every w[b] = 1;  dpred NULL: only the loss.  B > 0, per_sample > 0 and a multiple of 8 (else
 *   B2D_ERR_SHAPE); pred, target, dpred 16-byte aligned (else B2D_ERR_ALIGN).
 * partial_ws (loss and b2d_sumsq): fp32 scratch of B2D_REDUCE_PARTIALS = 296 floats (one per reduction block); the
 *   calls write exactly those and nothing beyond.
 * ------------------------------------------------------------------------------------------------------------- */
#define B2D_REDUCE_PARTIALS 296
int b2d_prep_noise_pack(const void* latents, const void* noise, const float* mean, const float* std,
                        const float* sigma, const float* sigma_ff, void* x_t, void* target, int32_t B, int32_t C,
                        int32_t F, int32_t HW, void* stream);
/* prep from VAE moments (training on precomputed moments, the reference's compute_posterior=False): moments bf16
 *   [B, 2C, F*HW] = [mean | logvar], eps bf16 [B, C, F*HW] (the caller's standard-normal draw).  The latent is sampled as
 *   x = mean + exp(0.5 * clamp(logvar, -30, 20)) * eps with each step rounded to bf16 as the reference's bf16 tensor ops
 *   round (finetrainers/models/utils.py:8-31; NaN logvar gives NaN x), then normalised, noised, packed and targeted
 *   exactly as b2d_prep_noise_pack does with latents = x.  latents_out NULL, or bf16 [B, C, F*HW] to receive x.
 *   B, C, F, HW must be positive (else B2D_ERR_SHAPE).  One launch. */
int b2d_prep_posterior_noise_pack(const void* moments, const void* eps, const void* noise, const float* mean,
                                  const float* std, const float* sigma, const float* sigma_ff, void* x_t, void* target,
                                  void* latents_out, int32_t B, int32_t C, int32_t F, int32_t HW, void* stream);
/* Wan step prologue (finetrainers/models/wan/base_specification.py:446-475 with compute_posterior forced False, and
 *   :571-576, finetrainers/models/utils.py:8-31, finetrainers/functional/diffusion.py:4-11), one launch.  moments bf16
 *   [B, 2C, F, H, W] = [mean | logvar], eps and noise bf16 [B, C, F, H, W] (eps drawn before the noise), mean and std fp32
 *   [B, C] (std is already 1 / latents_std), sigma fp32 [B].  Per element, rounding as the reference's tensor ops:
 *     mu, lv = bf16((v - mean) * std) of each half;  x = mu + exp(0.5 clamp(lv, -30, 20)) * eps, every op rounded to bf16;
 *     x_t = bf16((1 - sigma) x + sigma n);  target = bf16(n - x).
 *   x_t is written patchified for patch (1, 2, 2): [B, F (H/2) (W/2), 4C] with k = c*4 + kh*2 + kw (the Conv3d weight
 *   [D, C, 1, 2, 2] viewed as [D, 4C]); target in proj_out's layout, k = (kh*2 + kw)*C + c.  Non-NULL operands (else
 *   B2D_ERR_ARG); B, C, F, H, W positive and H, W even (else B2D_ERR_SHAPE). */
int b2d_wan_prep(const void* moments, const void* eps, const void* noise, const float* mean, const float* std,
                 const float* sigma, void* x_t, void* target, int32_t B, int32_t C, int32_t F, int32_t H, int32_t W,
                 void* stream);
/* Wan image-to-video step prologue: b2d_wan_prep plus the conditioning channels (finetrainers/models/wan/
 *   base_specification.py:446-483, compute_posterior forced False).  cond_moments bf16 [B, 2C, F, H, W] = [mean | logvar]
 *   of the conditioning video, cond_mask bf16 [B, Cm, F, H, W] (WanImageConditioningLatentEncodeProcessor's mask), other
 *   operands as b2d_wan_prep.  x_in [B, F (H/2) (W/2), 4 (2C + Cm)] is the transformer input cat([x_t, mask, condition],
 *   dim=1) patchified in the Conv3d order, k = ch*4 + kh*2 + kw over the 2C + Cm concatenated channels, with
 *     condition = bf16((cond_mean - mean) * std)   (DiagonalGaussianDistribution.mode() of the normalised condition: no
 *                                                    random draw; its logvar is not read)
 *   x_t and target are bit-identical to b2d_wan_prep's on the same inputs.  Non-NULL operands (else B2D_ERR_ARG);
 *   B, C, Cm, F, H, W positive, Cm <= C, H, W even (else B2D_ERR_SHAPE).  Every operand is a dense array (the reference
 *   builds its mask as a transposed view: pass a contiguous copy).  One launch. */
int b2d_wan_i2v_prep(const void* moments, const void* cond_moments, const void* cond_mask, const void* eps,
                     const void* noise, const float* mean, const float* std, const float* sigma, void* x_in, void* target,
                     int32_t B, int32_t C, int32_t Cm, int32_t F, int32_t H, int32_t W, void* stream);
/* Exact (erf) GELU on n bf16 elements: y = bf16(0.5 x (1 + erf(x / sqrt(2)))) in fp32.  x == y allowed; n <= 0 is a
 *   no-op; x, y non-NULL (else B2D_ERR_ARG).  Applied to the bf16 output of a B2D_EPI_STORE GEMM, where nn.Linear and
 *   F.gelu round.
 * Replaces: diffusers WanImageEmbedding's FeedForward activation (activation_fn="gelu": F.gelu, approximate="none"). */
int b2d_gelu_erf(const void* x, void* y, int64_t n, void* stream);
/* Exact bf16 permute between [B, C, F, H, W] and the patchified [B, F (H/2) (W/2), 4C]: unpatchify = 0 packs, 1 unpacks;
 *   out_order = 0 uses the Conv3d order k = c*4 + kh*2 + kw, 1 proj_out's k = (kh*2 + kw)*C + c.  src != dst and both
 *   non-NULL, flags 0 or 1 (else B2D_ERR_ARG); sizes as b2d_wan_prep (else B2D_ERR_SHAPE).
 * Replaces: diffusers WanTransformer3DModel's Conv3d input patching (as a reorder: the projection is a GEMM) and the
 *   reshape / permute / flatten unpatchify of its output. */
int b2d_patch_permute(const void* src, void* dst, int32_t B, int32_t C, int32_t F, int32_t H, int32_t W,
                      int32_t out_order, int32_t unpatchify, void* stream);
int b2d_loss_mse(const void* pred, const void* target, const float* weight, float loss_scale, float* loss_out,
                 void* dpred, float* partial_ws, int32_t B, int64_t per_sample, void* stream);

/* sinusoidal timestep features (diffusers Timesteps(256, flip_sin_to_cos=True)): out bf16 [n, 256] = [cos | sin]. */
int b2d_timestep_sinusoid(const float* t, void* out, int32_t n, void* stream);

/* fp32 -> bf16 cast with scale (LoRA operand refresh each step).  n <= 0 is a no-op; src 16-byte and dst 8-byte aligned
 * (else B2D_ERR_ALIGN).  timestep_sinusoid with n <= 0 is a no-op too. */
int b2d_cast_f32_bf16(const float* src, void* dst, int64_t n, float scale, void* stream);

/* fp8 -> bf16 upcast of n stored weight codes (layerwise casting: frozen base weights stored in fp8, materialised in bf16
 * one DiT block ahead of compute).  fmt 0 = float8_e4m3fn, 1 = float8_e5m2 (else B2D_ERR_ARG).  Every code converts
 * exactly (bit-identical to torch's .to(torch.bfloat16) for finite codes, +-0 and +-Inf kept, NaN stays NaN).  Any n;
 * n <= 0 is a no-op.  src and dst 16-byte aligned (else B2D_ERR_ALIGN).
 * Replaces: diffusers' layerwise-casting pre-forward hook (module.to(compute_dtype)) applied by
 *   finetrainers/trainer/sft_trainer/trainer.py:108-118. */
int b2d_upcast_fp8_bf16(const void* src, void* dst, int64_t n, int32_t fmt, void* stream);

/* One denoising step of the validation sampler: classifier-free guidance + the flow-match Euler update, in one launch.
 *   guided != 0: pred bf16 [2B, n] = [uncond; cond] (torch.cat([negative, positive]) order), x_next bf16 [2B, n];
 *   guided == 0 (no guidance; guidance is not read): pred and x_next [B, n].  The caller decides, as it built the batch
 *   (LTXPipeline: do_classifier_free_guidance = guidance_scale > 1 in double precision; guidance then enters the
 *   arithmetic rounded to fp32, as torch's fp32 scalar ops take it).  latents fp32 [B, n] is updated in place.  dt: one fp32 in device
 *   memory (sigma_next - sigma), so a captured CUDA graph replays every step.  Per element, rounding as the pipeline's
 *   fp32 tensor ops round (no FMA contraction):
 *     v = u + guidance * (c - u)   (v = the prediction without guidance; u, c the bf16 predictions upcast to fp32)
 *     x' = x + dt * v;   latents = x';   every row block of x_next = bf16_rn(x')  (the next step's input)
 *   NaN and Inf propagate as in fp32 arithmetic.  Checks: pred, latents, x_next, dt non-NULL (else B2D_ERR_ARG); B > 0,
 *   n > 0 (else B2D_ERR_SHAPE); pred, latents, x_next 16-byte aligned (else B2D_ERR_ALIGN).  Nothing outside the
 *   listed extents is written.
 * Replaces: diffusers LTXPipeline.__call__'s guidance arithmetic (noise_pred.float(), chunk(2), u + g (c - u)),
 *   FlowMatchEulerDiscreteScheduler.step (sample + (sigma_next - sigma) * model_output) and the next step's
 *   torch.cat([latents] * 2).to(bf16); called by the transformer-only half of SFTTrainer._validate
 *   (finetrainers/trainer/sft_trainer/trainer.py:583-700). */
int b2d_cfg_euler_step(const void* pred, float* latents, void* x_next, int32_t B, int64_t n, int32_t guided,
                       float guidance, const float* dt, void* stream);

/* One denoising step of the image-to-video sampler: b2d_cfg_euler_step on the elements e of each sample with
 * e >= n_cond (e counted within the sample's n elements), with the same layouts, arguments and per-element arithmetic.
 * The first n_cond elements of each sample (the conditioning frame: n_cond = H W C of packed [B, F H W, C] latents) are
 * left alone: pred is not read there, and latents and every row block of x_next are not written there, so they keep
 * the frozen latents and their bf16 copy.  128-bit accesses where n % 8 == 0 (from the first multiple of 8 at or after
 * n_cond in each sample), element by element elsewhere.  Checks as b2d_cfg_euler_step, and 0 <= n_cond < n (else
 * B2D_ERR_SHAPE).
 * Replaces: diffusers LTXImageToVideoPipeline.__call__'s denoising loop body after the transformer call: guidance on
 *   noise_pred.float(), scheduler.step(noise_pred[:, :, 1:], t, latents[:, :, 1:]) on the unpacked latents,
 *   torch.cat([latents[:, :, :1], pred_latents], 2) and the next step's torch.cat([latents] * 2).to(bf16). */
int b2d_cfg_euler_step_cond(const void* pred, float* latents, void* x_next, int32_t B, int64_t n, int64_t n_cond,
                            int32_t guided, float guidance, const float* dt, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Flat-buffer optimiser path ("next" row: clip + AdamW; finetrainers/utils/torch.py:99-161, optimizer.py:117-125).
 * ------------------------------------------------------------------------------------------------------------- */
/* x 16-byte aligned (else B2D_ERR_ALIGN); partial_ws: B2D_REDUCE_PARTIALS floats. */
int b2d_sumsq(const float* x, int64_t n, float* out_sumsq /* += */, float* partial_ws, void* stream);
/* p, g, m, v: 16-byte aligned (any n; four elements per thread as 128-bit accesses); g is zeroed (fused zero_grad).
 * The applied gradient is g * grad_div * min(1, max_norm / (sqrt(*sumsq) * grad_div + 1e-6)); max_norm <= 0 turns
 * clipping off and sumsq is then not read. */
int b2d_adamw_clip(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq, float max_norm, float lr,
                   float beta1, float beta2, float eps, float wd, int32_t step, float grad_div, void* stream);

#ifdef __cplusplus
}
#endif
#endif
