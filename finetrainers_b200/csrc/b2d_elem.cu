// b2d_elem.cu — the HBM-bound satellites of the DiT step: fused norm+AdaLN modulate (fwd/bwd), q/k RMSNorm + RoPE +
// head split (fwd/bwd), RoPE table, noise/pack prologue, MSE loss + dpred, sinusoid, casts, flat clip + AdamW, and the
// sampler's guided Euler step.
// All: 128-bit coalesced global access, fp32 math, warp-shuffle reductions; one row per CTA of 256 threads.
#include <algorithm>
#include <initializer_list>

#include <cuda_fp16.h>

#include "b2d_internal.h"
#include "b2d_ptx.cuh"

namespace b2d {

constexpr int ROW_THREADS = 256;
constexpr int MAX_CHUNKS = 4;  // D <= 8 * 256 * 4 = 8192

__device__ __forceinline__ uint4 ldg16(const void* p) { return *reinterpret_cast<const uint4*>(p); }
__device__ __forceinline__ void stg16(void* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }

__device__ __forceinline__ void unpack8(uint4 u, float (&f)[8]) {
    f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
    f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// block-wide sum of up to two values; all threads get the result
__device__ __forceinline__ float2 block_sum2(float a, float b) {
    __shared__ float sa[ROW_THREADS / 32], sb[ROW_THREADS / 32];
    __shared__ float ra, rb;
    a = warp_sum(a);
    b = warp_sum(b);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();  // protect sa/sb/ra/rb reuse across consecutive calls
    if (l == 0) { sa[w] = a; sb[w] = b; }
    __syncthreads();
    if (w == 0) {
        float x = l < ROW_THREADS / 32 ? sa[l] : 0.f;
        float y = l < ROW_THREADS / 32 ? sb[l] : 0.f;
        x = warp_sum(x);
        y = warp_sum(y);
        if (l == 0) { ra = x; rb = y; }
    }
    __syncthreads();
    return make_float2(ra, rb);
}

// ------------------------------------------------------------------------------------------------
// norm + modulate
// ------------------------------------------------------------------------------------------------
// Every global operand of a row is requested BEFORE the first block reduction: a row's critical path is then one memory
// round trip + the reductions instead of two or three dependent round trips (these kernels have ~16 KB in flight per
// CTA and 8 CTAs per SM, so the dependent-latency chain, not bandwidth, was what bounded them).
// AFFINE: an affine LayerNorm (diffusers FP32LayerNorm with weight and bias): y = norm(x) * scale_tab + shift_tab, the
// emb rows are not read.  AFFINE = false is the modulated form.
template <int NCH, bool AFFINE = false>
__global__ void __launch_bounds__(ROW_THREADS) norm_modulate_fwd_kernel(
    const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ shift_tab,
    const __nv_bfloat16* __restrict__ shift_emb, const __nv_bfloat16* __restrict__ scale_tab,
    const __nv_bfloat16* __restrict__ scale_emb, long long emb_stride, int D, int rows_per_sample, float eps,
    int layer_norm) {
    griddep_launch_dependents();
    griddep_wait();
    const int row = blockIdx.x;
    const int b = row / rows_per_sample;
    const __nv_bfloat16* xr = x + (long long)row * D;
    uint4 xq[NCH], q_sht[NCH], q_she[NCH], q_sct[NCH], q_sce[NCH];
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
            xq[c] = ldg16(xr + col);
            q_sht[c] = ldg16(shift_tab + col);
            q_sct[c] = ldg16(scale_tab + col);
            if (!AFFINE) {
                q_she[c] = ldg16(shift_emb + (long long)b * emb_stride + col);
                q_sce[c] = ldg16(scale_emb + (long long)b * emb_stride + col);
            }
        }
    }
    float v[NCH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
            unpack8(xq[c], v[c]);
#pragma unroll
            for (int e = 0; e < 8; ++e) { s1 += v[c][e]; s2 += v[c][e] * v[c][e]; }
        }
    }
    float2 tot = block_sum2(s1, s2);
    float mean = 0.f, rstd;
    if (layer_norm) {
        mean = tot.x / D;
        float var = 0.f;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            const int col = (c * ROW_THREADS + threadIdx.x) * 8;
            if (col < D) {
#pragma unroll
                for (int e = 0; e < 8; ++e) { float d = v[c][e] - mean; var += d * d; }
            }
        }
        float2 t2 = block_sum2(var, 0.f);
        rstd = rsqrtf(t2.x / D + eps);
    } else {
        rstd = rsqrtf(tot.y / D + eps);
    }
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
            float sh[8], sc[8], t[8];
            float o[8];
            unpack8(q_sht[c], sh);
            unpack8(q_sct[c], sc);
            if (AFFINE) {
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = (v[c][e] - mean) * rstd * sc[e] + sh[e];
            } else {
                unpack8(q_she[c], t);
#pragma unroll
                for (int e = 0; e < 8; ++e) sh[e] += t[e];
                unpack8(q_sce[c], t);
#pragma unroll
                for (int e = 0; e < 8; ++e) sc[e] += t[e];
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = (v[c][e] - mean) * rstd * (1.f + sc[e]) + sh[e];
            }
            stg16(y + (long long)row * D + col, pack8(o));
        }
    }
}

// AFFINE: the backward of the affine LayerNorm: g = dy * scale_tab (the weight), scale_emb not read.
template <int NCH, bool AFFINE = false>
__global__ void __launch_bounds__(ROW_THREADS) norm_modulate_bwd_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dx_in,
    __nv_bfloat16* __restrict__ dx_out, const __nv_bfloat16* __restrict__ scale_tab,
    const __nv_bfloat16* __restrict__ scale_emb, const __nv_bfloat16* __restrict__ gate2_tab,
    const __nv_bfloat16* __restrict__ gate2_emb, __nv_bfloat16* __restrict__ out2, long long emb_stride, int D,
    int rows_per_sample, float eps, int layer_norm) {
    griddep_launch_dependents();
    griddep_wait();
    const int row = blockIdx.x;
    const int b = row / rows_per_sample;
    const long long ro = (long long)row * D;
    uint4 q_x[NCH], q_dy[NCH], q_sct[NCH], q_sce[NCH], q_in[NCH], q_gt[NCH], q_ge[NCH];
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
            q_x[c] = ldg16(x + ro + col);
            q_dy[c] = ldg16(dy + ro + col);
            q_sct[c] = ldg16(scale_tab + col);
            if (!AFFINE) q_sce[c] = ldg16(scale_emb + (long long)b * emb_stride + col);
            q_in[c] = dx_in != nullptr ? ldg16(dx_in + ro + col) : make_uint4(0, 0, 0, 0);
            if (out2 != nullptr) {
                q_gt[c] = ldg16(gate2_tab + col);
                q_ge[c] = ldg16(gate2_emb + (long long)b * emb_stride + col);
            }
        }
    }
    float xv[NCH][8], g[NCH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
            unpack8(q_x[c], xv[c]);
#pragma unroll
            for (int e = 0; e < 8; ++e) { s1 += xv[c][e]; s2 += xv[c][e] * xv[c][e]; }
        }
    }
    float2 tot = block_sum2(s1, s2);
    float mean = 0.f, rstd;
    if (layer_norm) {
        mean = tot.x / D;
        float var = 0.f;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            const int col = (c * ROW_THREADS + threadIdx.x) * 8;
            if (col < D) {
#pragma unroll
                for (int e = 0; e < 8; ++e) { float d = xv[c][e] - mean; var += d * d; }
            }
        }
        rstd = rsqrtf(block_sum2(var, 0.f).x / D + eps);
    } else {
        rstd = rsqrtf(tot.y / D + eps);
    }
    // g = dy * (1 + scale);  xhat = (x - mean) * rstd;  a = sum(g), c = sum(g * xhat)
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
            float sc[8], t[8], d[8];
            unpack8(q_sct[c], sc);
            unpack8(q_dy[c], d);
            if (!AFFINE) unpack8(q_sce[c], t);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                g[c][e] = AFFINE ? d[e] * sc[e] : d[e] * (1.f + sc[e] + t[e]);
                xv[c][e] = (xv[c][e] - mean) * rstd;
                sg += g[c][e];
                sgx += g[c][e] * xv[c][e];
            }
        }
    }
    float2 t2 = block_sum2(sg, sgx);
    const float mg = layer_norm ? t2.x / D : 0.f;
    const float mgx = t2.y / D;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
            float o[8];
            unpack8(q_in[c], o);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] += rstd * (g[c][e] - mg - xv[c][e] * mgx);
            uint4 packed = pack8(o);
            stg16(dx_out + ro + col, packed);
            if (out2 != nullptr) {
                float r[8], gt[8], ge[8];
                unpack8(packed, r);  // the rounded value is what downstream sees
                unpack8(q_gt[c], gt);
                unpack8(q_ge[c], ge);
#pragma unroll
                for (int e = 0; e < 8; ++e) r[e] *= (gt[e] + ge[e]);
                stg16(out2 + ro + col, pack8(r));
            }
        }
    }
}

__global__ void colscale_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                const __nv_bfloat16* __restrict__ tab, const __nv_bfloat16* __restrict__ emb,
                                long long emb_stride, long long total8, int D, int rows_per_sample) {
    griddep_launch_dependents();
    griddep_wait();
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total8) return;
    long long e0 = i * 8;
    int row = (int)(e0 / D);
    int col = (int)(e0 % D);
    int b = row / rows_per_sample;
    float v[8], t[8], g[8];
    unpack8(ldg16(x + e0), v);
    unpack8(ldg16(tab + col), t);
    unpack8(ldg16(emb + (long long)b * emb_stride + col), g);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] *= (t[e] + g[e]);
    stg16(out + e0, pack8(v));
}

// ------------------------------------------------------------------------------------------------
// q/k RMSNorm (affine, across all heads) + RoPE + head split for up to three column segments of one packed row
// (q | k | v of the fused QKV projection, or k | v of cross attention):  src[row, col_off + i*D + c] -> dst_i[b, h, s, d].
// One CTA handles all segments of its row: the (cos, sin) row is read once for q AND k, every global operand is
// requested before the first reduction, and the two RMS statistics share one block reduction.
// HD is the head dimension (64 or 128): it only sets where a column lands in the head-split tensor, and a thread's 8
// consecutive columns never straddle a head for either value.  The RMS statistic stays over all D = H * HD columns.
// ------------------------------------------------------------------------------------------------
struct QkvSegArgs {
    const __nv_bfloat16* w[3];   // RMSNorm weight of segment i, or null: no norm
    __nv_bfloat16* dst[3];       // fwd: head-split outputs;  bwd: head-split upstream gradients (read)
    int nseg;
    int rope_mask;               // bit i: segment i is rotated
    int rows_per_w;              // > 0: rows are stacked DiT blocks, row r uses weights w[i] + (r / rows_per_w) * w_stride
    long long w_stride;
};

// PH (per-head RoPE): the tables are [S, HD/2], one (cos, sin) per rotary pair of a head, the same for every head (Wan's
// rotary embedding); otherwise [S, D/2] over the full width (LTX-Video's).  The row bodies are shared by two kernels
// per direction: qkv_norm_rope_*_kernel (PH = false) and per_head_rope_qk_norm_*_kernel (PH = true).
template <int NCH, int HD, bool PH>
__device__ __forceinline__ void qkv_norm_rope_fwd_row(
    const __nv_bfloat16* __restrict__ src, long long ld, long long col_off, const QkvSegArgs a,
    const float* __restrict__ cosT, const float* __restrict__ sinT, int S, int H, float eps) {
    const int D = H * HD;
    const int row = blockIdx.x;
    const int b = row / S, s = row % S;
    const __nv_bfloat16* xr = src + (long long)row * ld + col_off;
    const long long woff = a.rows_per_w > 0 ? (long long)(row / a.rows_per_w) * a.w_stride : 0;
    uint4 xq[3][NCH], wq[3][NCH];
    float4 c4[NCH], s4[NCH];
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                if (i < a.nseg) {
                    xq[i][c] = ldg16(xr + (long long)i * D + col);
                    if (a.w[i] != nullptr) wq[i][c] = ldg16(a.w[i] + woff + col);
                }
            }
            if (a.rope_mask) {
                // tables hold one (cos, sin) per rotary PAIR: [S, D/2] fp32 (the reference's repeat_interleave(2) is implicit)
                const long long ro = PH ? (long long)s * (HD / 2) + (col & (HD - 1)) / 2 : ((long long)s * D + col) / 2;
                c4[c] = *reinterpret_cast<const float4*>(cosT + ro);
                s4[c] = *reinterpret_cast<const float4*>(sinT + ro);
            }
        }
    }
    float ss[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (i < a.nseg && a.w[i] != nullptr) {
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                const int col = (c * ROW_THREADS + threadIdx.x) * 8;
                if (col < D) {
                    float v[8];
                    unpack8(xq[i][c], v);
#pragma unroll
                    for (int e = 0; e < 8; ++e) ss[i] += v[e] * v[e];
                }
            }
        }
    }
    float rstd[3] = {1.f, 1.f, 1.f};
    if (a.w[0] != nullptr || (a.nseg > 1 && a.w[1] != nullptr)) {
        const float2 t = block_sum2(ss[0], ss[1]);
        rstd[0] = rsqrtf(t.x / D + eps);
        rstd[1] = rsqrtf(t.y / D + eps);
    }
    if (a.nseg > 2 && a.w[2] != nullptr) rstd[2] = rsqrtf(block_sum2(ss[2], 0.f).x / D + eps);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (i < a.nseg) {
            const bool norm = a.w[i] != nullptr;
            const bool rope = (a.rope_mask >> i) & 1;
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                const int col = (c * ROW_THREADS + threadIdx.x) * 8;
                if (col < D) {
                    float n[8];
                    unpack8(xq[i][c], n);
                    if (norm) {
                        float w[8];
                        unpack8(wq[i][c], w);
#pragma unroll
                        for (int e = 0; e < 8; ++e) n[e] = n[e] * rstd[i] * w[e];
                    }
                    float o[8];
                    if (rope) {
                        const float cs[4] = {c4[c].x, c4[c].y, c4[c].z, c4[c].w};
                        const float sn[4] = {s4[c].x, s4[c].y, s4[c].z, s4[c].w};
#pragma unroll
                        for (int e = 0; e < 8; e += 2) {
                            o[e] = n[e] * cs[e >> 1] - n[e + 1] * sn[e >> 1];
                            o[e + 1] = n[e + 1] * cs[e >> 1] + n[e] * sn[e >> 1];
                        }
                    } else {
#pragma unroll
                        for (int e = 0; e < 8; ++e) o[e] = n[e];
                    }
                    const int h = col >> (HD == 64 ? 6 : 7), d = col & (HD - 1);
                    stg16(a.dst[i] + (((long long)b * H + h) * S + s) * HD + d, pack8(o));
                }
            }
        }
    }
}

template <int NCH, int HD, bool PH>
__device__ __forceinline__ void qkv_norm_rope_bwd_row(
    const __nv_bfloat16* __restrict__ x, long long ld, long long col_off, const QkvSegArgs a,
    const float* __restrict__ cosT, const float* __restrict__ sinT, __nv_bfloat16* __restrict__ dx, long long ld_dx,
    long long dx_col_off, int S, int H, float eps) {
    const int D = H * HD;
    const int row = blockIdx.x;
    const int b = row / S, s = row % S;
    const __nv_bfloat16* xr = x + (long long)row * ld + col_off;
    const long long woff = a.rows_per_w > 0 ? (long long)(row / a.rows_per_w) * a.w_stride : 0;
    uint4 xq[3][NCH], wq[3][NCH], dq[3][NCH];
    float4 c4[NCH], s4[NCH];
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const int col = (c * ROW_THREADS + threadIdx.x) * 8;
        if (col < D) {
            const int h = col >> (HD == 64 ? 6 : 7), d = col & (HD - 1);
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                if (i < a.nseg) {
                    dq[i][c] = ldg16(a.dst[i] + (((long long)b * H + h) * S + s) * HD + d);
                    if (a.w[i] != nullptr) {
                        xq[i][c] = ldg16(xr + (long long)i * D + col);
                        wq[i][c] = ldg16(a.w[i] + woff + col);
                    }
                }
            }
            if (a.rope_mask) {
                const long long ro = PH ? (long long)s * (HD / 2) + (col & (HD - 1)) / 2 : ((long long)s * D + col) / 2;
                c4[c] = *reinterpret_cast<const float4*>(cosT + ro);
                s4[c] = *reinterpret_cast<const float4*>(sinT + ro);
            }
        }
    }
    float ss[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (i < a.nseg && a.w[i] != nullptr) {
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                const int col = (c * ROW_THREADS + threadIdx.x) * 8;
                if (col < D) {
                    float v[8];
                    unpack8(xq[i][c], v);
#pragma unroll
                    for (int e = 0; e < 8; ++e) ss[i] += v[e] * v[e];
                }
            }
        }
    }
    float rstd[3] = {1.f, 1.f, 1.f};
    const bool n01 = a.w[0] != nullptr || (a.nseg > 1 && a.w[1] != nullptr);
    const bool n2 = a.nseg > 2 && a.w[2] != nullptr;
    if (n01) {
        const float2 t = block_sum2(ss[0], ss[1]);
        rstd[0] = rsqrtf(t.x / D + eps);
        rstd[1] = rsqrtf(t.y / D + eps);
    }
    if (n2) rstd[2] = rsqrtf(block_sum2(ss[2], 0.f).x / D + eps);
    // g = rope^T(dy) * w ; xhat = x * rstd ; dx = rstd * (g - xhat * mean(g * xhat))
    float g[3][NCH][8];
    float sgx[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (i < a.nseg) {
            const bool norm = a.w[i] != nullptr;
            const bool rope = (a.rope_mask >> i) & 1;
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                const int col = (c * ROW_THREADS + threadIdx.x) * 8;
                if (col < D) {
                    float dy[8];
                    unpack8(dq[i][c], dy);
                    if (rope) {
                        const float cs[4] = {c4[c].x, c4[c].y, c4[c].z, c4[c].w};
                        const float sn[4] = {s4[c].x, s4[c].y, s4[c].z, s4[c].w};
#pragma unroll
                        for (int e = 0; e < 8; e += 2) {
                            g[i][c][e] = dy[e] * cs[e >> 1] + dy[e + 1] * sn[e >> 1];
                            g[i][c][e + 1] = dy[e + 1] * cs[e >> 1] - dy[e] * sn[e >> 1];
                        }
                    } else {
#pragma unroll
                        for (int e = 0; e < 8; ++e) g[i][c][e] = dy[e];
                    }
                    if (norm) {
                        float w[8], xv[8];
                        unpack8(wq[i][c], w);
                        unpack8(xq[i][c], xv);
#pragma unroll
                        for (int e = 0; e < 8; ++e) {
                            g[i][c][e] *= w[e];
                            sgx[i] += g[i][c][e] * (xv[e] * rstd[i]);
                        }
                    }
                }
            }
        }
    }
    float mgx[3] = {0.f, 0.f, 0.f};
    if (n01) {
        const float2 t = block_sum2(sgx[0], sgx[1]);
        mgx[0] = t.x / D;
        mgx[1] = t.y / D;
    }
    if (n2) mgx[2] = block_sum2(sgx[2], 0.f).x / D;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (i < a.nseg) {
            const bool norm = a.w[i] != nullptr;
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                const int col = (c * ROW_THREADS + threadIdx.x) * 8;
                if (col < D) {
                    float o[8];
                    if (norm) {
                        float xv[8];
                        unpack8(xq[i][c], xv);
#pragma unroll
                        for (int e = 0; e < 8; ++e) o[e] = rstd[i] * (g[i][c][e] - (xv[e] * rstd[i]) * mgx[i]);
                    } else {
#pragma unroll
                        for (int e = 0; e < 8; ++e) o[e] = g[i][c][e];
                    }
                    stg16(dx + (long long)row * ld_dx + dx_col_off + (long long)i * D + col, pack8(o));
                }
            }
        }
    }
}

template <int NCH, int HD = 64>
__global__ void __launch_bounds__(ROW_THREADS) qkv_norm_rope_fwd_kernel(
    const __nv_bfloat16* __restrict__ src, long long ld, long long col_off, const QkvSegArgs a,
    const float* __restrict__ cosT, const float* __restrict__ sinT, int S, int H, float eps) {
    griddep_launch_dependents();
    griddep_wait();
    qkv_norm_rope_fwd_row<NCH, HD, false>(src, ld, col_off, a, cosT, sinT, S, H, eps);
}
template <int NCH, int HD>
__global__ void __launch_bounds__(ROW_THREADS) per_head_rope_qk_norm_fwd_kernel(
    const __nv_bfloat16* __restrict__ src, long long ld, long long col_off, const QkvSegArgs a,
    const float* __restrict__ cosT, const float* __restrict__ sinT, int S, int H, float eps) {
    griddep_launch_dependents();
    griddep_wait();
    qkv_norm_rope_fwd_row<NCH, HD, true>(src, ld, col_off, a, cosT, sinT, S, H, eps);
}
template <int NCH, int HD = 64>
__global__ void __launch_bounds__(ROW_THREADS) qkv_norm_rope_bwd_kernel(
    const __nv_bfloat16* __restrict__ x, long long ld, long long col_off, const QkvSegArgs a,
    const float* __restrict__ cosT, const float* __restrict__ sinT, __nv_bfloat16* __restrict__ dx, long long ld_dx,
    long long dx_col_off, int S, int H, float eps) {
    griddep_launch_dependents();
    griddep_wait();
    qkv_norm_rope_bwd_row<NCH, HD, false>(x, ld, col_off, a, cosT, sinT, dx, ld_dx, dx_col_off, S, H, eps);
}
template <int NCH, int HD>
__global__ void __launch_bounds__(ROW_THREADS) per_head_rope_qk_norm_bwd_kernel(
    const __nv_bfloat16* __restrict__ x, long long ld, long long col_off, const QkvSegArgs a,
    const float* __restrict__ cosT, const float* __restrict__ sinT, __nv_bfloat16* __restrict__ dx, long long ld_dx,
    long long dx_col_off, int S, int H, float eps) {
    griddep_launch_dependents();
    griddep_wait();
    qkv_norm_rope_bwd_row<NCH, HD, true>(x, ld, col_off, a, cosT, sinT, dx, ld_dx, dx_col_off, S, H, eps);
}

// RoPE table: diffusers LTXVideoRotaryPosEmbed, fp32, one (cos, sin) per rotary pair: [S, D/2].  One thread per (s, pair).
__global__ void rope_table_kernel(float* __restrict__ cosT, float* __restrict__ sinT, int F, int H, int W, int D,
                                  float sf, float sh, float sw) {
    const int nf = D / 6;
    const int pad = D % 6;
    const long long S = (long long)F * H * W;
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int pairs = D / 2;
    if (idx >= S * pairs) return;
    const int s = (int)(idx / pairs);
    const int pr = (int)(idx % pairs);
    const int col = pr * 2;
    float c = 1.f, sn = 0.f;
    if (col >= pad) {
        const int j = (col - pad) / 2;
        const int fi = j / 3, axis = j % 3;
        const int w = s % W, h = (s / W) % H, f = s / (W * H);
        float g = axis == 0 ? (float)f * sf : (axis == 1 ? (float)h * sh : (float)w * sw);
        // torch.linspace(0, 1, nf) (symmetric evaluation), theta ** x, * pi/2, * (2g - 1): same op order, fp32
        const float step = 1.0f / (float)(nf - 1);
        float lin = (fi < nf / 2) ? (float)fi * step : 1.0f - (float)(nf - 1 - fi) * step;
        float fr = powf(10000.0f, lin);
        fr = fr * 1.5707963267948966f;
        float ang = fr * (g * 2.0f - 1.0f);
        c = cosf(ang);
        sn = sinf(ang);
    }
    cosT[(long long)s * pairs + pr] = c;
    sinT[(long long)s * pairs + pr] = sn;
}

// ------------------------------------------------------------------------------------------------
// step prologue: normalise + flow-match x_t + pack [B,C,F,HW] -> [B, F*HW, C]; target = n - x0.
// Rounding points mirror the reference's bf16 tensors (base_specification.py:295-322): x0 rounded to bf16, x_t computed
// in fp32 from (bf16 x0, bf16 n, fp32 sigma) then rounded, target = bf16(n - x0).
// ------------------------------------------------------------------------------------------------
// normalise one bf16-valued latent x, noise it and write the packed x_t / target element idx
__device__ __forceinline__ void prep_noise_store(float x, long long idx, long long src, int b, int c, long long s,
                                                 const __nv_bfloat16* __restrict__ noise, const float* __restrict__ mean,
                                                 const float* __restrict__ stdv, const float* __restrict__ sigma,
                                                 const float* __restrict__ sigma_ff, __nv_bfloat16* __restrict__ x_t,
                                                 __nv_bfloat16* __restrict__ target, int C, int HW) {
    float x0f = __fdiv_rn(__fmul_rn(__fsub_rn(x, mean[b * C + c]), 1.0f), stdv[b * C + c]);
    float x0 = __bfloat162float(__float2bfloat16_rn(x0f));
    float n = __bfloat162float(noise[src]);
    float sg = sigma[b];
    if (sigma_ff != nullptr && s < HW) sg = sigma_ff[b];
    float xt = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, sg), x0), __fmul_rn(sg, n));
    x_t[idx] = __float2bfloat16_rn(xt);
    target[idx] = __float2bfloat16_rn(__fsub_rn(n, x0));
}

__global__ void prep_noise_pack_kernel(const __nv_bfloat16* __restrict__ lat, const __nv_bfloat16* __restrict__ noise,
                                       const float* __restrict__ mean, const float* __restrict__ stdv,
                                       const float* __restrict__ sigma, const float* __restrict__ sigma_ff,
                                       __nv_bfloat16* __restrict__ x_t, __nv_bfloat16* __restrict__ target, int B,
                                       int C, int F, int HW) {
    const long long S = (long long)F * HW;
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * S * C) return;
    const int c = (int)(idx % C);
    const long long s = (idx / C) % S;
    const int b = (int)(idx / (C * S));
    const long long src = ((long long)b * C + c) * S + s;
    float x = __bfloat162float(lat[src]);
    prep_noise_store(x, idx, src, b, c, s, noise, mean, stdv, sigma, sigma_ff, x_t, target, C, HW);
}

__device__ __forceinline__ float round_bf16(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// The same prologue fed with VAE moments [B, 2C, F*HW] = [mean | logvar] instead of latents: the latent is first sampled
// from the diagonal Gaussian, x = mean + exp(0.5 clamp(logvar, -30, 20)) * eps (finetrainers/models/utils.py:8-31),
// with eps [B, C, F*HW] drawn by the caller.  Every step is rounded to bf16 where the reference's bf16 tensor ops round:
// clamp (exact, NaN kept), 0.5 * logvar (exact), exp (fp32 expf, then bf16), std * eps, mean + that.  x never reaches
// memory unless latents_out [B, C, F*HW] is given.
__global__ void prep_posterior_noise_pack_kernel(const __nv_bfloat16* __restrict__ moments,
                                                 const __nv_bfloat16* __restrict__ eps,
                                                 const __nv_bfloat16* __restrict__ noise, const float* __restrict__ mean,
                                                 const float* __restrict__ stdv, const float* __restrict__ sigma,
                                                 const float* __restrict__ sigma_ff, __nv_bfloat16* __restrict__ x_t,
                                                 __nv_bfloat16* __restrict__ target,
                                                 __nv_bfloat16* __restrict__ latents_out, int B, int C, int F, int HW) {
    const long long S = (long long)F * HW;
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * S * C) return;
    const int c = (int)(idx % C);
    const long long s = (idx / C) % S;
    const int b = (int)(idx / (C * S));
    const long long src = ((long long)b * C + c) * S + s;
    const long long msrc = ((long long)b * 2 * C + c) * S + s;
    const float mu = __bfloat162float(moments[msrc]);
    float lv = __bfloat162float(moments[msrc + (long long)C * S]);
    if (!isnan(lv)) lv = fminf(fmaxf(lv, -30.0f), 20.0f);
    const float sd = round_bf16(expf(round_bf16(__fmul_rn(0.5f, lv))));
    const float x = round_bf16(__fadd_rn(mu, round_bf16(__fmul_rn(sd, __bfloat162float(eps[src])))));
    if (latents_out != nullptr) latents_out[src] = __float2bfloat16_rn(x);
    prep_noise_store(x, idx, src, b, c, s, noise, mean, stdv, sigma, sigma_ff, x_t, target, C, HW);
}

// ------------------------------------------------------------------------------------------------
// loss = mean_b( mean_i( w_b (p - t)^2 ) ) * loss_scale ; dpred = 2 w_b (p - t) / (n B) * loss_scale
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ROW_THREADS) loss_mse_kernel(const __nv_bfloat16* __restrict__ pred,
                                                               const __nv_bfloat16* __restrict__ target,
                                                               const float* __restrict__ weight, float loss_scale,
                                                               __nv_bfloat16* __restrict__ dpred,
                                                               float* __restrict__ partial, int B,
                                                               long long per_sample) {
    const long long total8 = (long long)B * per_sample / 8;
    float acc = 0.f;
    const float inv = loss_scale / ((float)per_sample * (float)B);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total8; i += (long long)gridDim.x * blockDim.x) {
        const long long e0 = i * 8;
        const int b = (int)(e0 / per_sample);
        const float w = weight ? weight[b] : 1.f;
        float p[8], t[8], g[8];
        unpack8(ldg16(pred + e0), p);
        unpack8(ldg16(target + e0), t);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float d = p[e] - t[e];
            acc += w * d * d;
            g[e] = 2.f * w * d * inv;
        }
        if (dpred) stg16(dpred + e0, pack8(g));
    }
    float2 r = block_sum2(acc, 0.f);
    if (threadIdx.x == 0) partial[blockIdx.x] = r.x * inv;
}
__global__ void final_sum_kernel(const float* __restrict__ partial, int n, float* __restrict__ out, int accumulate) {
    float a = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) a += partial[i];
    float2 r = block_sum2(a, 0.f);
    if (threadIdx.x == 0) *out = accumulate ? (*out + r.x) : r.x;
}

__global__ void timestep_sinusoid_kernel(const float* __restrict__ t, __nv_bfloat16* __restrict__ out, int n) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * 128) return;
    const int i = idx % 128, r = idx / 128;
    const float freq = expf(-9.210340371976184f * (float)i / 128.0f);
    const float a = t[r] * freq;
    out[(long long)r * 256 + i] = __float2bfloat16_rn(cosf(a));
    out[(long long)r * 256 + 128 + i] = __float2bfloat16_rn(sinf(a));
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n,
                                     float scale) {
    long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        float4 v = *reinterpret_cast<const float4*>(src + i);
        uint2 o = make_uint2(pack_bf16x2(v.x * scale, v.y * scale), pack_bf16x2(v.z * scale, v.w * scale));
        *reinterpret_cast<uint2*>(dst + i) = o;
    } else {
        for (; i < n; ++i) dst[i] = __float2bfloat16_rn(src[i] * scale);
    }
}

// deterministic split-K reduction: out[m, c] = bf16(alpha * (part[0, m, c] + part[1, m, c] + ... + part[s - 1, m, c]))
// over an [M, N] window of a bf16 matrix with leading dimension ldc.  Eight columns per thread: two 16-byte loads per
// slice, one 16-byte store.  The slices are added in slice order, so the result does not depend on which slice's CTAs
// finished first.
__global__ void __launch_bounds__(256) splitk_reduce_bf16_kernel(const float* __restrict__ part, int splits, int M, int N,
                                                                 float alpha, __nv_bfloat16* __restrict__ out,
                                                                 long long ldc) {
    griddep_launch_dependents();
    griddep_wait();
    const int n8 = N >> 3;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)M * n8) return;
    const long long row = idx / n8;
    const int col = (int)(idx - row * n8) * 8;
    const long long slice = (long long)M * N;
    const float* p = part + row * N + col;
    float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    for (int z = 1; z < splits; ++z) {
        const float4 u = *reinterpret_cast<const float4*>(p + z * slice);
        const float4 v = *reinterpret_cast<const float4*>(p + z * slice + 4);
        a.x += u.x; a.y += u.y; a.z += u.z; a.w += u.w;
        b.x += v.x; b.y += v.y; b.z += v.z; b.w += v.w;
    }
    const float f[8] = {alpha * a.x, alpha * a.y, alpha * a.z, alpha * a.w,
                        alpha * b.x, alpha * b.y, alpha * b.z, alpha * b.w};
    stg16(out + row * ldc + col, pack8(f));
}

// two fp8 codes (low byte = first element) -> two bf16 (low half = first element).  The hardware cvt gives f16, which
// holds every e4m3fn and e5m2 value (and Inf / NaN) exactly; f16 -> f32 -> bf16 is exact for them too, since an fp8
// mantissa has at most 3 bits and both exponent ranges fit bf16's.
template <int FMT>
__device__ __forceinline__ uint32_t fp8x2_to_bf16x2(uint32_t v) {
    uint32_t h;
    if (FMT == 0)
        asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"((unsigned short)v));
    else
        asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(h) : "h"((unsigned short)v));
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h));
    return pack_bf16x2(f.x, f.y);
}

// layerwise weight upcast: 16 fp8 codes per 128-bit load, two 128-bit bf16 stores; grid-stride over the 16-code vectors,
// the < 16-code tail goes to the first thread
template <int FMT>
__global__ void __launch_bounds__(256) upcast_fp8_bf16_kernel(const uint8_t* __restrict__ src,
                                                              __nv_bfloat16* __restrict__ dst, long long n) {
    griddep_launch_dependents();
    griddep_wait();
    const long long n16 = n >> 4;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) {
        const uint4 v = ldg16(src + i * 16);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t o[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            o[2 * j] = fp8x2_to_bf16x2<FMT>(w[j] & 0xffffu);
            o[2 * j + 1] = fp8x2_to_bf16x2<FMT>(w[j] >> 16);
        }
        stg16(dst + i * 16, make_uint4(o[0], o[1], o[2], o[3]));
        stg16(dst + i * 16 + 8, make_uint4(o[4], o[5], o[6], o[7]));
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        for (long long i = n16 * 16; i < n; ++i) {
            const uint32_t o = fp8x2_to_bf16x2<FMT>(src[i]);
            dst[i] = *reinterpret_cast<const __nv_bfloat16*>(&o);
        }
    }
}

// one denoising step of the flow-match Euler sampler with classifier-free guidance (LTXPipeline.__call__ + diffusers'
// FlowMatchEulerDiscreteScheduler.step), rounded where the pipeline's fp32 tensor ops round: v = u + g (c - u) on the
// bf16 prediction [u; c] upcast to fp32, x' = x + dt v.  The _rn intrinsics keep the compiler from contracting either
// pair into an FMA, which rounds once instead of twice.
template <bool CFG>
__device__ __forceinline__ float cfg_euler_one(float u, float c, float x, float g, float dt) {
    const float v = CFG ? __fadd_rn(u, __fmul_rn(g, __fsub_rn(c, u))) : u;
    return __fadd_rn(x, __fmul_rn(dt, v));
}

// pred [rows * total] bf16 (rows = 2 with CFG: the uncond block first), x [total] fp32 updated in place, x_next
// [rows * total] bf16 = bf16(x') in every block.  Eight elements per thread as 128-bit accesses over the first n8 * 8
// elements (n8 = 0 when an operand's block offset is not 16-byte aligned), grid-stride; the rest element by element.
template <bool CFG>
__global__ void __launch_bounds__(256) cfg_euler_step_kernel(const __nv_bfloat16* __restrict__ pred,
                                                             float* __restrict__ x, __nv_bfloat16* __restrict__ x_next,
                                                             long long total, long long n8, float g,
                                                             const float* __restrict__ dt_ptr) {
    griddep_launch_dependents();
    griddep_wait();
    const float dt = *dt_ptr;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (long long i = t0; i < n8; i += stride) {
        const long long e = i * 8;
        float u[8], c[8];
        unpack8(ldg16(pred + e), u);
        if (CFG) unpack8(ldg16(pred + total + e), c);
        const float4 xa = *reinterpret_cast<const float4*>(x + e), xb = *reinterpret_cast<const float4*>(x + e + 4);
        float o[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = cfg_euler_one<CFG>(u[k], CFG ? c[k] : 0.f, o[k], g, dt);
        *reinterpret_cast<float4*>(x + e) = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(x + e + 4) = make_float4(o[4], o[5], o[6], o[7]);
        const uint4 q = pack8(o);
        stg16(x_next + e, q);
        if (CFG) stg16(x_next + total + e, q);
    }
    for (long long e = n8 * 8 + t0; e < total; e += stride) {
        const float u = __bfloat162float(pred[e]);
        const float c = CFG ? __bfloat162float(pred[total + e]) : 0.f;
        const float o = cfg_euler_one<CFG>(u, c, x[e], g, dt);
        x[e] = o;
        x_next[e] = __float2bfloat16_rn(o);
        if (CFG) x_next[total + e] = __float2bfloat16_rn(o);
    }
}

// cfg_euler_step_kernel's step on the elements n_cond .. n of each of the B samples (n elements each); the first n_cond
// of every sample (the conditioning frame) are neither read in pred nor written.  total = B n.  With vec (n % 8 == 0),
// each sample's elements from c8 (n_cond rounded up to a multiple of 8) run eight per thread as 128-bit accesses and
// those before c8 element by element; without vec, c8 = n and all run element by element.  Grid-stride.
template <bool CFG>
__global__ void __launch_bounds__(256) cfg_euler_step_cond_kernel(const __nv_bfloat16* __restrict__ pred,
                                                                  float* __restrict__ x,
                                                                  __nv_bfloat16* __restrict__ x_next, int B,
                                                                  long long n, long long n_cond, long long c8, float g,
                                                                  const float* __restrict__ dt_ptr) {
    griddep_launch_dependents();
    griddep_wait();
    const float dt = *dt_ptr;
    const long long total = (long long)B * n;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long m8 = (n - c8) / 8;  // vectors per sample
    for (long long i = t0; i < B * m8; i += stride) {
        const long long b = i / m8;
        const long long e = b * n + c8 + (i - b * m8) * 8;
        float u[8], c[8];
        unpack8(ldg16(pred + e), u);
        if (CFG) unpack8(ldg16(pred + total + e), c);
        const float4 xa = *reinterpret_cast<const float4*>(x + e), xb = *reinterpret_cast<const float4*>(x + e + 4);
        float o[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = cfg_euler_one<CFG>(u[k], CFG ? c[k] : 0.f, o[k], g, dt);
        *reinterpret_cast<float4*>(x + e) = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(x + e + 4) = make_float4(o[4], o[5], o[6], o[7]);
        const uint4 q = pack8(o);
        stg16(x_next + e, q);
        if (CFG) stg16(x_next + total + e, q);
    }
    const long long ms = c8 - n_cond;  // scalar elements per sample
    for (long long i = t0; i < B * ms; i += stride) {
        const long long b = i / ms;
        const long long e = b * n + n_cond + (i - b * ms);
        const float u = __bfloat162float(pred[e]);
        const float c = CFG ? __bfloat162float(pred[total + e]) : 0.f;
        const float o = cfg_euler_one<CFG>(u, c, x[e], g, dt);
        x[e] = o;
        x_next[e] = __float2bfloat16_rn(o);
        if (CFG) x_next[total + e] = __float2bfloat16_rn(o);
    }
}

__global__ void __launch_bounds__(ROW_THREADS) sumsq_kernel(const float* __restrict__ x, long long n,
                                                            float* __restrict__ partial) {
    float acc = 0.f;
    const long long n4 = n / 4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 v = reinterpret_cast<const float4*>(x)[i];
        acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0)
        for (long long i = n4 * 4; i < n; ++i) acc += x[i] * x[i];
    float2 r = block_sum2(acc, 0.f);
    if (threadIdx.x == 0) partial[blockIdx.x] = r.x;
}

// clip (utils/torch.py:99-161: coef = min(1, max_norm / (norm + 1e-6))) + AdamW (torch.optim.AdamW math) + zero grad
__device__ __forceinline__ void adamw_one(float& pi, float& gi_io, float& mi, float& vi, float coef, float lr, float b1,
                                          float b2, float eps, float wd, float bc1, float bc2_sqrt) {
    const float gi = gi_io * coef;
    pi *= (1.f - lr * wd);
    mi = b1 * mi + (1.f - b1) * gi;
    vi = b2 * vi + (1.f - b2) * gi * gi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    pi -= (lr / bc1) * (mi / denom);
    gi_io = 0.f;
}

// four elements per thread as 16-byte accesses (7 streams of 4 B per element: the kernel is pure HBM traffic, and with one
// element per thread it ran at ~60 % of the copy bandwidth); n4 = n / 4 vectors, the < 4-element tail goes to the last thread
__global__ void __launch_bounds__(256) adamw_clip_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                                         float* __restrict__ v, long long n, const float* __restrict__ sumsq,
                                                         float max_norm, float lr, float b1, float b2, float eps, float wd,
                                                         float bc1, float bc2_sqrt, float grad_div) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n4 = n >> 2;
    float coef = grad_div;
    if (max_norm > 0.f) {
        float norm = sqrtf(*sumsq) * grad_div;
        coef *= fminf(1.f, max_norm / (norm + 1e-6f));
    }
    if (i < n4) {
        float4 pp = reinterpret_cast<float4*>(p)[i], gg = reinterpret_cast<float4*>(g)[i];
        float4 mm = reinterpret_cast<float4*>(m)[i], vv = reinterpret_cast<float4*>(v)[i];
        adamw_one(pp.x, gg.x, mm.x, vv.x, coef, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
        adamw_one(pp.y, gg.y, mm.y, vv.y, coef, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
        adamw_one(pp.z, gg.z, mm.z, vv.z, coef, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
        adamw_one(pp.w, gg.w, mm.w, vv.w, coef, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
        reinterpret_cast<float4*>(p)[i] = pp;
        reinterpret_cast<float4*>(g)[i] = gg;
        reinterpret_cast<float4*>(m)[i] = mm;
        reinterpret_cast<float4*>(v)[i] = vv;
    }
    if (i == n4) {
        for (long long j = n4 << 2; j < n; ++j) adamw_one(p[j], g[j], m[j], v[j], coef, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    }
}

// ------------------------------------------------------------------------------------------------
// Wan-2.1 (diffusers WanTransformer3DModel): per-head RoPE table, step prologue, patch permutes
// ------------------------------------------------------------------------------------------------
// WanRotaryPosEmbed: head_dim HD splits into t / h / w parts of HD - 2 (HD / 6) / 2 (HD / 6) / 2 (HD / 6) dims (44 / 42 /
// 42 at 128); pair i of a part of dim n rotates by pos * theta^(-2i / n), pos the integer grid index along its axis.  The
// frequency and the angle are float64 as in diffusers (freqs_dtype=torch.float64), cos / sin rounded once to fp32.
// [S, HD/2], one thread per (token, pair).
__global__ void rope_table_wan_kernel(float* __restrict__ cosT, float* __restrict__ sinT, int F, int H, int W, int HD,
                                      double theta) {
    const int pairs = HD / 2;
    const long long S = (long long)F * H * W;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= S * pairs) return;
    const int s = (int)(idx / pairs), j = (int)(idx % pairs);
    const int nhw = HD / 6, nt = pairs - 2 * nhw;  // pairs of the t part, of the h part, of the w part
    int i, n, pos;
    if (j < nt) { i = j; n = 2 * nt; pos = s / (W * H); }
    else if (j < nt + nhw) { i = j - nt; n = 2 * nhw; pos = (s / W) % H; }
    else { i = j - nt - nhw; n = 2 * nhw; pos = s % W; }
    const double freq = 1.0 / pow(theta, (double)(2 * i) / (double)n);
    const double ang = (double)pos * freq;
    cosT[idx] = (float)cos(ang);
    sinT[idx] = (float)sin(ang);
}

// Wan step prologue, per latent element (b, c, f, h, w) of C channels:
//   mu, logvar = moments[:, :C], moments[:, C:]  normalised as bf16((v - mean[b, c]) * std[b, c]) (std = 1 / latents_std)
//   x = mu + exp(0.5 clamp(logvar, -30, 20)) * eps   rounded at every bf16 tensor op (DiagonalGaussianDistribution.sample)
//   x_t = bf16((1 - sigma) x + sigma n),  target = bf16(n - x)   (flow_match_xt / flow_match_target)
// x_t goes to the patchified [B, F (H/2) (W/2), 4C] rows at k = c 4 + kh 2 + kw (the Conv3d weight's order), target to
// k = (kh 2 + kw) C + c (proj_out's output order, which diffusers unpatchifies).
__device__ __forceinline__ long long patch_index(int b, int c, int f, int h, int w, int C, int F, int H, int W,
                                                 int out_order) {
    const int Hp = H >> 1, Wp = W >> 1, p = (h & 1) * 2 + (w & 1);
    const long long tok = ((long long)b * F + f) * Hp * Wp + (long long)(h >> 1) * Wp + (w >> 1);
    return tok * 4 * C + (out_order ? p * C + c : c * 4 + p);
}

//
// I2V: x_t goes instead to the [B, F (H/2) (W/2), 4 (2C + Cm)] rows of the transformer input cat([x_t, mask, condition])
// in the Conv3d order over the concatenated channels; the same thread also writes the condition channel c
// (bf16((cond_mean - mean) * std), the mode of the normalised condition posterior) and, for c < Cm, mask channel c.
template <bool I2V = false>
__global__ void wan_prep_kernel(const __nv_bfloat16* __restrict__ moments, const __nv_bfloat16* __restrict__ eps,
                                const __nv_bfloat16* __restrict__ noise, const float* __restrict__ mean,
                                const float* __restrict__ stdv, const float* __restrict__ sigma,
                                __nv_bfloat16* __restrict__ x_t, __nv_bfloat16* __restrict__ target, int B, int C, int F,
                                int H, int W, const __nv_bfloat16* __restrict__ cond_moments = nullptr,
                                const __nv_bfloat16* __restrict__ cond_mask = nullptr, int Cm = 0) {
    const long long HW = (long long)H * W, S = F * HW;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // source order [B, C, F, H, W]
    if (idx >= (long long)B * C * S) return;
    const long long sp = idx % S;
    const int c = (int)((idx / S) % C), b = (int)(idx / (S * C));
    const int f = (int)(sp / HW), h = (int)((sp % HW) / W), w = (int)(sp % W);
    const long long msrc = ((long long)b * 2 * C + c) * S + sp;
    const float m = mean[b * C + c], sd = stdv[b * C + c];
    const float mu = round_bf16(__fmul_rn(__fsub_rn(__bfloat162float(moments[msrc]), m), sd));
    float lv = round_bf16(__fmul_rn(__fsub_rn(__bfloat162float(moments[msrc + (long long)C * S]), m), sd));
    if (!isnan(lv)) lv = fminf(fmaxf(lv, -30.0f), 20.0f);
    const float sdv = round_bf16(expf(round_bf16(__fmul_rn(0.5f, lv))));
    const float x = round_bf16(__fadd_rn(mu, round_bf16(__fmul_rn(sdv, __bfloat162float(eps[idx])))));
    const float n = __bfloat162float(noise[idx]);
    const float sg = sigma[b];
    const __nv_bfloat16 xt = __float2bfloat16_rn(__fadd_rn(__fmul_rn(__fsub_rn(1.0f, sg), x), __fmul_rn(sg, n)));
    if constexpr (I2V) {
        const int Ct = 2 * C + Cm;  // channels of the concatenated input
        const long long row = ((long long)b * F + f) * (H >> 1) * (W >> 1) + (long long)(h >> 1) * (W >> 1) + (w >> 1);
        __nv_bfloat16* xr = x_t + row * 4 * Ct + (h & 1) * 2 + (w & 1);
        xr[c * 4] = xt;
        xr[(C + Cm + c) * 4] = __float2bfloat16_rn(__fmul_rn(__fsub_rn(__bfloat162float(cond_moments[msrc]), m), sd));
        if (c < Cm) xr[(C + c) * 4] = cond_mask[((long long)b * Cm + c) * S + sp];
    } else {
        x_t[patch_index(b, c, f, h, w, C, F, H, W, 0)] = xt;
    }
    target[patch_index(b, c, f, h, w, C, F, H, W, 1)] = __float2bfloat16_rn(__fsub_rn(n, x));
}

// y = bf16(0.5 x (1 + erf(x / sqrt 2))) in fp32, as torch's exact GELU (F.gelu(approximate="none")) on bf16 tensors
__global__ void gelu_erf_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = __bfloat162float(x[i]);
    y[i] = __float2bfloat16_rn(__fmul_rn(__fmul_rn(v, 0.5f), __fadd_rn(1.0f, erff(__fmul_rn(v, 0.7071067811865476f)))));
}

// exact bf16 permute between [B, C, F, H, W] and the patchified [B, F (H/2) (W/2), 4C] (either channel order)
__global__ void patch_permute_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int B,
                                     int C, int F, int H, int W, int out_order, int unpatchify) {
    const long long HW = (long long)H * W, S = F * HW;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * C * S) return;
    const long long sp = idx % S;
    const int c = (int)((idx / S) % C), b = (int)(idx / (S * C));
    const long long pk = patch_index(b, c, (int)(sp / HW), (int)((sp % HW) / W), (int)(sp % W), C, F, H, W, out_order);
    if (unpatchify) dst[idx] = src[pk];
    else dst[pk] = src[idx];
}

}  // namespace b2d

using namespace b2d;
#define STREAM reinterpret_cast<cudaStream_t>(stream)

// instantiate the row kernels for 1..4 chunks of 2048 columns (registers scale with the chunk count)
#define ROW_DISPATCH(D_, KERNEL, GRID, ...)                                             \
    do {                                                                                \
        const int nch__ = ((D_) + 8 * ROW_THREADS - 1) / (8 * ROW_THREADS);             \
        if (nch__ <= 1) launch_k(KERNEL<1>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);       \
        else if (nch__ == 2) launch_k(KERNEL<2>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);  \
        else launch_k(KERNEL<4>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);                  \
    } while (0)

// the q/k-norm + RoPE kernels take the head dimension as a second template parameter that defaults to 64, so ROW_DISPATCH
// launches their head_dim-64 instantiations; this launches the head_dim-128 ones
#define ROW_DISPATCH_HD128(D_, KERNEL, GRID, ...)                                            \
    do {                                                                                     \
        const int nch__ = ((D_) + 8 * ROW_THREADS - 1) / (8 * ROW_THREADS);                  \
        if (nch__ <= 1) launch_k(KERNEL<1, 128>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);       \
        else if (nch__ == 2) launch_k(KERNEL<2, 128>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);  \
        else launch_k(KERNEL<4, 128>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);                  \
    } while (0)

// the per-head-RoPE kernels (head dimension HD_)
#define ROW_DISPATCH_PH(D_, KERNEL, HD_, GRID, ...)                                          \
    do {                                                                                     \
        const int nch__ = ((D_) + 8 * ROW_THREADS - 1) / (8 * ROW_THREADS);                  \
        if (nch__ <= 1) launch_k(KERNEL<1, HD_>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);       \
        else if (nch__ == 2) launch_k(KERNEL<2, HD_>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);  \
        else launch_k(KERNEL<4, HD_>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);                  \
    } while (0)

// the affine-LayerNorm instantiations of the norm + modulate kernels
#define ROW_DISPATCH_AFFINE(D_, KERNEL, GRID, ...)                                           \
    do {                                                                                     \
        const int nch__ = ((D_) + 8 * ROW_THREADS - 1) / (8 * ROW_THREADS);                  \
        if (nch__ <= 1) launch_k(KERNEL<1, true>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);       \
        else if (nch__ == 2) launch_k(KERNEL<2, true>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);  \
        else launch_k(KERNEL<4, true>, dim3(GRID), dim3(ROW_THREADS), 0, STREAM, __VA_ARGS__);                  \
    } while (0)

static int check_rowop(int rows, int D, int rps) {
    if (rows <= 0 || D <= 0 || rps <= 0) return set_error(B2D_ERR_SHAPE, "rows/D/rows_per_sample must be positive");
    if (D % 8 != 0 || D > 8 * ROW_THREADS * MAX_CHUNKS) return set_error(B2D_ERR_SHAPE, "D=%d must be a multiple of 8 and <= %d", D, 8 * ROW_THREADS * MAX_CHUNKS);
    return 0;
}

// true when any pointer is not a multiple of `align` bytes.  The kernels access these operands as 16-byte (or 8-byte)
// vectors, and a misaligned vector access faults the whole context, so the entry points refuse them up front.  NULL
// (an absent optional operand) passes.
static bool misaligned(std::initializer_list<const void*> ptrs, uintptr_t align = 16) {
    uintptr_t bits = 0;
    for (const void* p : ptrs) bits |= reinterpret_cast<uintptr_t>(p);
    return (bits & (align - 1)) != 0;
}

extern "C" int b2d_norm_modulate_fwd(const void* x, void* y, const void* shift_tab, const void* shift_emb,
                                     const void* scale_tab, const void* scale_emb, int64_t emb_stride, int32_t rows,
                                     int32_t D, int32_t rows_per_sample, float eps, int32_t layer_norm, void* stream) {
    B2D_BIND(x);
    if (int rc = check_rowop(rows, D, rows_per_sample)) return rc;
    if (misaligned({x, y, shift_tab, shift_emb, scale_tab, scale_emb}) || emb_stride % 8)
        return set_error(B2D_ERR_ALIGN, "norm_modulate_fwd: pointers must be 16-byte aligned, emb_stride a multiple of 8");
    ROW_DISPATCH(D, norm_modulate_fwd_kernel, rows,
        (const __nv_bfloat16*)x, (__nv_bfloat16*)y, (const __nv_bfloat16*)shift_tab, (const __nv_bfloat16*)shift_emb,
        (const __nv_bfloat16*)scale_tab, (const __nv_bfloat16*)scale_emb, emb_stride, D, rows_per_sample, eps, layer_norm);
    B2D_CHECK_LAUNCH("norm_modulate_fwd");
    return 0;
}

extern "C" int b2d_norm_modulate_bwd(const void* dy, const void* x, const void* dx_in, void* dx_out,
                                     const void* scale_tab, const void* scale_emb, const void* gate2_tab,
                                     const void* gate2_emb, void* out2, int64_t emb_stride, int32_t rows, int32_t D,
                                     int32_t rows_per_sample, float eps, int32_t layer_norm, void* stream) {
    B2D_BIND(dy);
    if (int rc = check_rowop(rows, D, rows_per_sample)) return rc;
    if (misaligned({dy, x, dx_in, dx_out, scale_tab, scale_emb, gate2_tab, gate2_emb, out2}) || emb_stride % 8)
        return set_error(B2D_ERR_ALIGN, "norm_modulate_bwd: pointers must be 16-byte aligned, emb_stride a multiple of 8");
    ROW_DISPATCH(D, norm_modulate_bwd_kernel, rows,
        (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dx_in, (__nv_bfloat16*)dx_out,
        (const __nv_bfloat16*)scale_tab, (const __nv_bfloat16*)scale_emb, (const __nv_bfloat16*)gate2_tab,
        (const __nv_bfloat16*)gate2_emb, (__nv_bfloat16*)out2, emb_stride, D, rows_per_sample, eps, layer_norm);
    B2D_CHECK_LAUNCH("norm_modulate_bwd");
    return 0;
}

extern "C" int b2d_colscale(const void* x, void* out, const void* tab, const void* emb, int64_t emb_stride,
                            int32_t rows, int32_t D, int32_t rows_per_sample, void* stream) {
    B2D_BIND(x);
    if (D % 8) return set_error(B2D_ERR_SHAPE, "colscale: D %% 8");
    if (rows_per_sample <= 0) return set_error(B2D_ERR_SHAPE, "colscale: rows_per_sample must be positive");
    if (misaligned({x, out, tab, emb}) || emb_stride % 8)
        return set_error(B2D_ERR_ALIGN, "colscale: pointers must be 16-byte aligned, emb_stride a multiple of 8");
    long long total8 = (long long)rows * D / 8;
    launch_k(colscale_kernel, dim3((unsigned)((total8 + 255) / 256)), dim3(256), 0, STREAM, (const __nv_bfloat16*)x,
             (__nv_bfloat16*)out, (const __nv_bfloat16*)tab, (const __nv_bfloat16*)emb, emb_stride, total8, D,
             rows_per_sample);
    B2D_CHECK_LAUNCH("colscale");
    return 0;
}

// segment arguments shared by both directions: every segment has its head-split tensor (dst_i / dy_i), rope_mask names
// only existing segments, and every vector-accessed operand (src or x, dx, dst_i / dy_i, w_i, the tables) is aligned
static int check_qkv_segs(const void* src, const void* dx, const QkvSegArgs& a, const void* cos, const void* sin,
                          const char* what) {
    for (int i = 0; i < a.nseg; ++i)
        if (a.dst[i] == nullptr) return set_error(B2D_ERR_ARG, "%s: segment %d has no head-split tensor", what, i);
    if (a.rope_mask < 0 || (a.rope_mask >> a.nseg) != 0)
        return set_error(B2D_ERR_ARG, "%s: rope_mask 0x%x names a segment >= nseg = %d", what, a.rope_mask, a.nseg);
    if (misaligned({src, dx, a.dst[0], a.dst[1], a.dst[2], a.w[0], a.w[1], a.w[2], cos, sin}))
        return set_error(B2D_ERR_ALIGN, "%s: pointers must be 16-byte aligned", what);
    return 0;
}

static int launch_qkv_fwd(const void* src, int64_t ld, int64_t col_off, const QkvSegArgs& a, const void* cos,
                          const void* sin, int B, int S, int H, int head_dim, float eps, void* stream,
                          int per_head = 0) {
    if (head_dim != 64 && head_dim != 128)
        return set_error(B2D_ERR_SHAPE, "qkv_norm_rope: head_dim=%d, the kernels are built for 64 and 128", head_dim);
    if (int rc = check_rowop(B * S, H * head_dim, S)) return rc;
    if ((ld % 8) || (col_off % 8)) return set_error(B2D_ERR_ALIGN, "qkv_norm_rope: ld/col_off must be multiples of 8");
    if (a.nseg < 1 || a.nseg > 3) return set_error(B2D_ERR_SHAPE, "qkv_norm_rope: 1..3 segments");
    if (a.rope_mask && (cos == nullptr || sin == nullptr)) return set_error(B2D_ERR_SHAPE, "qkv_norm_rope: rope needs tables");
    if (int rc = check_qkv_segs(src, nullptr, a, cos, sin, "qkv_norm_rope")) return rc;
    if (per_head && head_dim == 64)
        ROW_DISPATCH_PH(H * 64, per_head_rope_qk_norm_fwd_kernel, 64, B * S, (const __nv_bfloat16*)src, ld, col_off, a,
                        (const float*)cos, (const float*)sin, S, H, eps);
    else if (per_head)
        ROW_DISPATCH_PH(H * 128, per_head_rope_qk_norm_fwd_kernel, 128, B * S, (const __nv_bfloat16*)src, ld, col_off, a,
                        (const float*)cos, (const float*)sin, S, H, eps);
    else if (head_dim == 64)
        ROW_DISPATCH(H * 64, qkv_norm_rope_fwd_kernel, B * S, (const __nv_bfloat16*)src, ld, col_off, a, (const float*)cos,
                     (const float*)sin, S, H, eps);
    else
        ROW_DISPATCH_HD128(H * 128, qkv_norm_rope_fwd_kernel, B * S, (const __nv_bfloat16*)src, ld, col_off, a,
                           (const float*)cos, (const float*)sin, S, H, eps);
    B2D_CHECK_LAUNCH("qkv_norm_rope_fwd");
    return 0;
}

static int launch_qkv_bwd(const void* x, int64_t ld, int64_t col_off, const QkvSegArgs& a, const void* cos,
                          const void* sin, void* dx, int64_t ld_dx, int64_t dx_col_off, int B, int S, int H, int head_dim,
                          float eps, void* stream, int per_head = 0) {
    if (head_dim != 64 && head_dim != 128)
        return set_error(B2D_ERR_SHAPE, "qkv_norm_rope_bwd: head_dim=%d, the kernels are built for 64 and 128", head_dim);
    if (int rc = check_rowop(B * S, H * head_dim, S)) return rc;
    if ((ld % 8) || (col_off % 8) || (ld_dx % 8) || (dx_col_off % 8))
        return set_error(B2D_ERR_ALIGN, "qkv_norm_rope_bwd: ld/col_off must be multiples of 8");
    if (a.nseg < 1 || a.nseg > 3) return set_error(B2D_ERR_SHAPE, "qkv_norm_rope_bwd: 1..3 segments");
    if (a.rope_mask && (cos == nullptr || sin == nullptr)) return set_error(B2D_ERR_SHAPE, "qkv_norm_rope_bwd: rope needs tables");
    if (int rc = check_qkv_segs(x, dx, a, cos, sin, "qkv_norm_rope_bwd")) return rc;
    if (per_head && head_dim == 64)
        ROW_DISPATCH_PH(H * 64, per_head_rope_qk_norm_bwd_kernel, 64, B * S, (const __nv_bfloat16*)x, ld, col_off, a,
                        (const float*)cos, (const float*)sin, (__nv_bfloat16*)dx, ld_dx, dx_col_off, S, H, eps);
    else if (per_head)
        ROW_DISPATCH_PH(H * 128, per_head_rope_qk_norm_bwd_kernel, 128, B * S, (const __nv_bfloat16*)x, ld, col_off, a,
                        (const float*)cos, (const float*)sin, (__nv_bfloat16*)dx, ld_dx, dx_col_off, S, H, eps);
    else if (head_dim == 64)
        ROW_DISPATCH(H * 64, qkv_norm_rope_bwd_kernel, B * S, (const __nv_bfloat16*)x, ld, col_off, a, (const float*)cos,
                     (const float*)sin, (__nv_bfloat16*)dx, ld_dx, dx_col_off, S, H, eps);
    else
        ROW_DISPATCH_HD128(H * 128, qkv_norm_rope_bwd_kernel, B * S, (const __nv_bfloat16*)x, ld, col_off, a,
                           (const float*)cos, (const float*)sin, (__nv_bfloat16*)dx, ld_dx, dx_col_off, S, H, eps);
    B2D_CHECK_LAUNCH("qkv_norm_rope_bwd");
    return 0;
}

extern "C" int b2d_qknorm_rope_fwd(const void* src, int64_t ld, int64_t col_off, const void* weight, const void* cos,
                                   const void* sin, void* dst, int32_t B, int32_t S, int32_t H, int32_t norm,
                                   float eps, void* stream) {
    B2D_BIND(src);
    QkvSegArgs a = {};
    a.nseg = 1;
    a.w[0] = norm ? (const __nv_bfloat16*)weight : nullptr;
    if (norm && weight == nullptr) return set_error(B2D_ERR_SHAPE, "qknorm_rope: norm needs a weight");
    a.dst[0] = (__nv_bfloat16*)dst;
    a.rope_mask = cos != nullptr ? 1 : 0;
    return launch_qkv_fwd(src, ld, col_off, a, cos, sin, B, S, H, 64, eps, stream);
}

extern "C" int b2d_qknorm_rope_bwd(const void* dsrc_heads, const void* x, int64_t ld, int64_t col_off,
                                   const void* weight, const void* cos, const void* sin, void* dx, int64_t ld_dx,
                                   int64_t dx_col_off, int32_t B, int32_t S, int32_t H, int32_t norm, float eps,
                                   void* stream) {
    B2D_BIND(dsrc_heads);
    QkvSegArgs a = {};
    a.nseg = 1;
    a.w[0] = norm ? (const __nv_bfloat16*)weight : nullptr;
    if (norm && weight == nullptr) return set_error(B2D_ERR_SHAPE, "qknorm_rope_bwd: norm needs a weight");
    a.dst[0] = (__nv_bfloat16*)const_cast<void*>(dsrc_heads);
    a.rope_mask = cos != nullptr ? 1 : 0;
    return launch_qkv_bwd(x, ld, col_off, a, cos, sin, dx, ld_dx, dx_col_off, B, S, H, 64, eps, stream);
}

static int qkv_fwd_entry(const void* src, int64_t ld, int64_t col_off, int32_t nseg, const void* w0, const void* w1,
                         const void* w2, int32_t rope_mask, const void* cos, const void* sin, void* dst0, void* dst1,
                         void* dst2, int32_t B, int32_t S, int32_t H, int32_t head_dim, int32_t rope_per_head, float eps,
                         int32_t rows_per_w, int64_t w_stride, void* stream) {
    B2D_BIND(src);
    QkvSegArgs a = {};
    a.nseg = nseg;
    a.w[0] = (const __nv_bfloat16*)w0; a.w[1] = (const __nv_bfloat16*)w1; a.w[2] = (const __nv_bfloat16*)w2;
    a.dst[0] = (__nv_bfloat16*)dst0; a.dst[1] = (__nv_bfloat16*)dst1; a.dst[2] = (__nv_bfloat16*)dst2;
    a.rope_mask = rope_mask;
    a.rows_per_w = rows_per_w; a.w_stride = w_stride;
    if (rows_per_w < 0 || (w_stride % 8) != 0) return set_error(B2D_ERR_ARG, "qkv_norm_rope: bad weight stacking");
    return launch_qkv_fwd(src, ld, col_off, a, cos, sin, B, S, H, head_dim, eps, stream, rope_per_head);
}

extern "C" int b2d_qkv_norm_rope_hd_fwd(const void* src, int64_t ld, int64_t col_off, int32_t nseg, const void* w0,
                                        const void* w1, const void* w2, int32_t rope_mask, const void* cos,
                                        const void* sin, void* dst0, void* dst1, void* dst2, int32_t B, int32_t S,
                                        int32_t H, int32_t head_dim, float eps, int32_t rows_per_w, int64_t w_stride,
                                        void* stream) {
    return qkv_fwd_entry(src, ld, col_off, nseg, w0, w1, w2, rope_mask, cos, sin, dst0, dst1, dst2, B, S, H, head_dim, 0,
                         eps, rows_per_w, w_stride, stream);
}

extern "C" int b2d_qkv_norm_rope_ph_fwd(const void* src, int64_t ld, int64_t col_off, int32_t nseg, const void* w0,
                                        const void* w1, const void* w2, int32_t rope_mask, const void* cos,
                                        const void* sin, void* dst0, void* dst1, void* dst2, int32_t B, int32_t S,
                                        int32_t H, int32_t head_dim, float eps, int32_t rows_per_w, int64_t w_stride,
                                        void* stream) {
    return qkv_fwd_entry(src, ld, col_off, nseg, w0, w1, w2, rope_mask, cos, sin, dst0, dst1, dst2, B, S, H, head_dim, 1,
                         eps, rows_per_w, w_stride, stream);
}

extern "C" int b2d_qkv_norm_rope_fwd(const void* src, int64_t ld, int64_t col_off, int32_t nseg, const void* w0,
                                     const void* w1, const void* w2, int32_t rope_mask, const void* cos, const void* sin,
                                     void* dst0, void* dst1, void* dst2, int32_t B, int32_t S, int32_t H, float eps,
                                     int32_t rows_per_w, int64_t w_stride, void* stream) {
    return b2d_qkv_norm_rope_hd_fwd(src, ld, col_off, nseg, w0, w1, w2, rope_mask, cos, sin, dst0, dst1, dst2, B, S, H, 64,
                                    eps, rows_per_w, w_stride, stream);
}

static int qkv_bwd_entry(const void* dy0, const void* dy1, const void* dy2, const void* x, int64_t ld, int64_t col_off,
                         int32_t nseg, const void* w0, const void* w1, const void* w2, int32_t rope_mask, const void* cos,
                         const void* sin, void* dx, int64_t ld_dx, int64_t dx_col_off, int32_t B, int32_t S, int32_t H,
                         int32_t head_dim, int32_t rope_per_head, float eps, int32_t rows_per_w, int64_t w_stride,
                         void* stream) {
    B2D_BIND(dy0);
    QkvSegArgs a = {};
    a.nseg = nseg;
    a.w[0] = (const __nv_bfloat16*)w0; a.w[1] = (const __nv_bfloat16*)w1; a.w[2] = (const __nv_bfloat16*)w2;
    a.dst[0] = (__nv_bfloat16*)const_cast<void*>(dy0);
    a.dst[1] = (__nv_bfloat16*)const_cast<void*>(dy1);
    a.dst[2] = (__nv_bfloat16*)const_cast<void*>(dy2);
    a.rope_mask = rope_mask;
    a.rows_per_w = rows_per_w; a.w_stride = w_stride;
    if (rows_per_w < 0 || (w_stride % 8) != 0) return set_error(B2D_ERR_ARG, "qkv_norm_rope_bwd: bad weight stacking");
    return launch_qkv_bwd(x, ld, col_off, a, cos, sin, dx, ld_dx, dx_col_off, B, S, H, head_dim, eps, stream,
                          rope_per_head);
}

extern "C" int b2d_qkv_norm_rope_hd_bwd(const void* dy0, const void* dy1, const void* dy2, const void* x, int64_t ld,
                                        int64_t col_off, int32_t nseg, const void* w0, const void* w1, const void* w2,
                                        int32_t rope_mask, const void* cos, const void* sin, void* dx, int64_t ld_dx,
                                        int64_t dx_col_off, int32_t B, int32_t S, int32_t H, int32_t head_dim, float eps,
                                        int32_t rows_per_w, int64_t w_stride, void* stream) {
    return qkv_bwd_entry(dy0, dy1, dy2, x, ld, col_off, nseg, w0, w1, w2, rope_mask, cos, sin, dx, ld_dx, dx_col_off, B,
                         S, H, head_dim, 0, eps, rows_per_w, w_stride, stream);
}

extern "C" int b2d_qkv_norm_rope_ph_bwd(const void* dy0, const void* dy1, const void* dy2, const void* x, int64_t ld,
                                        int64_t col_off, int32_t nseg, const void* w0, const void* w1, const void* w2,
                                        int32_t rope_mask, const void* cos, const void* sin, void* dx, int64_t ld_dx,
                                        int64_t dx_col_off, int32_t B, int32_t S, int32_t H, int32_t head_dim, float eps,
                                        int32_t rows_per_w, int64_t w_stride, void* stream) {
    return qkv_bwd_entry(dy0, dy1, dy2, x, ld, col_off, nseg, w0, w1, w2, rope_mask, cos, sin, dx, ld_dx, dx_col_off, B,
                         S, H, head_dim, 1, eps, rows_per_w, w_stride, stream);
}

extern "C" int b2d_qkv_norm_rope_bwd(const void* dy0, const void* dy1, const void* dy2, const void* x, int64_t ld,
                                     int64_t col_off, int32_t nseg, const void* w0, const void* w1, const void* w2,
                                     int32_t rope_mask, const void* cos, const void* sin, void* dx, int64_t ld_dx,
                                     int64_t dx_col_off, int32_t B, int32_t S, int32_t H, float eps, int32_t rows_per_w,
                                     int64_t w_stride, void* stream) {
    return b2d_qkv_norm_rope_hd_bwd(dy0, dy1, dy2, x, ld, col_off, nseg, w0, w1, w2, rope_mask, cos, sin, dx, ld_dx,
                                    dx_col_off, B, S, H, 64, eps, rows_per_w, w_stride, stream);
}

extern "C" int b2d_rope_table(float* cos, float* sin, int32_t F, int32_t H, int32_t W, int32_t D, float sf, float sh,
                              float sw, void* stream) {
    B2D_BIND(cos);
    if (D % 2 || D / 6 < 2) return set_error(B2D_ERR_SHAPE, "rope_table: D must be even and >= 12");
    if (F <= 0 || H <= 0 || W <= 0) return set_error(B2D_ERR_SHAPE, "rope_table: F, H, W must be positive");
    long long n = (long long)F * H * W * (D / 2);
    rope_table_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>(cos, sin, F, H, W, D, sf, sh, sw);
    B2D_CHECK_LAUNCH("rope_table");
    return 0;
}

extern "C" int b2d_rope_table_wan(float* cos, float* sin, int32_t F, int32_t H, int32_t W, int32_t head_dim,
                                  double theta, void* stream) {
    B2D_BIND(cos);
    if (cos == nullptr || sin == nullptr) return set_error(B2D_ERR_ARG, "rope_table_wan: NULL table");
    if (head_dim % 2 || head_dim / 6 < 1) return set_error(B2D_ERR_SHAPE, "rope_table_wan: head_dim must be even and >= 6");
    if (F <= 0 || H <= 0 || W <= 0) return set_error(B2D_ERR_SHAPE, "rope_table_wan: F, H, W must be positive");
    const long long n = (long long)F * H * W * (head_dim / 2);
    rope_table_wan_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>(cos, sin, F, H, W, head_dim, theta);
    B2D_CHECK_LAUNCH("rope_table_wan");
    return 0;
}

extern "C" int b2d_wan_prep(const void* moments, const void* eps, const void* noise, const float* mean, const float* std,
                            const float* sigma, void* x_t, void* target, int32_t B, int32_t C, int32_t F, int32_t H,
                            int32_t W, void* stream) {
    B2D_BIND(moments);
    if (!moments || !eps || !noise || !mean || !std || !sigma || !x_t || !target)
        return set_error(B2D_ERR_ARG, "wan_prep: NULL operand");
    if (B <= 0 || C <= 0 || F <= 0 || H <= 0 || W <= 0 || H % 2 || W % 2)
        return set_error(B2D_ERR_SHAPE, "wan_prep: B, C, F, H, W must be positive, H and W even (B=%d C=%d F=%d H=%d W=%d)",
                         (int)B, (int)C, (int)F, (int)H, (int)W);
    const long long n = (long long)B * C * F * H * W;
    wan_prep_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)moments, (const __nv_bfloat16*)eps, (const __nv_bfloat16*)noise, mean, std, sigma,
        (__nv_bfloat16*)x_t, (__nv_bfloat16*)target, B, C, F, H, W);
    B2D_CHECK_LAUNCH("wan_prep");
    return 0;
}

extern "C" int b2d_wan_i2v_prep(const void* moments, const void* cond_moments, const void* cond_mask, const void* eps,
                                const void* noise, const float* mean, const float* std, const float* sigma, void* x_in,
                                void* target, int32_t B, int32_t C, int32_t Cm, int32_t F, int32_t H, int32_t W,
                                void* stream) {
    B2D_BIND(moments);
    if (!moments || !cond_moments || !cond_mask || !eps || !noise || !mean || !std || !sigma || !x_in || !target)
        return set_error(B2D_ERR_ARG, "wan_i2v_prep: NULL operand");
    if (B <= 0 || C <= 0 || Cm <= 0 || Cm > C || F <= 0 || H <= 0 || W <= 0 || H % 2 || W % 2)
        return set_error(B2D_ERR_SHAPE,
                         "wan_i2v_prep: B, C, Cm, F, H, W must be positive, Cm <= C, H and W even (B=%d C=%d Cm=%d F=%d "
                         "H=%d W=%d)", (int)B, (int)C, (int)Cm, (int)F, (int)H, (int)W);
    const long long n = (long long)B * C * F * H * W;
    wan_prep_kernel<true><<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)moments, (const __nv_bfloat16*)eps, (const __nv_bfloat16*)noise, mean, std, sigma,
        (__nv_bfloat16*)x_in, (__nv_bfloat16*)target, B, C, F, H, W, (const __nv_bfloat16*)cond_moments,
        (const __nv_bfloat16*)cond_mask, Cm);
    B2D_CHECK_LAUNCH("wan_i2v_prep");
    return 0;
}

extern "C" int b2d_gelu_erf(const void* x, void* y, int64_t n, void* stream) {
    if (n <= 0) return 0;
    B2D_BIND(x);
    if (!x || !y) return set_error(B2D_ERR_ARG, "gelu_erf: NULL operand");
    gelu_erf_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y,
                                                                     (long long)n);
    B2D_CHECK_LAUNCH("gelu_erf");
    return 0;
}

extern "C" int b2d_patch_permute(const void* src, void* dst, int32_t B, int32_t C, int32_t F, int32_t H, int32_t W,
                                 int32_t out_order, int32_t unpatchify, void* stream) {
    B2D_BIND(src);
    if (!src || !dst) return set_error(B2D_ERR_ARG, "patch_permute: NULL operand");
    if ((out_order != 0 && out_order != 1) || (unpatchify != 0 && unpatchify != 1))
        return set_error(B2D_ERR_ARG, "patch_permute: out_order and unpatchify are 0 or 1");
    if (B <= 0 || C <= 0 || F <= 0 || H <= 0 || W <= 0 || H % 2 || W % 2)
        return set_error(B2D_ERR_SHAPE, "patch_permute: B, C, F, H, W must be positive, H and W even");
    if (src == dst) return set_error(B2D_ERR_ARG, "patch_permute: src and dst must not be the same buffer");
    const long long n = (long long)B * C * F * H * W;
    patch_permute_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)src, (__nv_bfloat16*)dst, B, C, F, H, W, out_order, unpatchify);
    B2D_CHECK_LAUNCH("patch_permute");
    return 0;
}

extern "C" int b2d_layer_norm_affine_fwd(const void* x, void* y, const void* weight, const void* bias, int32_t rows,
                                         int32_t D, float eps, void* stream) {
    B2D_BIND(x);
    if (!x || !y || !weight || !bias) return set_error(B2D_ERR_ARG, "layer_norm_affine_fwd: NULL operand");
    if (int rc = check_rowop(rows, D, 1)) return rc;
    if (misaligned({x, y, weight, bias}))
        return set_error(B2D_ERR_ALIGN, "layer_norm_affine_fwd: pointers must be 16-byte aligned");
    ROW_DISPATCH_AFFINE(D, norm_modulate_fwd_kernel, rows,
        (const __nv_bfloat16*)x, (__nv_bfloat16*)y, (const __nv_bfloat16*)bias, (const __nv_bfloat16*)nullptr,
        (const __nv_bfloat16*)weight, (const __nv_bfloat16*)nullptr, 0LL, D, 1, eps, 1);
    B2D_CHECK_LAUNCH("layer_norm_affine_fwd");
    return 0;
}

extern "C" int b2d_layer_norm_affine_bwd(const void* dy, const void* x, const void* dx_in, void* dx_out,
                                         const void* weight, const void* gate2_tab, const void* gate2_emb, void* out2,
                                         int64_t emb_stride, int32_t rows, int32_t D, int32_t rows_per_sample, float eps,
                                         void* stream) {
    B2D_BIND(dy);
    if (!dy || !x || !dx_out || !weight) return set_error(B2D_ERR_ARG, "layer_norm_affine_bwd: NULL operand");
    if (out2 != nullptr && (gate2_tab == nullptr || gate2_emb == nullptr))
        return set_error(B2D_ERR_ARG, "layer_norm_affine_bwd: out2 needs gate2_tab and gate2_emb");
    if (int rc = check_rowop(rows, D, rows_per_sample)) return rc;
    if (misaligned({dy, x, dx_in, dx_out, weight, gate2_tab, gate2_emb, out2}) || emb_stride % 8)
        return set_error(B2D_ERR_ALIGN, "layer_norm_affine_bwd: pointers must be 16-byte aligned, emb_stride a multiple of 8");
    ROW_DISPATCH_AFFINE(D, norm_modulate_bwd_kernel, rows,
        (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dx_in, (__nv_bfloat16*)dx_out,
        (const __nv_bfloat16*)weight, (const __nv_bfloat16*)nullptr, (const __nv_bfloat16*)gate2_tab,
        (const __nv_bfloat16*)gate2_emb, (__nv_bfloat16*)out2, emb_stride, D, rows_per_sample, eps, 1);
    B2D_CHECK_LAUNCH("layer_norm_affine_bwd");
    return 0;
}

extern "C" int b2d_prep_noise_pack(const void* latents, const void* noise, const float* mean, const float* std,
                                   const float* sigma, const float* sigma_ff, void* x_t, void* target, int32_t B,
                                   int32_t C, int32_t F, int32_t HW, void* stream) {
    B2D_BIND(latents);
    long long n = (long long)B * C * F * HW;
    if (n <= 0) return set_error(B2D_ERR_SHAPE, "prep: empty");
    prep_noise_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)latents, (const __nv_bfloat16*)noise, mean, std, sigma, sigma_ff, (__nv_bfloat16*)x_t,
        (__nv_bfloat16*)target, B, C, F, HW);
    B2D_CHECK_LAUNCH("prep_noise_pack");
    return 0;
}

extern "C" int b2d_prep_posterior_noise_pack(const void* moments, const void* eps, const void* noise, const float* mean,
                                             const float* std, const float* sigma, const float* sigma_ff, void* x_t,
                                             void* target, void* latents_out, int32_t B, int32_t C, int32_t F,
                                             int32_t HW, void* stream) {
    B2D_BIND(moments);
    if (B <= 0 || C <= 0 || F <= 0 || HW <= 0)
        return set_error(B2D_ERR_SHAPE, "prep_posterior: B, C, F, HW must be positive (B=%d C=%d F=%d HW=%d)", (int)B,
                         (int)C, (int)F, (int)HW);
    long long n = (long long)B * C * F * HW;
    prep_posterior_noise_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)moments, (const __nv_bfloat16*)eps, (const __nv_bfloat16*)noise, mean, std, sigma,
        sigma_ff, (__nv_bfloat16*)x_t, (__nv_bfloat16*)target, (__nv_bfloat16*)latents_out, B, C, F, HW);
    B2D_CHECK_LAUNCH("prep_posterior_noise_pack");
    return 0;
}

constexpr int REDUCE_BLOCKS = B2D_REDUCE_PARTIALS;

extern "C" int b2d_loss_mse(const void* pred, const void* target, const float* weight, float loss_scale,
                            float* loss_out, void* dpred, float* partial_ws, int32_t B, int64_t per_sample,
                            void* stream) {
    B2D_BIND(pred);
    if (B <= 0 || per_sample <= 0) return set_error(B2D_ERR_SHAPE, "loss: B and per_sample must be positive");
    if (per_sample % 8) return set_error(B2D_ERR_SHAPE, "loss: per_sample %% 8");
    if (misaligned({pred, target, dpred})) return set_error(B2D_ERR_ALIGN, "loss: pred, target, dpred must be 16-byte aligned");
    loss_mse_kernel<<<REDUCE_BLOCKS, ROW_THREADS, 0, STREAM>>>((const __nv_bfloat16*)pred, (const __nv_bfloat16*)target,
                                                               weight, loss_scale, (__nv_bfloat16*)dpred, partial_ws, B,
                                                               per_sample);
    B2D_CHECK_LAUNCH("loss_mse");
    final_sum_kernel<<<1, ROW_THREADS, 0, STREAM>>>(partial_ws, REDUCE_BLOCKS, loss_out, 0);
    B2D_CHECK_LAUNCH("loss_final");
    return 0;
}

extern "C" int b2d_timestep_sinusoid(const float* t, void* out, int32_t n, void* stream) {
    B2D_BIND(t);
    if (n <= 0) return 0;
    timestep_sinusoid_kernel<<<(n * 128 + 255) / 256, 256, 0, STREAM>>>(t, (__nv_bfloat16*)out, n);
    B2D_CHECK_LAUNCH("timestep_sinusoid");
    return 0;
}

extern "C" int b2d_cast_f32_bf16(const float* src, void* dst, int64_t n, float scale, void* stream) {
    B2D_BIND(src);
    if (n <= 0) return 0;
    if (misaligned({src}) || misaligned({dst}, 8))
        return set_error(B2D_ERR_ALIGN, "cast_f32_bf16: src must be 16-byte and dst 8-byte aligned");
    long long n4 = (n + 3) / 4;
    cast_f32_bf16_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, STREAM>>>(src, (__nv_bfloat16*)dst, n, scale);
    B2D_CHECK_LAUNCH("cast_f32_bf16");
    return 0;
}

extern "C" int b2d_splitk_reduce_bf16(const float* part, int32_t splits, int32_t M, int32_t N, float alpha, void* out,
                                      int64_t ldc, void* stream) {
    if (part == nullptr || out == nullptr) return set_error(B2D_ERR_ARG, "splitk_reduce_bf16: null pointer");
    B2D_BIND(part);
    if (splits < 1 || splits > B2D_SPLITK_MAX)
        return set_error(B2D_ERR_ARG, "splitk_reduce_bf16: splits = %d outside 1..%d", (int)splits, B2D_SPLITK_MAX);
    if (M <= 0 || N <= 0 || N % 8) return set_error(B2D_ERR_SHAPE, "splitk_reduce_bf16: M, N positive, N %% 8 == 0 (M=%d N=%d)", (int)M, (int)N);
    if (ldc < N) return set_error(B2D_ERR_SHAPE, "splitk_reduce_bf16: ldc %lld < N %d", (long long)ldc, (int)N);
    if (misaligned({part, out}) || ldc % 8)
        return set_error(B2D_ERR_ALIGN, "splitk_reduce_bf16: part and out must be 16-byte aligned, ldc a multiple of 8");
    const long long threads = (long long)M * (N / 8);
    launch_k(splitk_reduce_bf16_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, STREAM, part, (int)splits,
             (int)M, (int)N, alpha, (__nv_bfloat16*)out, (long long)ldc);
    B2D_CHECK_LAUNCH("splitk_reduce_bf16");
    return 0;
}

extern "C" int b2d_upcast_fp8_bf16(const void* src, void* dst, int64_t n, int32_t fmt, void* stream) {
    B2D_BIND(src);
    if (fmt != 0 && fmt != 1) return set_error(B2D_ERR_ARG, "upcast_fp8_bf16: fmt must be 0 (e4m3fn) or 1 (e5m2)");
    if (n <= 0) return 0;
    if (misaligned({src, dst})) return set_error(B2D_ERR_ALIGN, "upcast_fp8_bf16: src and dst must be 16-byte aligned");
    const int nsm = device_sm_count();
    if (nsm <= 0) return set_error(B2D_ERR_CUDA, "upcast_fp8_bf16: cannot query the SM count");
    // 4 CTAs of 256 threads per SM keep enough 128-bit loads in flight to saturate HBM; small n needs fewer
    const long long n16 = (n + 15) / 16;
    const unsigned grid = (unsigned)std::max(1LL, std::min((long long)nsm * 4, (n16 + 255) / 256));
    if (fmt == 0)
        launch_k(upcast_fp8_bf16_kernel<0>, dim3(grid), dim3(256), 0, STREAM, (const uint8_t*)src, (__nv_bfloat16*)dst,
                 (long long)n);
    else
        launch_k(upcast_fp8_bf16_kernel<1>, dim3(grid), dim3(256), 0, STREAM, (const uint8_t*)src, (__nv_bfloat16*)dst,
                 (long long)n);
    B2D_CHECK_LAUNCH("upcast_fp8_bf16");
    return 0;
}

extern "C" int b2d_cfg_euler_step(const void* pred, float* latents, void* x_next, int32_t B, int64_t n, int32_t guided,
                                  float guidance, const float* dt, void* stream) {
    if (pred == nullptr || latents == nullptr || x_next == nullptr || dt == nullptr)
        return set_error(B2D_ERR_ARG, "cfg_euler_step: null pointer");
    B2D_BIND(latents);
    if (B <= 0 || n <= 0)
        return set_error(B2D_ERR_SHAPE, "cfg_euler_step: B and n must be positive (B=%d n=%lld)", (int)B, (long long)n);
    if (misaligned({pred, latents, x_next}))
        return set_error(B2D_ERR_ALIGN, "cfg_euler_step: pred, latents and x_next must be 16-byte aligned");
    const bool cfg = guided != 0;  // the caller built the batch: 2B rows iff guided
    const long long total = (long long)B * n;
    // the second (conditional) block of pred / x_next starts `total` elements in: 16-byte aligned iff total % 8 == 0
    const long long n8 = (!cfg || total % 8 == 0) ? total / 8 : 0;
    const int nsm = device_sm_count();
    if (nsm <= 0) return set_error(B2D_ERR_CUDA, "cfg_euler_step: cannot query the SM count");
    const long long work = n8 ? n8 : total;
    const unsigned grid = (unsigned)std::max(1LL, std::min((long long)nsm * 4, (work + 255) / 256));
    if (cfg)
        launch_k(cfg_euler_step_kernel<true>, dim3(grid), dim3(256), 0, STREAM, (const __nv_bfloat16*)pred, latents,
                 (__nv_bfloat16*)x_next, total, n8, guidance, dt);
    else
        launch_k(cfg_euler_step_kernel<false>, dim3(grid), dim3(256), 0, STREAM, (const __nv_bfloat16*)pred, latents,
                 (__nv_bfloat16*)x_next, total, n8, guidance, dt);
    B2D_CHECK_LAUNCH("cfg_euler_step");
    return 0;
}

extern "C" int b2d_cfg_euler_step_cond(const void* pred, float* latents, void* x_next, int32_t B, int64_t n,
                                       int64_t n_cond, int32_t guided, float guidance, const float* dt, void* stream) {
    if (pred == nullptr || latents == nullptr || x_next == nullptr || dt == nullptr)
        return set_error(B2D_ERR_ARG, "cfg_euler_step_cond: null pointer");
    B2D_BIND(latents);
    if (B <= 0 || n <= 0)
        return set_error(B2D_ERR_SHAPE, "cfg_euler_step_cond: B and n must be positive (B=%d n=%lld)", (int)B,
                         (long long)n);
    if (n_cond < 0 || n_cond >= n)
        return set_error(B2D_ERR_SHAPE, "cfg_euler_step_cond: n_cond must be in [0, n) (n_cond=%lld n=%lld)",
                         (long long)n_cond, (long long)n);
    if (misaligned({pred, latents, x_next}))
        return set_error(B2D_ERR_ALIGN, "cfg_euler_step_cond: pred, latents and x_next must be 16-byte aligned");
    // every sample's (and the conditional block's) start is 16-byte aligned iff n % 8 == 0
    const long long c8 = n % 8 == 0 ? (n_cond + 7) / 8 * 8 : n;
    const int nsm = device_sm_count();
    if (nsm <= 0) return set_error(B2D_ERR_CUDA, "cfg_euler_step_cond: cannot query the SM count");
    const long long work = (long long)B * ((n - c8) / 8 + (c8 - n_cond));
    const unsigned grid = (unsigned)std::max(1LL, std::min((long long)nsm * 4, (work + 255) / 256));
    if (guided != 0)
        launch_k(cfg_euler_step_cond_kernel<true>, dim3(grid), dim3(256), 0, STREAM, (const __nv_bfloat16*)pred,
                 latents, (__nv_bfloat16*)x_next, (int)B, (long long)n, (long long)n_cond, c8, guidance, dt);
    else
        launch_k(cfg_euler_step_cond_kernel<false>, dim3(grid), dim3(256), 0, STREAM, (const __nv_bfloat16*)pred,
                 latents, (__nv_bfloat16*)x_next, (int)B, (long long)n, (long long)n_cond, c8, guidance, dt);
    B2D_CHECK_LAUNCH("cfg_euler_step_cond");
    return 0;
}

extern "C" int b2d_sumsq(const float* x, int64_t n, float* out_sumsq, float* partial_ws, void* stream) {
    B2D_BIND(x);
    if (misaligned({x})) return set_error(B2D_ERR_ALIGN, "sumsq: x must be 16-byte aligned");
    sumsq_kernel<<<REDUCE_BLOCKS, ROW_THREADS, 0, STREAM>>>(x, n, partial_ws);
    B2D_CHECK_LAUNCH("sumsq");
    final_sum_kernel<<<1, ROW_THREADS, 0, STREAM>>>(partial_ws, REDUCE_BLOCKS, out_sumsq, 1);
    B2D_CHECK_LAUNCH("sumsq_final");
    return 0;
}

extern "C" int b2d_adamw_clip(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq, float max_norm,
                              float lr, float beta1, float beta2, float eps, float wd, int32_t step, float grad_div,
                              void* stream) {
    B2D_BIND(p);
    if (n <= 0) return 0;
    float bc1 = 1.f - powf(beta1, (float)step);
    float bc2s = sqrtf(1.f - powf(beta2, (float)step));
    if (misaligned({p, g, m, v}))
        return set_error(B2D_ERR_ALIGN, "adamw_clip: p, g, m, v must be 16-byte aligned");
    adamw_clip_kernel<<<(unsigned)((n / 4 + 1 + 255) / 256), 256, 0, STREAM>>>(p, g, m, v, n, sumsq, max_norm, lr, beta1,
                                                                                beta2, eps, wd, bc1, bc2s, grad_div);
    B2D_CHECK_LAUNCH("adamw_clip");
    return 0;
}
