// b2d_attn.cu — attention for d_head = 64 and 128 on sm_90a warpgroup MMAs (forward + backward), non-causal, optional
// additive key bias.  Every kernel is a template on the head dimension HD.
//
// Layouts: q,k,v,dq,dk,dv are [B, H, S, HD] bf16; out / dout are token-major [B, S, H*HD] so that to_out's GEMM consumes
// them without a transpose.  All of them are addressed through 4-D tensor maps whose box is 64 head-dim columns wide:
// 64 bf16 = 128 B = one 128B-swizzle row.  A tile of HD columns is stored in shared memory as HD/64 such panels (columns
// 0-63 of all its rows, then columns 64-127), each one TMA box.  The same bytes serve as a K-major operand (contract
// over d: k-steps 0-3 read panel 0, k-steps 4-7 panel 1) and as an MN-major operand (contract over the rows: the
// descriptor's leading byte offset is the panel stride).
//
// Every kernel is one producer warpgroup (one elected thread issues TMA into an mbarrier ring) and two math
// warpgroups, each owning 64 rows of the CTA's 128-row tile.  Scores live in wgmma accumulator registers; the
// probabilities / dS are packed to bf16 in registers and fed back as the register A operand of the next MMA (the
// m64nNk16 accumulator layout of a 16-column slice is exactly the A-fragment layout), so they never touch shared memory.
//
// Forward (attn_fwd_kernel), CTA per (128-query tile, b, h): S = Q K_j^T over 128-key tiles, online softmax in the
// log2 domain, O += P V_j.
// Backward = delta pre-pass + two kernels (deterministic: no atomics; a short key range split over query ranges is
// summed by a separate pass in a fixed order):
//   attn_bwd_kernel<true>  (dK/dV): CTA per 128-key tile: S^T = K Q_i^T, dP^T = V dO_i^T, P^T, dS^T -> dV += P^T dO_i,
//                                   dK += dS^T Q_i
//   attn_bwd_kernel<false> (dQ)   : CTA per 128-query tile: S = Q K_j^T, dP = dO V_j^T, dS -> dQ += dS K_j
// The streamed tiles (Q_i, dO_i or K_j, V_j) are YR rows: 128 at d = 64, so that S and dP are m64n128k16 MMAs and the
// per-tile cost (barrier turns, wgmma drains, ring round trip) is paid half as often; 64 at d = 128, where S and dP of
// 128 columns do not fit in registers next to dK and dV, and in the split dK/dV pass.  The per-column terms of a
// streamed tile (-lse log2e and delta, or the key bias) are staged in shared memory by a producer warp, next to the tile.
// The dQ pass is pipelined like the forward: S and dP of tile j+1 are issued with dQ += dS_j K_j.
// Two-context forms (Wan image-to-video cross attention, DUAL template flag): the forward streams a second key / value
// context after the first with its own softmax; the dQ pass streams both contexts into one accumulator.
#include <float.h>
#include <stdlib.h>
#include <type_traits>
#include "b2d_internal.h"
#include "b2d_ptx.cuh"

namespace b2d {

constexpr int ATT_THREADS = 384;  // producer warpgroup + 2 math warpgroups
constexpr int TILE = 128;         // rows of the stationary tile (64 per math warpgroup)
constexpr int PANEL = 64;         // head-dim columns of one 128-byte swizzle row
constexpr int TILE_PANEL_BYTES = TILE * PANEL * 2;  // 16 KB: one panel of a 128-row tile
constexpr int HALF_PANEL_BYTES = 64 * PANEL * 2;    // 8 KB: one panel of a math warpgroup's rows
constexpr int ATT_SMEM_LIMIT = 227 * 1024;          // dynamic shared memory per block on sm_90
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

template <int HD>
struct AttnShape {
    static_assert(HD == 64 || HD == 128, "attention is built for head_dim 64 and 128");
    static constexpr int PANELS = HD / PANEL;
    static constexpr int TILE_BYTES = PANELS * TILE_PANEL_BYTES;  // a 128-row tile
};

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// m64nN accumulator (fp32, N = 16 KK) -> KK register A fragments (bf16) of m64nNk16 MMAs: the 16-column slice kk of
// the accumulator is exactly the A-fragment layout
template <int KK>
__device__ __forceinline__ void acc_to_a(const float (&s)[8 * KK], uint32_t (&a)[KK][4]) {
#pragma unroll
    for (int kk = 0; kk < KK; ++kk) {
        a[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
        a[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
        a[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
        a[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
    }
}

// S (+)= X Y^T for a 64-row warpgroup slice: X [64 x HD] and Y [N x HD] both K-major (contract over d), stored as
// 64-column panels XP and YP bytes apart
template <int N, int HD, int XP, int YP>
__device__ __forceinline__ void mma_xyt(float (&s)[N / 2], uint32_t x_smem, uint32_t y_smem) {
    const uint32_t xlo = sdesc_lo_kmajor(x_smem), ylo = sdesc_lo_kmajor(y_smem);
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) {
        const uint32_t xk = xlo + (k / 4) * (XP >> 4) + (k % 4) * SDESC_KSTEP_KMAJOR;
        const uint32_t yk = ylo + (k / 4) * (YP >> 4) + (k % 4) * SDESC_KSTEP_KMAJOR;
        Wgmma<N, 0, 0>::ss(s, sdesc(xk), sdesc(yk), k > 0 ? 1u : 0u);
    }
}

// O [64 x HD] += A Z, A = register fragments of a [64 x 16*KK] bf16 matrix, Z = [16*KK rows x HD] row-major in smem as
// 64-column panels ZP bytes apart (an MN-major operand: contract over its rows)
template <int KK, int HD, int ZP>
__device__ __forceinline__ void mma_az(float (&o)[HD / 2], const uint32_t (&a)[KK][4], uint32_t z_smem) {
    const uint32_t zlo = HD == PANEL ? sdesc_lo_mnmajor(z_smem) : sdesc_lo_mnmajor(z_smem, ZP);
#pragma unroll
    for (int kk = 0; kk < KK; ++kk) Wgmma<HD, 0, 1>::rs(o, a[kk], sdesc(zlo + kk * SDESC_KSTEP_MNMAJOR), 1u);
}

// a [rows x HD] tile at row `row` of head (b, h): one TMA box per 64-column panel, panels P bytes apart
template <int HD, int P>
__device__ __forceinline__ void tma_load_tile(uint8_t* dst, const CUtensorMap* m, uint64_t* bar, int h, int row, int b) {
#pragma unroll
    for (int i = 0; i < HD / PANEL; ++i) tma_load_4d(dst + i * P, m, bar, i * PANEL, h, row, b);
}

// ================================================================================================
// forward
// ================================================================================================
struct AttnFwdParams {
    CUtensorMap tmQ, tmK, tmV;
    const float* key_bias;  // [B, Sk] or null
    __nv_bfloat16* out;     // [B, Sq, H*HD]
    float* lse;             // [B, H, Sq]
    int B, H, Sq, Sk;
    float scale_log2;  // scale * log2(e)
    // two-context forward only: the second context's keys / values, its lse, and the optional branch outputs
    CUtensorMap tmK2, tmV2;
    float* lse2;                // [B, H, Sq]
    __nv_bfloat16* out_ctx[2];  // bf16(O1), bf16(O2) [B, Sq, H*HD], each optional
    int Sk2;
};

// K/V ring depth: at d = 128 a stage is 64 KB
template <int HD>
constexpr int FWD_STAGES = HD == 64 ? 3 : 2;
template <int HD>
constexpr int FWD_SMEM = AttnShape<HD>::TILE_BYTES /*Q*/ + FWD_STAGES<HD> * 2 * AttnShape<HD>::TILE_BYTES /*K, V*/ + 1024 + 256;
// the two-context forward also keeps bf16(O1) of the CTA's 128 rows in shared memory, after the barriers
template <int HD>
constexpr int FWD_O1_BYTES = TILE * HD * 2;
static_assert(FWD_SMEM<64> + FWD_O1_BYTES<64> <= ATT_SMEM_LIMIT && FWD_SMEM<128> + FWD_O1_BYTES<128> <= ATT_SMEM_LIMIT,
              "attn_fwd shared memory");

// DUAL: two independent softmaxes over two key / value contexts sharing Q (Wan image-to-video cross attention).  The
// ring streams context 1's tiles, then context 2's; each context runs exactly the single-context loop and epilogue
// arithmetic, so its lse and bf16 output are those of a single-context launch.  While context 2 runs, bf16(O1) waits in
// shared memory (each thread's HD / 4 packed words, word-major so that a warp's accesses hit 32 banks): in registers, next
// to O, S and P, it spilled at d = 128 even with a 24 / 240 setmaxnreg split.  out = bf16(float(bf16(O1)) +
// float(bf16(O2))).
template <int HD, bool DUAL = false>
__global__ void __launch_bounds__(ATT_THREADS, 1) attn_fwd_kernel(const __grid_constant__ AttnFwdParams p) {
    constexpr int TILE_BYTES = AttnShape<HD>::TILE_BYTES, STAGES = FWD_STAGES<HD>;
    griddep_launch_dependents();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sKV = smem + TILE_BYTES;  // stage s: K at s * 2 * TILE_BYTES, V right after
    uint64_t* q_bar = reinterpret_cast<uint64_t*>(sKV + STAGES * 2 * TILE_BYTES);
    uint64_t* full_bar = q_bar + 1;
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, bh = blockIdx.y;
    const int b = bh / p.H, h = bh % p.H;
    const int n_kt = (p.Sk + TILE - 1) / TILE;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.tmQ);
        tma_prefetch_desc(&p.tmK);
        tma_prefetch_desc(&p.tmV);
        if constexpr (DUAL) {
            tma_prefetch_desc(&p.tmK2);
            tma_prefetch_desc(&p.tmV2);
        }
        mbar_init(q_bar, 1);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 256);
        }
        fence_mbar_init();
    }
    __syncthreads();
    griddep_wait();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            mbar_expect_tx(q_bar, TILE_BYTES);
            tma_load_tile<HD, TILE_PANEL_BYTES>(sQ, &p.tmQ, q_bar, h, qt * TILE, b);
            int stage = 0;
            uint32_t phase = 0;
            auto stream_kv = [&](const CUtensorMap* mK, const CUtensorMap* mV, int n) {
                for (int j = 0; j < n; ++j) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* sK = sKV + stage * 2 * TILE_BYTES;
                    mbar_expect_tx(&full_bar[stage], 2 * TILE_BYTES);
                    tma_load_tile<HD, TILE_PANEL_BYTES>(sK, mK, &full_bar[stage], h, j * TILE, b);
                    tma_load_tile<HD, TILE_PANEL_BYTES>(sK + TILE_BYTES, mV, &full_bar[stage], h, j * TILE, b);
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            };
            stream_kv(&p.tmK, &p.tmV, n_kt);
            if constexpr (DUAL) stream_kv(&p.tmK2, &p.tmV2, (p.Sk2 + TILE - 1) / TILE);
        }
        return;
    }
    setmaxnreg_inc<232>();
    const int cw = (warp >> 2) - 1, wq = warp & 3;
    const int qd = lane & 3;
    const uint32_t q_smem = smem_u32(sQ) + cw * HALF_PANEL_BYTES;
    const float* kb = (!DUAL && p.key_bias) ? p.key_bias + (long long)b * p.Sk : nullptr;  // DUAL: no key bias
    const float sl2 = p.scale_log2;
    bool second = false;  // DUAL: context 2 is being streamed
    auto sk = [&] { return DUAL && second ? p.Sk2 : p.Sk; };  // keys of the context being streamed

    // key bias of tile j in the log2 domain (0 without a bias and past Sk), loaded while the tile's MMAs run
    // (at d = 128 there is no room for it next to O: there the softmax loads the bias itself)
    float kbias[32];
    auto bias_of = [&](int key) { return (kb != nullptr && key < sk()) ? kb[key] * LOG2E : 0.f; };
    auto load_bias = [&](int j) {
        if (HD != 64) return;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int key = j * TILE + 8 * jj + 2 * qd + e;
                kbias[2 * jj + e] = bias_of(key);
            }
    };
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    // The running max starts at -FLT_MAX, not -inf: while every key so far is masked (-inf) it stays finite, so that
    // corr = exp2(m - m) = 1 and P = exp2(-inf - m) = 0 rather than NaN, with no extra work per tile.  Finite scores
    // are above -FLT_MAX (key-bias contract, include/b2d.h), so the first unmasked one replaces it and gets corr = 0.
    float m[2] = {-FLT_MAX, -FLT_MAX}, l[2] = {0.f, 0.f};
    // S of tile j -> P in place (log2 domain, keys past Sk get -inf: only the last tile can hold such keys); returns
    // the factor that rescales O and l from the previous running max
    auto softmax = [&](float (&s)[64], int j, float (&corr)[2]) {
        float mx[2] = {-INFINITY, -INFINITY};
        if ((j + 1) * TILE > sk()) {
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int key = j * TILE + 8 * jj + 2 * qd + e;
                    const float bias = HD == 64 ? kbias[2 * jj + e] : bias_of(key);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        float v = key < sk() ? fmaf(s[4 * jj + 2 * hh + e], sl2, bias) : -INFINITY;
                        s[4 * jj + 2 * hh + e] = v;
                        mx[hh] = fmaxf(mx[hh], v);
                    }
                }
        } else {
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float bias = HD == 64 ? kbias[2 * jj + e] : bias_of(j * TILE + 8 * jj + 2 * qd + e);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        float v = fmaf(s[4 * jj + 2 * hh + e], sl2, bias);
                        s[4 * jj + 2 * hh + e] = v;
                        mx[hh] = fmaxf(mx[hh], v);
                    }
                }
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
            mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
            const float mn = fmaxf(m[hh], mx[hh]);
            corr[hh] = fast_exp2(m[hh] - mn);  // m = -FLT_MAX on the first tile: 0
            m[hh] = mn;
            l[hh] *= corr[hh];
        }
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float pv = fast_exp2(s[4 * jj + 2 * hh + e] - m[hh]);
                    s[4 * jj + 2 * hh + e] = pv;
                    l[hh] += pv;
                }
    };
    auto rescale_o = [&](const float (&corr)[2]) {
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                o[4 * jj + 2 * hh] *= corr[hh];
                o[4 * jj + 2 * hh + 1] *= corr[hh];
            }
    };
    // The two math warpgroups take turns issuing MMAs (named barriers 1 and 2, warpgroup 0 first), so that one's
    // softmax runs while the other's MMAs keep the tensor cores busy.  Every warpgroup issues n_kt + 1 times per context; the
    // second one's initial arrive stands in for its last one, so no arrival is left pending at exit.
    auto turn_begin = [&] { named_bar_sync(1 + cw, 256); };
    auto turn_end = [&](bool last) {
        if (cw == 0 || !last) named_bar_arrive(2 - cw, 256);
    };
    if (cw == 1) named_bar_arrive(1, 256);

    // Pipelined over key tiles: S_{j+1} = Q K_{j+1}^T is issued together with O += P_j V_j, and its softmax runs while
    // PV_j is still on the tensor cores.  Per element the arithmetic is the same as one tile at a time: O is rescaled
    // by corr_{j+1} after P_j V_j has been added and before P_{j+1} V_{j+1} is.
    mbar_wait(q_bar, 0);
    float s[64], corr[2];
    uint32_t pa[8][4];
    int stage = 0;
    uint32_t phase = 0;
    // streams n key tiles from the ring (from the stage after the current one unless `first`) into O, m, l; `last`:
    // the kernel's final turn
    auto attend = [&](int n, bool first, bool last) {
        if (!first && ++stage == STAGES) {
            stage = 0;
            phase ^= 1;
        }
        mbar_wait(&full_bar[stage], phase);
        turn_begin();
        wgmma_fence();
        mma_xyt<128, HD, TILE_PANEL_BYTES, TILE_PANEL_BYTES>(s, q_smem, smem_u32(sKV + stage * 2 * TILE_BYTES));
        wgmma_commit();
        turn_end(false);
        load_bias(0);
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        softmax(s, 0, corr);  // O is still 0: nothing to rescale
        acc_to_a<8>(s, pa);
        for (int j = 1; j < n; ++j) {
            const int prev = stage;
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1;
            }
            mbar_wait(&full_bar[stage], phase);
            turn_begin();
            wgmma_fence();
            mma_xyt<128, HD, TILE_PANEL_BYTES, TILE_PANEL_BYTES>(s, q_smem, smem_u32(sKV + stage * 2 * TILE_BYTES));
            wgmma_commit();
            mma_az<8, HD, TILE_PANEL_BYTES>(o, pa, smem_u32(sKV + prev * 2 * TILE_BYTES) + TILE_BYTES);
            wgmma_commit();
            turn_end(false);
            load_bias(j);
            wgmma_wait<1>();
            wgmma_fence_regs(s);
            softmax(s, j, corr);
            wgmma_wait<0>();
            wgmma_fence_regs(o);
            mbar_arrive(&empty_bar[prev]);
            rescale_o(corr);
            acc_to_a<8>(s, pa);
        }
        turn_begin();
        wgmma_fence();
        mma_az<8, HD, TILE_PANEL_BYTES>(o, pa, smem_u32(sKV + stage * 2 * TILE_BYTES) + TILE_BYTES);
        wgmma_commit();
        turn_end(last);
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        mbar_arrive(&empty_bar[stage]);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
            l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
        }
    };
    const int r0 = qt * TILE + cw * 64 + wq * 16 + (lane >> 2);
    // a row whose every key is masked has l = 0: out = 0 and lse = +inf, so that its backward terms are 0 too
    auto inv_of = [&](int hh) { return l[hh] > 0.f ? 1.f / l[hh] : 0.f; };
    auto lse_of = [&](int hh) { return l[hh] > 0.f ? (m[hh] + __log2f(l[hh])) * LN2 : INFINITY; };
    auto orow_of = [&](__nv_bfloat16* base, int row) { return base + (((long long)b * p.Sq + row) * p.H + h) * HD; };
    if constexpr (!DUAL) {
        attend(n_kt, true, true);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int row = r0 + 8 * hh;
            if (row >= p.Sq) continue;
            const float inv = inv_of(hh);
            __nv_bfloat16* orow = orow_of(p.out, row);
#pragma unroll
            for (int jj = 0; jj < HD / 8; ++jj)
                *reinterpret_cast<uint32_t*>(orow + 8 * jj + 2 * qd) =
                    pack_bf16x2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
            if (qd == 0) p.lse[(long long)bh * p.Sq + row] = lse_of(hh);
        }
    } else {
        attend(n_kt, true, false);
        // word (jj, hh) of math thread t at o1s[(2 jj + hh) * 256 + t]; only this thread reads it back
        uint32_t* o1s = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(q_bar) + 256) + (threadIdx.x - 128);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int row = r0 + 8 * hh;
            const float inv = inv_of(hh);
            __nv_bfloat16* orow1 = p.out_ctx[0] != nullptr && row < p.Sq ? orow_of(p.out_ctx[0], row) : nullptr;
#pragma unroll
            for (int jj = 0; jj < HD / 8; ++jj) {
                const uint32_t o1 = pack_bf16x2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
                o1s[(2 * jj + hh) * 256] = o1;
                if (orow1 != nullptr) *reinterpret_cast<uint32_t*>(orow1 + 8 * jj + 2 * qd) = o1;
            }
            if (qd == 0 && row < p.Sq) p.lse[(long long)bh * p.Sq + row] = lse_of(hh);
        }
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            m[hh] = -FLT_MAX;
            l[hh] = 0.f;
        }
        second = true;
        attend((p.Sk2 + TILE - 1) / TILE, false, true);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int row = r0 + 8 * hh;
            if (row >= p.Sq) continue;
            const float inv = inv_of(hh);
            __nv_bfloat16* orow = orow_of(p.out, row);
            __nv_bfloat16* orow2 = p.out_ctx[1] != nullptr ? orow_of(p.out_ctx[1], row) : nullptr;
#pragma unroll
            for (int jj = 0; jj < HD / 8; ++jj) {
                const uint32_t o1 = o1s[(2 * jj + hh) * 256];
                const uint32_t o2 = pack_bf16x2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
                if (orow2 != nullptr) *reinterpret_cast<uint32_t*>(orow2 + 8 * jj + 2 * qd) = o2;
                *reinterpret_cast<uint32_t*>(orow + 8 * jj + 2 * qd) =
                    pack_bf16x2(bf16_lo(o1) + bf16_lo(o2), bf16_hi(o1) + bf16_hi(o2));
            }
            if (qd == 0) p.lse2[(long long)bh * p.Sq + row] = lse_of(hh);
        }
    }
}

// ================================================================================================
// backward
// ================================================================================================
// delta[b,h,q] = sum_d out[b,q,h,d] * dout[b,q,h,d]     (HD/8 lanes per head-row, 8 elements each)
template <int HD>
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                                  const float* __restrict__ lse, float* __restrict__ delta, float* __restrict__ nlse2,
                                  int B, int H, int Sq) {
    constexpr int LANES = HD / 8, LOG2_LANES = HD == 64 ? 3 : 4;
    static_assert((1 << LOG2_LANES) == LANES, "lanes per head row");
    griddep_launch_dependents();
    griddep_wait();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * Sq * H * LANES;
    const bool ok = t < total;
    const long long e0 = (ok ? t : 0) * 8;
    uint4 a = *reinterpret_cast<const uint4*>(out + e0);
    uint4 d = *reinterpret_cast<const uint4*>(dout + e0);
    float acc = bf16_lo(a.x) * bf16_lo(d.x) + bf16_hi(a.x) * bf16_hi(d.x) + bf16_lo(a.y) * bf16_lo(d.y) +
                bf16_hi(a.y) * bf16_hi(d.y) + bf16_lo(a.z) * bf16_lo(d.z) + bf16_hi(a.z) * bf16_hi(d.z) +
                bf16_lo(a.w) * bf16_lo(d.w) + bf16_hi(a.w) * bf16_hi(d.w);
#pragma unroll
    for (int o = 1; o < LANES; o <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (ok && (t & (LANES - 1)) == 0) {
        const long long hr = t >> LOG2_LANES;  // (b*Sq + q)*H + h
        const int h = (int)(hr % H);
        const long long bq = hr / H;
        const int q = (int)(bq % Sq);
        const int b = (int)(bq / Sq);
        const long long o = ((long long)b * H + h) * Sq + q;
        delta[o] = acc;
        nlse2[o] = -lse[o] * LOG2E;  // exponent offset in the log2 domain
    }
}

struct AttnBwdParams {
    CUtensorMap tmX1, tmX2, tmY1, tmY2;  // stationary pair (128-row boxes) and streamed pair (YR-row boxes)
    const float* key_bias;               // [B, Sk] or null
    const float* delta;                  // [B, H, Sq]
    const float* nlse2;                  // [B, H, Sq]  = -lse * log2(e), stored right after delta
    __nv_bfloat16* out1;                 // dkv: dV [B,H,Sk,HD]
    __nv_bfloat16* out2;                 // dkv: dK [B,H,Sk,HD];  dq: dQ [B,H,Sq,HD]
    float* acc1;                         // split mode (gridDim.z > 1): fp32 partial dV / dK of query range z at
    float* acc2;                         // acc1 / acc2 + z * part_stride, same layout as dv / dk
    long long part_stride;
    int y_per_split;                     // streamed YR-row tiles per z-slice
    int B, H, Sq, Sk;
    float scale, scale_log2;
    // two-context dQ only: the second context's streamed K / V maps, its delta (its -lse log2e right after, as for delta)
    // and key count
    CUtensorMap tmY3, tmY4;
    const float* delta2;
    int Sk2;
};

constexpr int ATT_MAX_SPLITS = 8;  // query ranges of the split dK/dV pass (workspace: include/b2d.h)
// Streamed tiles of YR rows: one ring stage holds Y1 and Y2 (2 x YR x HD bf16) and the stage's per-column terms
// (2 x YR fp32).
template <int HD, int YR>
struct BwdShape {
    static_assert(YR == 64 || YR == 128, "streamed tiles are 64 or 128 rows");
    static constexpr int Y_PANEL_BYTES = YR * PANEL * 2;  // one panel of a streamed tile
    static constexpr int Y_BYTES = AttnShape<HD>::PANELS * Y_PANEL_BYTES;
    static constexpr int COLS = 2 * YR;                   // floats of per-column terms per stage
    static constexpr int STAGES = HD == 64 && YR == 128 ? 3 : 4;  // 3, 4 and 5 measured within 1 % (DESIGN §4.10)
    static constexpr int SMEM = 2 * AttnShape<HD>::TILE_BYTES + STAGES * (2 * Y_BYTES + COLS * 4) + 1024 + 256;
};
static_assert(BwdShape<64, 64>::SMEM <= ATT_SMEM_LIMIT && BwdShape<64, 128>::SMEM <= ATT_SMEM_LIMIT &&
                  BwdShape<128, 64>::SMEM <= ATT_SMEM_LIMIT,
              "attn_bwd shared memory");
// Registers per thread after setmaxnreg.  At d = 128 a dK/dV math thread holds dV and dK (64 + 64 fp32) next to S and dP
// (32 + 32); the producer gives up 16 more registers so that this fits.  At d = 64 (dV, dK 32 + 32 next to S, dP 64 + 64
// with 128-row streamed tiles) 232 is enough.  Both splits keep the 384-thread total at the launch allocation
// (168 x 384), so setmaxnreg.inc never waits for registers another CTA holds.
template <int HD>
constexpr int BWD_REGS_PRODUCER = HD == 64 ? 40 : 24;
template <int HD>
constexpr int BWD_REGS_MATH = HD == 64 ? 232 : 240;
static_assert(BWD_REGS_PRODUCER<64> * 128 + BWD_REGS_MATH<64> * 256 == 168 * ATT_THREADS &&
                  BWD_REGS_PRODUCER<128> * 128 + BWD_REGS_MATH<128> * 256 == 168 * ATT_THREADS,
              "setmaxnreg split");

// Shared skeleton: X1, X2 = stationary [128 x HD] tiles (X rows = this CTA's rows), Y1, Y2 = streamed [YR x HD] tiles.
//   DKV : X = (K, V), Y = (Q, dO):  S^T = K Q^T, dP^T = V dO^T;  dV += P^T dO, dK += dS^T Q
//   !DKV: X = (Q, dO), Y = (K, V):  S = Q K^T,   dP = dO V^T;    dQ += dS K
// In both, the accumulator rows are the CTA's rows and its YR columns are the streamed rows; the probability of
// (query, key) is exp2(s * scale log2e + bias[key] log2e - lse[query] log2e).
//
// DUAL (dQ only, no key bias): the streamed tiles are context 1's K / V tiles, then context 2's, into the one fp32 dQ
// accumulator; the row terms (-lse log2e, delta) switch to context 2's at its first tile.
//
// Producer warpgroup: warp 0 issues the TMA loads of the ring, warp 1 fills each stage's per-column terms (columns =
// streamed rows: DKV -> -lse log2e and delta of the queries, !DKV -> key bias log2e of the keys, 0 without a bias;
// 0 past S_y) with plain loads: a bulk copy would need 16-byte aligned rows, and bh * Sq * 4 bytes is not for odd Sq.
// A stage's full barrier completes when both have arrived (count 2, plus the TMA bytes).
template <bool DKV, int HD, int YR, bool DUAL = false>
__global__ void __launch_bounds__(ATT_THREADS, 1) attn_bwd_kernel(const __grid_constant__ AttnBwdParams p) {
    static_assert(!(DKV && DUAL), "the two-context backward has no dK / dV pass for its second context");
    using Shape = BwdShape<HD, YR>;
    constexpr int TILE_BYTES = AttnShape<HD>::TILE_BYTES, Y_BYTES = Shape::Y_BYTES, STAGES = Shape::STAGES;
    constexpr int COLS = Shape::COLS, KK = YR / 16;
    griddep_launch_dependents();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sX = smem;                   // X1 then X2
    uint8_t* sY = smem + 2 * TILE_BYTES;  // stage s: Y1 at s * 2 * Y_BYTES, Y2 right after
    float* sC = reinterpret_cast<float*>(sY + STAGES * 2 * Y_BYTES);  // stage s: COLS floats at s * COLS
    uint64_t* x_bar = reinterpret_cast<uint64_t*>(sC + STAGES * COLS);
    uint64_t* full_bar = x_bar + 1;
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int xt = blockIdx.x, bh = blockIdx.y;
    const int b = bh / p.H, h = bh % p.H;
    const int S_x = DKV ? p.Sk : p.Sq, S_y = DKV ? p.Sq : p.Sk;
    // streamed tiles [y_begin, y_end) of this z-slice; each role computes the end itself, after its setmaxnreg (a value
    // live across the register reallocation is kept in local memory)
    const int y_begin = blockIdx.z * p.y_per_split;
    auto y_end_of_slice = [&] {
        if constexpr (DUAL) return (S_y + YR - 1) / YR + (p.Sk2 + YR - 1) / YR;
        return min((S_y + YR - 1) / YR, y_begin + p.y_per_split);
    };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.tmX1);
        tma_prefetch_desc(&p.tmX2);
        tma_prefetch_desc(&p.tmY1);
        tma_prefetch_desc(&p.tmY2);
        if constexpr (DUAL) {
            tma_prefetch_desc(&p.tmY3);
            tma_prefetch_desc(&p.tmY4);
        }
        mbar_init(x_bar, 1);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 2);
            mbar_init(&empty_bar[i], 256);
        }
        fence_mbar_init();
    }
    __syncthreads();
    griddep_wait();

    if (warp < 4) {
        setmaxnreg_dec<BWD_REGS_PRODUCER<HD>>();
        const int y_end = y_end_of_slice();
        if (warp == 0 && elect_one()) {
            mbar_expect_tx(x_bar, 2 * TILE_BYTES);
            tma_load_tile<HD, TILE_PANEL_BYTES>(sX, &p.tmX1, x_bar, h, xt * TILE, b);
            tma_load_tile<HD, TILE_PANEL_BYTES>(sX + TILE_BYTES, &p.tmX2, x_bar, h, xt * TILE, b);
            int stage = 0;
            uint32_t phase = 0;
            const int n1 = (S_y + YR - 1) / YR;  // DUAL: context 2's tiles follow
            for (int y = y_begin; y < y_end; ++y) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* s1 = sY + stage * 2 * Y_BYTES;
                mbar_expect_tx(&full_bar[stage], 2 * Y_BYTES);
                const bool ctx2 = DUAL && y >= n1;
                const int row = (ctx2 ? y - n1 : y) * YR;
                tma_load_tile<HD, Shape::Y_PANEL_BYTES>(s1, ctx2 ? &p.tmY3 : &p.tmY1, &full_bar[stage], h, row, b);
                tma_load_tile<HD, Shape::Y_PANEL_BYTES>(s1 + Y_BYTES, ctx2 ? &p.tmY4 : &p.tmY2, &full_bar[stage], h, row, b);
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        } else if (warp == 1) {
            const float* kb = (!DUAL && p.key_bias) ? p.key_bias + (long long)b * p.Sk : nullptr;
            const float* nlse2 = p.nlse2 + (long long)bh * p.Sq;
            const float* delta = p.delta + (long long)bh * p.Sq;
            int stage = 0;
            uint32_t phase = 0;
            for (int y = y_begin; y < y_end; ++y) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                float* c_off = sC + stage * COLS;  // then c_delta = c_off + YR (DKV)
#pragma unroll
                for (int i = lane; i < YR; i += 32) {
                    const int c = y * YR + i;
                    const bool ok = c < S_y;
                    if (DKV) {
                        c_off[i] = ok ? nlse2[c] : 0.f;
                        c_off[YR + i] = ok ? delta[c] : 0.f;
                    } else {
                        c_off[i] = (ok && kb != nullptr) ? kb[c] * LOG2E : 0.f;
                    }
                }
                __syncwarp();
                if (elect_one()) mbar_arrive(&full_bar[stage]);
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
        return;
    }
    setmaxnreg_inc<BWD_REGS_MATH<HD>>();
    const int y_end = y_end_of_slice();
    const int cw = (warp >> 2) - 1, wq = warp & 3;
    const int qd = lane & 3;
    const uint32_t x1 = smem_u32(sX) + cw * HALF_PANEL_BYTES, x2 = x1 + TILE_BYTES;
    const float* kb = (!DUAL && p.key_bias) ? p.key_bias + (long long)b * p.Sk : nullptr;
    const float* nlse2 = p.nlse2 + (long long)bh * p.Sq;
    const float* delta = p.delta + (long long)bh * p.Sq;
    // -lse log2e of query q.  At d = 128 it is read as delta[q + B H Sq]: one pointer fewer than nlse2[q] is what keeps
    // the dK/dV pass free of spills.  d = 64 keeps nlse2[q]: the other form changed its register allocation and made its
    // backward 2 % slower on an H100.
    const int nq = p.B * p.H * p.Sq;
    auto neg_lse2 = [&](int q) { return HD == 64 ? nlse2[q] : delta[q + nq]; };
    const float sl2 = p.scale_log2;
    const int r0 = xt * TILE + cw * 64 + wq * 16 + (lane >> 2);  // this thread's rows r0, r0 + 8

    // per-row terms: DKV rows are keys (bias), !DKV rows are queries (-lse, delta)
    float row_off[2], row_delta[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int r = r0 + 8 * hh;
        if (DKV) {
            row_off[hh] = (kb != nullptr && r < p.Sk) ? kb[r] * LOG2E : 0.f;
            row_delta[hh] = 0.f;
        } else {
            row_off[hh] = r < p.Sq ? neg_lse2(r) : 0.f;
            row_delta[hh] = r < p.Sq ? delta[r] : 0.f;
        }
    }
    // DUAL: context 2's row terms (its -lse log2e is stored right after its delta, as context 1's)
    auto switch_rows = [&] {
        const float* delta2 = p.delta2 + (long long)bh * p.Sq;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = r0 + 8 * hh;
            row_off[hh] = r < p.Sq ? delta2[r + nq] : 0.f;
            row_delta[hh] = r < p.Sq ? delta2[r] : 0.f;
        }
    };
    float acc1[HD / 2], acc2[HD / 2];  // DKV: dV, dK;  !DKV: (unused), dQ
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) acc1[i] = acc2[i] = 0.f;
    float s[YR / 2], dp[YR / 2];
    // S -> P, dP -> dS in place, with the stage's per-column terms from shared memory; only the last streamed tile can
    // hold columns past S_y
    auto elementwise = [&](int y, int sy, const float* cols, auto ragged) {
#pragma unroll
        for (int jj = 0; jj < YR / 8; ++jj) {
            const float2 c_off = *reinterpret_cast<const float2*>(cols + 8 * jj + 2 * qd);
            const float2 c_delta = DKV ? *reinterpret_cast<const float2*>(cols + YR + 8 * jj + 2 * qd) : c_off;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const bool ok = !decltype(ragged)::value || y * YR + 8 * jj + 2 * qd + e < sy;
                const float co = e ? c_off.y : c_off.x;
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int i = 4 * jj + 2 * hh + e;
                    const float pr = ok ? fast_exp2(fmaf(s[i], sl2, row_off[hh] + co)) : 0.f;
                    const float dl = DKV ? (e ? c_delta.y : c_delta.x) : row_delta[hh];
                    s[i] = pr;
                    dp[i] = pr * (dp[i] - dl);
                }
            }
        }
    };
    // Ping-pong: the math warpgroups take turns issuing MMAs (named barriers 1 and 2, warpgroup 0 first), so that one's
    // elementwise pass runs while the other's MMAs keep the tensor cores busy.  Each warpgroup issues twice per streamed
    // tile; the second one's initial arrive stands in for its last one, so no arrival is left pending at exit.
    auto turn_begin = [&] { named_bar_sync(1 + cw, 256); };
    auto turn_end = [&](bool last) {
        if (cw == 0 || !last) named_bar_arrive(2 - cw, 256);
    };
    mbar_wait(x_bar, 0);
    if (cw == 1) named_bar_arrive(1, 256);
    int stage = 0;
    uint32_t phase = 0;
    auto advance = [&] {
        if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
        }
    };
    auto y1_of = [&](int st) { return smem_u32(sY + st * 2 * Y_BYTES); };  // Y2 is Y_BYTES further
    auto issue_s_dp = [&] {  // S, dP of the tile in `stage`, one commit group
        mma_xyt<YR, HD, TILE_PANEL_BYTES, Shape::Y_PANEL_BYTES>(s, x1, y1_of(stage));
        mma_xyt<YR, HD, TILE_PANEL_BYTES, Shape::Y_PANEL_BYTES>(dp, x2, y1_of(stage) + Y_BYTES);
        wgmma_commit();
    };
    auto elementwise_tile = [&](int y) {
        const float* cols = sC + stage * COLS;
        int sy = S_y;
        if constexpr (DUAL) {
            const int n1 = (S_y + YR - 1) / YR;
            if (y == n1) switch_rows();
            if (y >= n1) {
                y -= n1;
                sy = p.Sk2;
            }
        }
        if ((y + 1) * YR > sy)
            elementwise(y, sy, cols, std::true_type{});
        else
            elementwise(y, sy, cols, std::false_type{});
    };
    uint32_t pa[KK][4], da[KK][4];
    if constexpr (DKV) {
        // two turns per streamed tile; dV and dK next to S and dP leave no registers for a second tile's operands
        for (int y = y_begin; y < y_end; ++y) {
            mbar_wait(&full_bar[stage], phase);
            turn_begin();
            wgmma_fence();
            issue_s_dp();
            turn_end(false);
            wgmma_wait<0>();
            wgmma_fence_regs(s);
            wgmma_fence_regs(dp);
            elementwise_tile(y);
            acc_to_a<KK>(dp, da);
            const uint32_t y1 = y1_of(stage);
            turn_begin();
            wgmma_fence();
            acc_to_a<KK>(s, pa);
            mma_az<KK, HD, Shape::Y_PANEL_BYTES>(acc1, pa, y1 + Y_BYTES);  // dV += P^T dO
            mma_az<KK, HD, Shape::Y_PANEL_BYTES>(acc2, da, y1);            // dK += dS^T Q
            wgmma_commit();
            turn_end(y + 1 == y_end);
            wgmma_wait<0>();
            wgmma_fence_regs(acc1);
            wgmma_fence_regs(acc2);
            mbar_arrive(&empty_bar[stage]);
            advance();
        }
    } else {
        // Pipelined over streamed tiles like the forward: S and dP of tile y are issued in the same turn as
        // dQ += dS_{y-1} K_{y-1}, and tile y's elementwise pass runs while that MMA is still on the tensor cores.  dQ
        // takes the same k-steps in the same order as one tile at a time.  One turn per tile plus a last one.
        mbar_wait(&full_bar[stage], phase);
        turn_begin();
        wgmma_fence();
        issue_s_dp();
        turn_end(false);
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        wgmma_fence_regs(dp);
        elementwise_tile(y_begin);
        acc_to_a<KK>(dp, da);
        for (int y = y_begin + 1; y < y_end; ++y) {
            const int prev = stage;
            advance();
            mbar_wait(&full_bar[stage], phase);
            turn_begin();
            wgmma_fence();
            issue_s_dp();
            mma_az<KK, HD, Shape::Y_PANEL_BYTES>(acc2, da, y1_of(prev));  // dQ += dS K
            wgmma_commit();
            turn_end(false);
            wgmma_wait<1>();
            wgmma_fence_regs(s);
            wgmma_fence_regs(dp);
            elementwise_tile(y);
            wgmma_wait<0>();
            wgmma_fence_regs(acc2);
            mbar_arrive(&empty_bar[prev]);
            acc_to_a<KK>(dp, da);
        }
        turn_begin();
        wgmma_fence();
        mma_az<KK, HD, Shape::Y_PANEL_BYTES>(acc2, da, y1_of(stage));  // dQ += dS K
        wgmma_commit();
        turn_end(true);
        wgmma_wait<0>();
        wgmma_fence_regs(acc2);
        mbar_arrive(&empty_bar[stage]);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int r = r0 + 8 * hh;
        if (r >= S_x) continue;
        const long long base = ((long long)bh * S_x + r) * HD;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj) {
            const int c = 8 * jj + 2 * qd, i = 4 * jj + 2 * hh;
            const float g0 = acc2[i] * p.scale, g1 = acc2[i + 1] * p.scale;
            if (p.acc2 != nullptr) {
                const long long zoff = (long long)blockIdx.z * p.part_stride;
                *reinterpret_cast<float2*>(p.acc2 + zoff + base + c) = make_float2(g0, g1);
                if (DKV) *reinterpret_cast<float2*>(p.acc1 + zoff + base + c) = make_float2(acc1[i], acc1[i + 1]);
            } else {
                *reinterpret_cast<uint32_t*>(p.out2 + base + c) = pack_bf16x2(g0, g1);
                if (DKV) *reinterpret_cast<uint32_t*>(p.out1 + base + c) = pack_bf16x2(acc1[i], acc1[i + 1]);
            }
        }
    }
}

// dst[i] = bf16(sum_z part[z * stride + i]) for i < 2n (dV then dK), summed in split order so that the result does not
// depend on which split finished first
__global__ void attn_dkv_reduce_kernel(const float* __restrict__ part, int splits, long long stride, long long n,
                                       __nv_bfloat16* __restrict__ dv, __nv_bfloat16* __restrict__ dk) {
    griddep_launch_dependents();
    griddep_wait();
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 >= 2 * n) return;
    float4 a = *reinterpret_cast<const float4*>(part + i);
    for (int z = 1; z < splits; ++z) {
        const float4 v = *reinterpret_cast<const float4*>(part + z * stride + i);
        a.x += v.x;
        a.y += v.y;
        a.z += v.z;
        a.w += v.w;
    }
    __nv_bfloat16* dst = i < n ? dv + i : dk + (i - n);
    *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w));
}

// 4-D map over a head-split view: dims (innermost first) [hd, H, S, B]; strides in elements.  The box is one 64-column
// panel; a tile of hd columns is hd / 64 boxes.
static int make_head_map(CUtensorMap* m, const void* base, int hd, int B, int H, int S, long long stride_h,
                         long long stride_s, long long stride_b, int box_rows = 128) {
    uint64_t dims[4] = {(uint64_t)hd, (uint64_t)H, (uint64_t)S, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)stride_h * 2, (uint64_t)stride_s * 2, (uint64_t)stride_b * 2};
    uint32_t box[4] = {PANEL, 1, (uint32_t)box_rows, 1};
    return make_tmap_nd(m, base, 4, dims, strides, box, 2, 1);
}

// once per (kernel, device): keeps cudaFuncSetAttribute out of steady-state launches (and of CUDA-graph capture).
// Keyed by the kernel's address (template instantiations share one function-pointer TYPE).
static int set_smem(const void* kern, int bytes, const char* name) {
    static const void* done_k[64];
    static int done_dev[64];
    static int n_done = 0;
    int dev = 0;
    cudaGetDevice(&dev);
    for (int i = 0; i < n_done; ++i)
        if (done_k[i] == kern && done_dev[i] == dev) return 0;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return set_error(B2D_ERR_CUDA, "cudaFuncSetAttribute(%s): %s", name, cudaGetErrorString(e));
    if (n_done < 64) {
        done_k[n_done] = kern;
        done_dev[n_done] = dev;
        ++n_done;
    }
    return 0;
}

template <int HD, bool DUAL>
static int attn_fwd(const void* q, const void* k, const void* v, const float* key_bias, void* out, float* lse, int B,
                    int H, int Sq, int Sk, float scale, cudaStream_t st, const void* k2 = nullptr,
                    const void* v2 = nullptr, int Sk2 = 0, float* lse2 = nullptr, void* out1 = nullptr,
                    void* out2 = nullptr) {
    AttnFwdParams p;
    memset(&p, 0, sizeof(p));
    int rc;
    if ((rc = make_head_map(&p.tmQ, q, HD, B, H, Sq, (long long)Sq * HD, HD, (long long)H * Sq * HD))) return rc;
    if ((rc = make_head_map(&p.tmK, k, HD, B, H, Sk, (long long)Sk * HD, HD, (long long)H * Sk * HD))) return rc;
    if ((rc = make_head_map(&p.tmV, v, HD, B, H, Sk, (long long)Sk * HD, HD, (long long)H * Sk * HD))) return rc;
    if (DUAL) {
        if ((rc = make_head_map(&p.tmK2, k2, HD, B, H, Sk2, (long long)Sk2 * HD, HD, (long long)H * Sk2 * HD))) return rc;
        if ((rc = make_head_map(&p.tmV2, v2, HD, B, H, Sk2, (long long)Sk2 * HD, HD, (long long)H * Sk2 * HD))) return rc;
        p.lse2 = lse2;
        p.out_ctx[0] = (__nv_bfloat16*)out1;
        p.out_ctx[1] = (__nv_bfloat16*)out2;
        p.Sk2 = Sk2;
    }
    p.key_bias = key_bias;
    p.out = (__nv_bfloat16*)out;
    p.lse = lse;
    p.B = B; p.H = H; p.Sq = Sq; p.Sk = Sk;
    p.scale_log2 = scale * LOG2E;
    constexpr int smem = FWD_SMEM<HD> + (DUAL ? FWD_O1_BYTES<HD> : 0);
    if ((rc = set_smem((const void*)attn_fwd_kernel<HD, DUAL>, smem, DUAL ? "attn_dual_fwd" : "attn_fwd"))) return rc;
    launch_k(attn_fwd_kernel<HD, DUAL>, dim3((Sq + TILE - 1) / TILE, B * H), dim3(ATT_THREADS), smem, st, p);
    B2D_CHECK_LAUNCH(DUAL ? "attn_dual_fwd" : "attn_fwd");
    return 0;
}

// delta_ws[0, BHSq) = rowsum(out * dout), delta_ws[BHSq, 2 BHSq) = -lse log2e
template <int HD>
static int attn_delta(const void* out, const void* dout, const float* lse, float* delta_ws, int B, int H, int Sq,
                      cudaStream_t st) {
    long long total = (long long)B * Sq * H * (HD / 8);
    launch_k(attn_delta_kernel<HD>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st,
             (const __nv_bfloat16*)out, (const __nv_bfloat16*)dout, lse, delta_ws, delta_ws + (long long)B * H * Sq,
             B, H, Sq);
    B2D_CHECK_LAUNCH("attn_delta");
    return 0;
}

// The streamed tile is 128 rows at d = 64 (64 at d = 128: no register room for a 128-column S and dP next to dK and dV)
// and 64 rows in the split dK/dV pass, whose query ranges and fp32 partials then stay on 64-row boundaries.
template <int HD>
constexpr int BWD_YR = HD == 64 ? 128 : 64;

// the head map of a streamed operand: 128-row boxes when YR = 128, else 64
template <int HD>
static int make_stream_map(CUtensorMap* m, const void* base, int B, int H, int S) {
    const long long hs = (long long)S * HD;
    return make_head_map(m, base, HD, B, H, S, hs, HD, H * hs, BWD_YR<HD> == 128 ? 128 : 64);
}

// dK, dV from delta_ws as attn_delta left it
template <int HD>
static int attn_bwd_dkv(const void* q, const void* k, const void* v, const float* key_bias, const void* dout,
                        float* delta_ws, void* dk, void* dv, int B, int H, int Sq, int Sk, float scale,
                        cudaStream_t st) {
    constexpr int YR = BWD_YR<HD>;
    CUtensorMap mK, mV, mQ, mdO, mQy, mdOy;  // stationary role and YR = 128: 128-row boxes; 64-row boxes
    int rc;
    const long long hs_q = (long long)Sq * HD, hs_k = (long long)Sk * HD, tok = (long long)H * HD;
    if ((rc = make_head_map(&mQ, q, HD, B, H, Sq, hs_q, HD, H * hs_q))) return rc;
    if ((rc = make_head_map(&mK, k, HD, B, H, Sk, hs_k, HD, H * hs_k))) return rc;
    if ((rc = make_head_map(&mV, v, HD, B, H, Sk, hs_k, HD, H * hs_k))) return rc;
    if ((rc = make_head_map(&mdO, dout, HD, B, H, Sq, HD, tok, Sq * tok))) return rc;
    if ((rc = make_head_map(&mQy, q, HD, B, H, Sq, hs_q, HD, H * hs_q, 64))) return rc;
    if ((rc = make_head_map(&mdOy, dout, HD, B, H, Sq, HD, tok, Sq * tok, 64))) return rc;
    const int smem64 = BwdShape<HD, 64>::SMEM, smem_yr = BwdShape<HD, YR>::SMEM;
    if ((rc = set_smem((const void*)attn_bwd_kernel<true, HD, 64>, smem64, "attn_bwd_dkv"))) return rc;
    if ((rc = set_smem((const void*)attn_bwd_kernel<true, HD, YR>, smem_yr, "attn_bwd_dkv"))) return rc;
    AttnBwdParams p;
    memset(&p, 0, sizeof(p));
    p.key_bias = key_bias; p.delta = delta_ws; p.nlse2 = delta_ws + (long long)B * H * Sq;
    p.B = B; p.H = H; p.Sq = Sq; p.Sk = Sk;
    p.scale = scale; p.scale_log2 = scale * LOG2E;
    // With few key tiles (Sk <= 512, e.g. the text keys of cross attention) there are too few CTAs to fill the GPU: the
    // query range is split over gridDim.z (at most ATT_MAX_SPLITS ranges), every range writes its fp32 partial dV / dK
    // to its own slice of the tail of delta_ws, and one pass sums the slices in range order and rounds to bf16 - no
    // atomics, so the result is the same on every run.
    p.tmX1 = mK; p.tmX2 = mV;
    p.out1 = (__nv_bfloat16*)dv; p.out2 = (__nv_bfloat16*)dk;
    const int n_yq = (Sq + 63) / 64;
    const int kv_ctas = ((Sk + TILE - 1) / TILE) * B * H;
    const int nsm = device_sm_count();
    if (nsm <= 0) return B2D_ERR_CUDA;
    int splits = 1;
    if (Sk <= 512 && kv_ctas < nsm && n_yq >= 8) splits = min(ATT_MAX_SPLITS, min(n_yq / 4, (nsm + kv_ctas - 1) / kv_ctas));
    p.y_per_split = (n_yq + splits - 1) / splits;
    splits = (n_yq + p.y_per_split - 1) / p.y_per_split;
    if (splits > 1) {
        const long long n_kv = (long long)B * H * Sk * HD;
        p.tmY1 = mQy; p.tmY2 = mdOy;
        p.acc1 = delta_ws + 2LL * B * H * Sq;
        p.acc2 = p.acc1 + n_kv;
        p.part_stride = 2 * n_kv;
        launch_k(attn_bwd_kernel<true, HD, 64>, dim3((Sk + TILE - 1) / TILE, B * H, splits), dim3(ATT_THREADS), smem64,
                 st, p);
        B2D_CHECK_LAUNCH("attn_bwd_dkv(split)");
        launch_k(attn_dkv_reduce_kernel, dim3((unsigned)((2 * n_kv / 4 + 255) / 256)), dim3(256), 0, st, (const float*)p.acc1,
                 splits, 2 * n_kv, n_kv, (__nv_bfloat16*)dv, (__nv_bfloat16*)dk);
        B2D_CHECK_LAUNCH("attn_bwd_dkv(reduce)");
    } else {
        p.tmY1 = YR == 128 ? mQ : mQy; p.tmY2 = YR == 128 ? mdO : mdOy;
        p.y_per_split = (Sq + YR - 1) / YR;
        launch_k(attn_bwd_kernel<true, HD, YR>, dim3((Sk + TILE - 1) / TILE, B * H), dim3(ATT_THREADS), smem_yr, st, p);
        B2D_CHECK_LAUNCH("attn_bwd_dkv");
    }
    return 0;
}

// dQ from delta_ws as attn_delta left it; DUAL: then context 2's key tiles (k2, v2, Sk2) with its row terms in delta2_ws
template <int HD, bool DUAL>
static int attn_bwd_dq(const void* q, const void* k, const void* v, const float* key_bias, const void* dout,
                       const float* delta_ws, void* dq, int B, int H, int Sq, int Sk, float scale, cudaStream_t st,
                       const void* k2 = nullptr, const void* v2 = nullptr, int Sk2 = 0,
                       const float* delta2_ws = nullptr) {
    constexpr int YR = BWD_YR<HD>;
    AttnBwdParams p;
    memset(&p, 0, sizeof(p));
    int rc;
    const long long hs_q = (long long)Sq * HD, tok = (long long)H * HD;
    if ((rc = make_head_map(&p.tmX1, q, HD, B, H, Sq, hs_q, HD, H * hs_q))) return rc;
    if ((rc = make_head_map(&p.tmX2, dout, HD, B, H, Sq, HD, tok, Sq * tok))) return rc;
    if ((rc = make_stream_map<HD>(&p.tmY1, k, B, H, Sk))) return rc;
    if ((rc = make_stream_map<HD>(&p.tmY2, v, B, H, Sk))) return rc;
    if (DUAL) {
        if ((rc = make_stream_map<HD>(&p.tmY3, k2, B, H, Sk2))) return rc;
        if ((rc = make_stream_map<HD>(&p.tmY4, v2, B, H, Sk2))) return rc;
        p.delta2 = delta2_ws;
        p.Sk2 = Sk2;
    }
    const int smem_yr = BwdShape<HD, YR>::SMEM;
    if ((rc = set_smem((const void*)attn_bwd_kernel<false, HD, YR, DUAL>, smem_yr, DUAL ? "attn_dual_bwd_dq" : "attn_bwd_dq")))
        return rc;
    p.key_bias = key_bias; p.delta = delta_ws; p.nlse2 = delta_ws + (long long)B * H * Sq;
    p.B = B; p.H = H; p.Sq = Sq; p.Sk = Sk;
    p.scale = scale; p.scale_log2 = scale * LOG2E;
    p.out2 = (__nv_bfloat16*)dq;
    p.y_per_split = (Sk + YR - 1) / YR;
    launch_k(attn_bwd_kernel<false, HD, YR, DUAL>, dim3((Sq + TILE - 1) / TILE, B * H), dim3(ATT_THREADS), smem_yr, st, p);
    B2D_CHECK_LAUNCH(DUAL ? "attn_dual_bwd_dq" : "attn_bwd_dq");
    return 0;
}

template <int HD>
static int attn_bwd(const void* q, const void* k, const void* v, const float* key_bias, const void* out,
                    const void* dout, const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int B, int H,
                    int Sq, int Sk, float scale, cudaStream_t st) {
    int rc;
    if ((rc = attn_delta<HD>(out, dout, lse, delta_ws, B, H, Sq, st))) return rc;
    if ((rc = attn_bwd_dkv<HD>(q, k, v, key_bias, dout, delta_ws, dk, dv, B, H, Sq, Sk, scale, st))) return rc;
    return attn_bwd_dq<HD, false>(q, k, v, key_bias, dout, delta_ws, dq, B, H, Sq, Sk, scale, st);
}

// floats of b2d_attn_bwd_hd's workspace (include/b2d.h)
static long long attn_bwd_ws_floats(int B, int H, int Sq, int Sk, int HD) {
    return 2LL * B * H * Sq + (Sk <= 512 ? (long long)ATT_MAX_SPLITS * 2 * B * H * Sk * HD : 0);
}

// context 1: the single-context delta and dK / dV passes on ws; context 2: its delta on the 2 B H Sq floats after them;
// then one dQ launch over both contexts
template <int HD>
static int attn_dual_bwd(const void* q, const void* k1, const void* v1, int Sk1, const void* k2, const void* v2, int Sk2,
                         const void* out1, const void* out2, const void* dout, const float* lse1, const float* lse2,
                         float* ws, void* dq, void* dk1, void* dv1, int B, int H, int Sq, float scale, cudaStream_t st) {
    float* ws2 = ws + attn_bwd_ws_floats(B, H, Sq, Sk1, HD);
    int rc;
    if ((rc = attn_delta<HD>(out1, dout, lse1, ws, B, H, Sq, st))) return rc;
    if ((rc = attn_bwd_dkv<HD>(q, k1, v1, nullptr, dout, ws, dk1, dv1, B, H, Sq, Sk1, scale, st))) return rc;
    if ((rc = attn_delta<HD>(out2, dout, lse2, ws2, B, H, Sq, st))) return rc;
    return attn_bwd_dq<HD, true>(q, k1, v1, nullptr, dout, ws, dq, B, H, Sq, Sk1, scale, st, k2, v2, Sk2, ws2);
}

}  // namespace b2d

using namespace b2d;

extern "C" int b2d_attn_fwd_hd(const void* q, const void* k, const void* v, const float* key_bias, void* out, float* lse,
                               int32_t B, int32_t H, int32_t Sq, int32_t Sk, int32_t head_dim, float scale,
                               void* stream) {
    B2D_BIND(q);
    if (B <= 0 || H <= 0 || Sq <= 0 || Sk <= 0) return set_error(B2D_ERR_SHAPE, "attn_fwd: bad dims");
    if (head_dim != 64 && head_dim != 128)
        return set_error(B2D_ERR_SHAPE, "attn_fwd: head_dim %d is not supported (64 or 128)", (int)head_dim);
    if (reinterpret_cast<uintptr_t>(out) & 31) return set_error(B2D_ERR_ALIGN, "attn_fwd: out must be 32-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return head_dim == 64 ? b2d::attn_fwd<64, false>(q, k, v, key_bias, out, lse, B, H, Sq, Sk, scale, st)
                          : b2d::attn_fwd<128, false>(q, k, v, key_bias, out, lse, B, H, Sq, Sk, scale, st);
}

extern "C" int b2d_attn_bwd_hd(const void* q, const void* k, const void* v, const float* key_bias, const void* out,
                               const void* dout, const float* lse, float* delta_ws, void* dq, void* dk, void* dv,
                               int32_t B, int32_t H, int32_t Sq, int32_t Sk, int32_t head_dim, float scale,
                               void* stream) {
    B2D_BIND(q);
    if (B <= 0 || H <= 0 || Sq <= 0 || Sk <= 0) return set_error(B2D_ERR_SHAPE, "attn_bwd: bad dims");
    if (head_dim != 64 && head_dim != 128)
        return set_error(B2D_ERR_SHAPE, "attn_bwd: head_dim %d is not supported (64 or 128)", (int)head_dim);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return head_dim == 64
               ? b2d::attn_bwd<64>(q, k, v, key_bias, out, dout, lse, delta_ws, dq, dk, dv, B, H, Sq, Sk, scale, st)
               : b2d::attn_bwd<128>(q, k, v, key_bias, out, dout, lse, delta_ws, dq, dk, dv, B, H, Sq, Sk, scale, st);
}

extern "C" int b2d_attn_dual_fwd_hd(const void* q, const void* k1, const void* v1, int32_t Sk1, const void* k2,
                                    const void* v2, int32_t Sk2, void* out, float* lse1, float* lse2, void* out1,
                                    void* out2, int32_t B, int32_t H, int32_t Sq, int32_t head_dim, float scale,
                                    void* stream) {
    B2D_BIND(q);
    if (!q || !k1 || !v1 || !k2 || !v2 || !out || !lse1 || !lse2) return set_error(B2D_ERR_ARG, "attn_dual_fwd: NULL operand");
    if (B <= 0 || H <= 0 || Sq <= 0 || Sk1 <= 0 || Sk2 <= 0) return set_error(B2D_ERR_SHAPE, "attn_dual_fwd: bad dims");
    if (head_dim != 64 && head_dim != 128)
        return set_error(B2D_ERR_SHAPE, "attn_dual_fwd: head_dim %d is not supported (64 or 128)", (int)head_dim);
    if ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(out1) | reinterpret_cast<uintptr_t>(out2)) & 31)
        return set_error(B2D_ERR_ALIGN, "attn_dual_fwd: out, out1, out2 must be 32-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return head_dim == 64
               ? b2d::attn_fwd<64, true>(q, k1, v1, nullptr, out, lse1, B, H, Sq, Sk1, scale, st, k2, v2, Sk2, lse2,
                                         out1, out2)
               : b2d::attn_fwd<128, true>(q, k1, v1, nullptr, out, lse1, B, H, Sq, Sk1, scale, st, k2, v2, Sk2, lse2,
                                          out1, out2);
}

extern "C" int b2d_attn_dual_bwd_hd(const void* q, const void* k1, const void* v1, int32_t Sk1, const void* k2,
                                    const void* v2, int32_t Sk2, const void* out1, const void* out2, const void* dout,
                                    const float* lse1, const float* lse2, float* ws, void* dq, void* dk1, void* dv1,
                                    int32_t B, int32_t H, int32_t Sq, int32_t head_dim, float scale, void* stream) {
    B2D_BIND(q);
    if (!q || !k1 || !v1 || !k2 || !v2 || !out1 || !out2 || !dout || !lse1 || !lse2 || !ws || !dq || !dk1 || !dv1)
        return set_error(B2D_ERR_ARG, "attn_dual_bwd: NULL operand");
    if (B <= 0 || H <= 0 || Sq <= 0 || Sk1 <= 0 || Sk2 <= 0) return set_error(B2D_ERR_SHAPE, "attn_dual_bwd: bad dims");
    if (head_dim != 64 && head_dim != 128)
        return set_error(B2D_ERR_SHAPE, "attn_dual_bwd: head_dim %d is not supported (64 or 128)", (int)head_dim);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return head_dim == 64 ? b2d::attn_dual_bwd<64>(q, k1, v1, Sk1, k2, v2, Sk2, out1, out2, dout, lse1, lse2, ws, dq, dk1,
                                                   dv1, B, H, Sq, scale, st)
                          : b2d::attn_dual_bwd<128>(q, k1, v1, Sk1, k2, v2, Sk2, out1, out2, dout, lse1, lse2, ws, dq,
                                                    dk1, dv1, B, H, Sq, scale, st);
}
