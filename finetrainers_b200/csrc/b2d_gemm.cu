// b2d_gemm.cu — persistent warp-specialised wgmma GEMM for sm_90a.
//
//   warpgroup 0    : TMA producer (one elected thread)   global -> 128B-swizzled smem ring (mbarrier full/empty)
//   warpgroups 1-2 : math, wgmma m64nBNk16 with fp32 accumulators in registers (one k-block of MMAs stays in flight
//                    while the previous stage is released), then the fused epilogue straight from the accumulator
//                    registers (ping-pong: through shared memory and the TMA) to global memory.  Two schedules:
//                    - ping-pong (BN <= 128, more tiles than CTAs; single CTAs, or 2-CTA clusters that share the A
//                      tile of two neighbouring N tiles): each warpgroup owns whole 128 x BN tiles, alternate tiles of
//                      the CTA's work list, and issues two m64 MMAs per k16 step (one per 64-row half).  The
//                      warpgroups take turns on the main loop (named barriers 1 and 2), so one's epilogue runs while
//                      the other's MMAs keep the tensor cores busy.  The epilogue's [M, N] operand (residual or GELU'
//                      aux) and a gate/residual tile's gate vector arrive in shared memory by TMA during the main
//                      loop; out, and then or before it out2, leave by TMA store.
//                    - cooperative (BN > 128, where two 128-row accumulators do not fit, CTA pairs of 256 x BN tiles,
//                      launches with at most one tile per CTA, and gated launches whose tiles can straddle samples or
//                      that have two gates): each warpgroup owns 64 rows of every tile.
//                    The epilogue kind is chosen once per tile and each kind is its own compact unrolled path: a tile
//                    that carried every kind's code behind per-fragment tests ran 100-400 KB of instructions per tile,
//                    far beyond the instruction caches, and serialised each operand load behind the previous pair's
//                    store.  Both schedules issue the same MMAs in the same k-order for every output element, so their
//                    results are bit-identical.
//
// Operands may be K-major or MN-major (transposed views of row-major activations/weights), which covers
// forward (x W^T), backward-dX (dY W) and backward-dW (dY^T X) without materialising transposes.
// An optional second operand pair extends the contraction (LoRA: [x | u] [W | B]^T in one accumulator).
#include "b2d_internal.h"
#include "b2d_ptx.cuh"

namespace b2d {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int GEMM_THREADS = 384;  // producer warpgroup + 2 math warpgroups
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB

struct GemmKParams {
    CUtensorMap tmA, tmB, tmA2, tmB2;
    CUtensorMap tmX;  // ping-pong GATE_RES / MUL_DGELU: res or aux, [M, N] in boxes of 128 rows x 64 columns
    CUtensorMap tmC;  // ping-pong bf16 kinds: out, [batch, M, N] (batch stride c_boff) in boxes of 128 rows x 64 columns
    CUtensorMap tmC2;  // ping-pong, second output: out2, the same layout with leading dimension ldc2
    int M, N, K, K2;
    int a2_group_n;
    int splits, batch;
    int a_brow, a_bcol, b_brow, b_bcol;
    int a2_brow, b2_brow;
    long long c_boff, bias_boff;
    int epi;
    float alpha;
    void* out;
    long long ldc;
    void* out2;
    long long ldc2;
    const __nv_bfloat16* bias;
    const __nv_bfloat16* res;
    long long ldres;
    const __nv_bfloat16* aux;
    long long ldaux;
    const __nv_bfloat16* gate_table;
    const __nv_bfloat16* gate_temb;
    const __nv_bfloat16* gate2_table;
    const __nv_bfloat16* gate2_temb;
    long long temb_stride;
    int rows_per_sample;
    int m_tiles, n_tiles, kb_main, kb_ext, total_work;
};

template <int BN, int B_MN, bool PP>
struct GemmCfg {
    // K-major B: one [BN x 64] box.  MN-major B: ceil(BN/64) boxes of [64 k-rows x 64 n] (BN = 160 loads 192 columns
    // and multiplies the first 160: the last 64-wide atom is used half).
    static constexpr int B_STAGE_BYTES = B_MN ? ((BN + 63) / 64) * 8192 : BN * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
    // ping-pong: one [128 x BN] bf16 tile of the epilogue's [M, N] operand per math warpgroup, the BN columns of one
    // gate's table and temb rows (bf16) per math warpgroup, and the stages that fit beside them in 227 KB (BN = 128:
    // 5 stages + 64 KB + 1 KB; BN = 64: 8 stages + 32 KB + 512 B)
    static constexpr int X_TILE_BYTES = BLOCK_M * BN * 2;
    static constexpr int X_BYTES = PP ? 2 * X_TILE_BYTES : 0;
    static constexpr int G_TILE_BYTES = 2 * BN * 2;
    static constexpr int G_BYTES = PP ? 2 * G_TILE_BYTES : 0;
    static constexpr int STAGE_BUDGET = PP ? 227 * 1024 - 1024 - 256 - X_BYTES - G_BYTES : 220 * 1024;
    static constexpr int STAGES = (STAGE_BUDGET / STAGE_BYTES) > 8 ? 8 : (STAGE_BUDGET / STAGE_BYTES);
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + X_BYTES + G_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(SMEM_BYTES <= 227 * 1024, "GEMM shared memory exceeds the 227 KB a CTA may use on sm_90");
    static_assert(!PP || STAGES == (BN == 128 ? 5 : 8), "ping-pong keeps its ring depth: 5 stages at BN 128, 8 at 64");
};

// bf16 pairs: one 4-byte access.  Every pair starts at an even column, and b2d_gemm admits only 16-byte aligned
// pointers with leading dimensions, batch offsets and temb strides that keep every row 16-byte aligned, so a pair is
// always 4-byte aligned (an fp32 pair 8-byte aligned).  Loads take the read-only path, so that they need not wait for
// the stores of earlier pairs: the kernel never writes what its epilogue reads, except an in-place residual
// (out == res), whose element is read before it is overwritten, by the thread that overwrites it.
__device__ __forceinline__ float2 ld_bf16x2(const __nv_bfloat16* p) {
    return unpack_bf16x2(__ldg(reinterpret_cast<const unsigned int*>(p)));
}
__device__ __forceinline__ void st_bf16x2(__nv_bfloat16* p, float a, float b) {
    *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(a, b);
}

// Byte offset of element (r, c) in a [128 x BN] tile loaded as 64-column TMA boxes of 128 rows with the 128-byte
// swizzle (16-byte chunk k of row r stored at chunk k ^ (r % 8)): the 8 rows one warp reads per column pair then fall
// in 8 different chunks, so its 32 lanes hit 32 different banks.
__device__ __forceinline__ uint32_t x_tile_offset(int r, int c) {
    const uint32_t b = (c & 63) * 2;
    return (c >> 6) * (BLOCK_M * 128) + r * 128 + ((((b >> 4) ^ (r & 7)) << 4) | (b & 15));
}

// Phase timeline of one launch, for tools/gemm_timeline.py: built only with -DB2D_GEMM_TRACE (into a library of its
// own), so the default kernel carries no trace code.  The first thread of each math warpgroup writes %globaltimer stamps
// for each of its tiles into a record of GEMM_TRACE_SLOTS u64; record (cta, t, role) is the CTA's t-th work item seen by
// math warpgroup `role` (0, 1) or by the producer (role 2).  t = max_tiles - 1 is reserved for the warpgroups' exit.
#ifdef B2D_GEMM_TRACE
enum {
    TR_TURN_WAIT, TR_TURN, TR_LAST_MMA, TR_DRAINED, TR_X, TR_PASS1, TR_ST1_ISSUE, TR_ST1_READ, TR_PASS2, TR_ST2_ISSUE,
    TR_ST2_READ, TR_END, TR_SM, TR_MT, TR_NT, TR_KIND, GEMM_TRACE_SLOTS
};
// producer record: TR_TURN_WAIT = ns spent waiting on empty_bar over the tile's k-blocks, TR_TURN / TR_END = first and
// last k-block load issued; TR_KIND: 1 = tile record, 2 = exit record (TR_END = exit time)
struct GemmTrace {
    unsigned long long* buf;
    int max_tiles;
};
__device__ GemmTrace g_gemm_trace;
__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ unsigned long long* trace_rec(int t, int role) {
    if (g_gemm_trace.buf == nullptr || t >= g_gemm_trace.max_tiles) return nullptr;
    return g_gemm_trace.buf + ((size_t)(blockIdx.x * g_gemm_trace.max_tiles + t) * 3 + role) * GEMM_TRACE_SLOTS;
}
__device__ __forceinline__ uint32_t sm_id() {
    uint32_t s;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
    return s;
}
#define B2D_TRACE_ONLY(...) __VA_ARGS__
#define B2D_TSTAMP(slot) \
    if (trec != nullptr && threadIdx.x % 128 == 0) trec[slot] = gtimer()
#else
#define B2D_TRACE_ONLY(...)
#define B2D_TSTAMP(slot)
#endif

// epilogue kinds whose primary output is bf16 (the others are the fp32 store and atomics)
__host__ __device__ constexpr bool gemm_bf16_out(int epi) {
    return epi == B2D_EPI_STORE || epi == B2D_EPI_GELU || epi == B2D_EPI_SILU || epi == B2D_EPI_GATE_RES ||
           epi == B2D_EPI_MUL_DGELU;
}

// What the epilogue of one output pair reads besides the accumulator: bias, the [M, N] operand (res or aux) and the
// gates, loaded ahead of the arithmetic.
struct EpiIn {
    float2 bias, x, g, g2;
};

// What an epilogue pass does with the second output.  Ping-pong tiles write out2 through the x tile in a pass of its own
// (the tile holds one bf16 output at a time): OUT2_PRE writes the GELU / SiLU pre-activation there in place of out, and
// the pass that writes out then skips out2 (OUT2_NONE); the gated copy of a gate/residual tile is made from the stored
// out tile (gemm_gate2_pass).  The cooperative schedule stores both pairs to global memory (OUT2_GLOBAL).
enum { OUT2_GLOBAL = 0, OUT2_NONE = 1, OUT2_PRE = 2 };

// Fused epilogue of the output pair (row, col), (row, col + 1) for the epilogue kind EPI; v0, v1 = alpha * accumulator.
// oc / oc2: element offsets of the pair in out / out2 (batch offset included); sv: when non-null, where the packed bf16
// pair of out goes instead (ping-pong: the tile is written to shared memory and leaves by TMA store).
template <int EPI, int O2>
__device__ __forceinline__ void gemm_epilogue_pair(const GemmKParams& p, long long cbase, long long oc, long long oc2,
                                                   uint32_t* sv, int row, int col, float v0, float v1, const EpiIn& in) {
    if constexpr (EPI == B2D_EPI_F32_ATOMIC) {
        atomicAdd(reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + oc), make_float2(v0, v1));
        return;
    } else if constexpr (EPI == B2D_EPI_F32_ATOMIC_T) {
        float* o = reinterpret_cast<float*>(p.out) + cbase + row;
        atomicAdd(o + (long long)col * p.ldc, v0);
        atomicAdd(o + (long long)(col + 1) * p.ldc, v1);
        return;
    } else {
        if (p.bias != nullptr) {
            v0 += in.bias.x;
            v1 += in.bias.y;
        }
        if constexpr (EPI == B2D_EPI_F32_STORE) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + oc) = make_float2(v0, v1);
            return;
        }
        float u0 = 0.f, u1 = 0.f;
        bool has2 = false;
        if constexpr (EPI == B2D_EPI_GELU || EPI == B2D_EPI_SILU) {
            if constexpr (O2 == OUT2_PRE) {
                *sv = pack_bf16x2(v0, v1);
                return;
            }
            has2 = O2 == OUT2_GLOBAL && p.out2 != nullptr;
            u0 = v0;
            u1 = v1;
            v0 = (EPI == B2D_EPI_GELU) ? gelu_tanh(v0) : silu(v0);
            v1 = (EPI == B2D_EPI_GELU) ? gelu_tanh(v1) : silu(v1);
        } else if constexpr (EPI == B2D_EPI_GATE_RES) {
            v0 = in.x.x + in.g.x * v0;
            v1 = in.x.y + in.g.y * v1;
            if (O2 == OUT2_GLOBAL && p.gate2_table != nullptr && p.out2 != nullptr) {
                has2 = true;
                // the bf16-rounded primary output is what the next op sees
                u0 = __bfloat162float(__float2bfloat16_rn(v0)) * in.g2.x;
                u1 = __bfloat162float(__float2bfloat16_rn(v1)) * in.g2.y;
            }
        } else if constexpr (EPI == B2D_EPI_MUL_DGELU) {
            v0 *= dgelu_tanh(in.x.x);
            v1 *= dgelu_tanh(in.x.y);
        }
        if (sv != nullptr)
            *sv = pack_bf16x2(v0, v1);
        else
            st_bf16x2(reinterpret_cast<__nv_bfloat16*>(p.out) + oc, v0, v1);
        if (has2) st_bf16x2(reinterpret_cast<__nv_bfloat16*>(p.out2) + oc2, u0, u1);
    }
}

// Ping-pong epilogue of a bf16 kind: the warpgroup's whole 128 x BN tile goes to the swizzled shared tile at xs (the
// tile whose origin is (m0, n0)), over the copy of its [M, N] operand (res or aux) that the TMA left there, and leaves by
// TMA store.  Shared memory is read and written four 8 x 8 matrices per warp instruction (ldmatrix / stmatrix: a
// thread's pairs of two column groups and two 8-row halves of one 64-row block): while the other warpgroup's main loop
// streams operands through shared memory, the epilogue's 4-byte accesses, one per column pair and row, each waited for
// the shared-memory pipe and made the epilogue outlast that main loop.  The bias of all of the thread's column pairs is
// loaded before the first is used, instead of one round trip per column chunk.  Every pair is computed, the rows and
// columns past M and N too (their operands are zero-filled, and the bias is 0 there); the TMA store does not write them.
// A ping-pong gate/residual tile lies in one sample and its launch has at most one gate (b2d_gemm keeps the others
// cooperative), so that gate is one vector over the tile's columns: its table and temb slices sit at shared address gs
// (BN bf16 each), and each column pair's gate is read and summed once for all of the thread's rows.
template <int EPI, int BN, int O2>
__device__ __forceinline__ void gemm_epilogue_tile_smem(const GemmKParams& p, const float (&acc)[2][BN / 2], int row0,
                                                        int col0, int z, uint32_t xs, uint32_t gs, int m0, int n0) {
    constexpr bool XS = EPI == B2D_EPI_GATE_RES || EPI == B2D_EPI_MUL_DGELU;
    const int lane = threadIdx.x & 31;
    // the row of matrix lane / 8 = (8-row half h, column group jj) = (lane / 8 % 2, lane / 16) this lane addresses
    const int mrow = (row0 - m0) - (lane >> 2) + 8 * ((lane >> 3) & 1) + (lane & 7);
    const int mcol = 8 * (lane >> 4);
    const __nv_bfloat16* bias = p.bias != nullptr ? p.bias + (long long)z * p.bias_boff : nullptr;
    uint32_t bw[BN / 8];
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int col = col0 + 8 * j;
        bw[j] = (bias != nullptr && col < p.N) ? __ldg(reinterpret_cast<const unsigned int*>(bias + col)) : 0u;
    }
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += 2) {
        uint32_t xv[2][4], ov[2][4];  // per 64-row block b: matrices (h, jj) in registers 2 jj + h
        if constexpr (XS) {
#pragma unroll
            for (int b = 0; b < 2; ++b) ldsm_x4(xs + x_tile_offset(mrow + 64 * b, mcol + 8 * j0), xv[b]);
        }
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int j = j0 + jj;
            const int col = col0 + 8 * j;
            float2 gg = make_float2(1.f, 1.f);
            if constexpr (EPI == B2D_EPI_GATE_RES) {
                if (p.gate_table != nullptr && col < p.N) {
                    const float2 gt = unpack_bf16x2(lds32(gs + (col - n0) * 2));
                    const float2 ge = unpack_bf16x2(lds32(gs + BN * 2 + (col - n0) * 2));
                    gg = make_float2(gt.x + ge.x, gt.y + ge.y);
                }
            }
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int b = r >> 1, h = r & 1, i = 4 * j + 2 * h;
                EpiIn in;
                in.bias = unpack_bf16x2(bw[j]);
                in.x = XS ? unpack_bf16x2(xv[b][2 * jj + h]) : make_float2(1.f, 1.f);
                in.g = gg;
                in.g2 = make_float2(1.f, 1.f);
                gemm_epilogue_pair<EPI, O2>(p, 0, 0, 0, &ov[b][2 * jj + h], 0, col, acc[b][i] * p.alpha,
                                            acc[b][i + 1] * p.alpha, in);
            }
        }
#pragma unroll
        for (int b = 0; b < 2; ++b) stsm_x4(xs + x_tile_offset(mrow + 64 * b, mcol + 8 * j0), ov[b]);
    }
}

// Epilogue of a math warpgroup's accumulator for one epilogue kind, fixed at compile time so that a tile runs only its
// own straight-line code.  The warpgroup owns HALVES blocks of 64 rows (block b starts at row0 + 64 b), and a thread R =
// 2 HALVES rows of them: accumulator acc[b][4j + 2h + e] = (row0 + 64 b + 8h, col0 + 8j + e), thread row r = 2b + h.
// The inputs of CH column groups of all R rows are loaded before any of their pairs is computed, so the loads of a
// chunk overlap each other: CH x R = 8 (column group, row) inputs in flight per chunk in either schedule (CH divides
// BN / 8 for every tile width).  Ping-pong tiles of the bf16 kinds go through shared memory (gemm_epilogue_tile_smem).
template <int EPI, int BN, int HALVES, int O2>
__device__ __forceinline__ void gemm_epilogue_tile(const GemmKParams& p, const float (&acc)[HALVES][BN / 2], int row0,
                                                   int col0, int z, uint32_t xs, uint32_t gs, int m0, int n0) {
    if constexpr (HALVES == 2 && gemm_bf16_out(EPI)) {
        gemm_epilogue_tile_smem<EPI, BN, O2>(p, acc, row0, col0, z, xs, gs, m0, n0);
        return;
    }
    constexpr int R = 2 * HALVES;
    constexpr int CH = 4 / HALVES;
    constexpr bool BF16_IN = EPI != B2D_EPI_F32_ATOMIC && EPI != B2D_EPI_F32_ATOMIC_T;
    const long long cbase = (long long)z * p.c_boff;
    const __nv_bfloat16* bias = p.bias != nullptr ? p.bias + (long long)z * p.bias_boff : nullptr;
    int rows[R], smp[R];  // the thread's rows and their samples (per-sample gates)
#pragma unroll
    for (int r = 0; r < R; ++r) {
        rows[r] = row0 + 64 * (r >> 1) + 8 * (r & 1);
        smp[r] = p.rows_per_sample > 0 ? rows[r] / p.rows_per_sample : 0;
    }
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += CH) {
        EpiIn in[CH][R];
#pragma unroll
        for (int jj = 0; jj < CH; ++jj) {
            const int col = col0 + 8 * (j0 + jj);
            float2 bb = make_float2(0.f, 0.f);
            if (BF16_IN && p.bias != nullptr && col < p.N) bb = ld_bf16x2(bias + col);
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int row = rows[r];
                EpiIn& e = in[jj][r];
                e.bias = bb;
                e.x = e.g = e.g2 = make_float2(1.f, 1.f);
                if (col >= p.N || row >= p.M) continue;
                if constexpr (EPI == B2D_EPI_GATE_RES) {
                    e.x = ld_bf16x2(p.res + (long long)row * p.ldres + col);
                    if (p.gate_table != nullptr) {
                        const float2 gt = ld_bf16x2(p.gate_table + col);
                        const float2 ge = ld_bf16x2(p.gate_temb + (long long)smp[r] * p.temb_stride + col);
                        e.g = make_float2(gt.x + ge.x, gt.y + ge.y);
                    }
                    if (p.gate2_table != nullptr && p.out2 != nullptr) {
                        const float2 gt = ld_bf16x2(p.gate2_table + col);
                        const float2 ge = ld_bf16x2(p.gate2_temb + (long long)smp[r] * p.temb_stride + col);
                        e.g2 = make_float2(gt.x + ge.x, gt.y + ge.y);
                    }
                } else if constexpr (EPI == B2D_EPI_MUL_DGELU) {
                    e.x = ld_bf16x2(p.aux + (long long)row * p.ldaux + col);
                }
            }
        }
#pragma unroll
        for (int jj = 0; jj < CH; ++jj) {
            const int j = j0 + jj;
            const int col = col0 + 8 * j;
            if (col >= p.N) continue;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int row = rows[r], i = 4 * j + 2 * (r & 1);
                if (row < p.M)
                    gemm_epilogue_pair<EPI, O2>(p, cbase, cbase + (long long)row * p.ldc + col,
                                                cbase + (long long)row * p.ldc2 + col, nullptr, row, col,
                                                acc[r >> 1][i] * p.alpha, acc[r >> 1][i + 1] * p.alpha, in[jj][r]);
            }
        }
    }
}

// the launch's epilogue kind is decided once per tile, outside the per-fragment loops
template <int BN, int HALVES>
__device__ __forceinline__ void gemm_epilogue(const GemmKParams& p, const float (&acc)[HALVES][BN / 2], int row0,
                                              int col0, int z, uint32_t xs, uint32_t gs, int m0, int n0) {
    constexpr int O2 = HALVES == 2 ? OUT2_NONE : OUT2_GLOBAL;
#define B2D_EPI_TILE(E) gemm_epilogue_tile<E, BN, HALVES, O2>(p, acc, row0, col0, z, xs, gs, m0, n0)
    switch (p.epi) {
        case B2D_EPI_GELU: B2D_EPI_TILE(B2D_EPI_GELU); break;
        case B2D_EPI_SILU: B2D_EPI_TILE(B2D_EPI_SILU); break;
        case B2D_EPI_GATE_RES: B2D_EPI_TILE(B2D_EPI_GATE_RES); break;
        case B2D_EPI_MUL_DGELU: B2D_EPI_TILE(B2D_EPI_MUL_DGELU); break;
        case B2D_EPI_F32_ATOMIC: B2D_EPI_TILE(B2D_EPI_F32_ATOMIC); break;
        case B2D_EPI_F32_ATOMIC_T: B2D_EPI_TILE(B2D_EPI_F32_ATOMIC_T); break;
        case B2D_EPI_F32_STORE: B2D_EPI_TILE(B2D_EPI_F32_STORE); break;
        case B2D_EPI_STORE:
        default: B2D_EPI_TILE(B2D_EPI_STORE); break;
    }
#undef B2D_EPI_TILE
}

// Ping-pong gate/residual tile with gate2: out2 = bf16(out) * gate2, made in place from the bf16 out tile at xs (after
// its TMA store has read it) with the gate at gs, by the same threads on the same pairs as gemm_epilogue_tile_smem.
// bf16(out) is exactly the value the cooperative schedule multiplies, so out2 is bit-identical to it.
template <int BN>
__device__ __forceinline__ void gemm_gate2_pass(const GemmKParams& p, int row0, int col0, uint32_t xs, uint32_t gs,
                                                int m0, int n0) {
    const int lane = threadIdx.x & 31;
    const int mrow = (row0 - m0) - (lane >> 2) + 8 * ((lane >> 3) & 1) + (lane & 7);
    const int mcol = 8 * (lane >> 4);
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += 2) {
        float2 g2[2];
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int col = col0 + 8 * (j0 + jj);
            g2[jj] = make_float2(1.f, 1.f);
            if (col < p.N) {
                const float2 gt = unpack_bf16x2(lds32(gs + (col - n0) * 2));
                const float2 ge = unpack_bf16x2(lds32(gs + BN * 2 + (col - n0) * 2));
                g2[jj] = make_float2(gt.x + ge.x, gt.y + ge.y);
            }
        }
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const uint32_t a = xs + x_tile_offset(mrow + 64 * b, mcol + 8 * j0);
            uint32_t v[4];
            ldsm_x4(a, v);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 o = unpack_bf16x2(v[k]);
                v[k] = pack_bf16x2(o.x * g2[k >> 1].x, o.y * g2[k >> 1].y);
            }
            stsm_x4(a, v);
        }
    }
}

// one 64-wide k-block of a math warpgroup: per k16 step one m64nBNk16 MMA for each 64-row half it owns (the A tile's
// halves are 8 KB apart in both majornesses: 64 K-major rows, or one 64-column MN-major box)
template <int BN, int TA, int TB, int HALVES>
__device__ __forceinline__ void gemm_kblock(float (&acc)[HALVES][BN / 2], uint32_t alo, uint32_t blo, uint32_t astep,
                                            uint32_t bstep, bool first) {
#pragma unroll
    for (int k = 0; k < BLOCK_K / 16; ++k)
#pragma unroll
        for (int h = 0; h < HALVES; ++h)
            Wgmma<BN, TA, TB>::ss(acc[h], sdesc(alo + h * (8192 >> 4) + k * astep), sdesc(blo + k * bstep),
                                  (!first || k > 0) ? 1u : 0u);
}

// PAIR: the two CTAs of a 2-CTA cluster share one operand tile per k-block; each CTA loads half of it and the TMA
// multicasts that half into the shared memory of both CTAs, so per-SM ingest from L2 drops from 32 KB to 24 KB per
// k-block at BN = 128.  A stage of either CTA is refilled only after the math warpgroups of BOTH CTAs that read it have
// released it.  K-major A, no split-K.
//   cooperative (M-pairs): the CTAs compute the two 128-row halves of one 256 x BN tile and share the B tile; every math
//                          thread arrives on its own and on its peer's empty barrier.
//   ping-pong (N-pairs):   the CTAs compute tiles (m, 2 np) and (m, 2 np + 1) and share the A tile (and the LoRA A2
//                          slice: b2d_gemm pairs only launches whose a2_group_n is a multiple of 2 BN).  Both CTAs walk
//                          the same list of pair items, so warpgroup w of each CTA owns the same tiles and ring stages;
//                          every thread of the owning warpgroup arrives on both CTAs' empty barriers.  With an odd
//                          number of N tiles the last pair's second CTA runs the main loop on zero-filled B (its A half
//                          feeds its peer) and skips the epilogue.  Every epilogue stays per CTA.
template <int BN, int A_MN, int B_MN, bool PAIR, bool PP>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_kernel(const __grid_constant__ GemmKParams p) {
    griddep_launch_dependents();
    static_assert(!PP || BN <= 128, "ping-pong: 2 x BN / 2 accumulators per math thread");
    constexpr int HALVES = PP ? 2 : 1;       // 64-row halves of a tile one math warpgroup owns
    constexpr bool MC_A = PAIR && PP;        // the pair shares (multicasts) A, or B
    constexpr bool MC_B = PAIR && !PP;
    using Cfg = GemmCfg<BN, B_MN, PP>;
    static_assert(!PAIR || A_MN == 0, "CTA pairs take a K-major A operand");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* x_tiles = smem + Cfg::STAGES * Cfg::STAGE_BYTES;  // ping-pong: each math warpgroup's res / aux tile
    uint8_t* g_tiles = x_tiles + Cfg::X_BYTES;                  // ping-pong: each math warpgroup's gate slices
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(g_tiles + Cfg::G_BYTES);
    uint64_t* empty_bar = full_bar + Cfg::STAGES;
    uint64_t* x_bar = empty_bar + Cfg::STAGES;  // ping-pong: x tile of math warpgroup 0 / 1 has landed
    // The ping-pong epilogue reads its [M, N] operand from a copy the TMA made during the main loop, instead of
    // waiting on global loads with one warpgroup's threads.
    const bool stage_x = PP && (p.epi == B2D_EPI_GATE_RES || p.epi == B2D_EPI_MUL_DGELU);
    // ...and writes its bf16 out tile into that buffer, from where one TMA store per tile takes it to global memory:
    // a warp's 4-byte stores of 8 rows each touched 8 rows of L2 sectors, and queued the next chunk's loads behind them.
    const bool smem_out = PP && gemm_bf16_out(p.epi);
    // A gate/residual tile's gate (gate or gate2: b2d_gemm admits at most one, and only tiles inside one sample) comes
    // with the x tile: its table and temb slices over the tile's columns.
    const bool stage_gate = stage_x && p.epi == B2D_EPI_GATE_RES && (p.gate_table != nullptr || p.gate2_table != nullptr);
    // The second output leaves through the x tile too, in a pass of its own: the GELU / SiLU pre-activation before out,
    // the gated copy of a gate/residual tile after it.
    const bool out2_pre = PP && (p.epi == B2D_EPI_GELU || p.epi == B2D_EPI_SILU) && p.out2 != nullptr;
    const bool out2_gate = PP && p.epi == B2D_EPI_GATE_RES && p.gate2_table != nullptr;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int rank = PAIR ? (int)cluster_ctarank() : 0;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.tmA);
        tma_prefetch_desc(&p.tmB);
        if (p.K2 > 0) {
            tma_prefetch_desc(&p.tmA2);
            tma_prefetch_desc(&p.tmB2);
        }
        for (int i = 0; i < Cfg::STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            // every math thread of both CTAs that reads the stage (ping-pong: only the owning warpgroups)
            mbar_init(&empty_bar[i], MC_A ? 256 : PAIR ? 512 : PP ? 128 : 256);
        }
        if (smem_out) tma_prefetch_desc(&p.tmC);
        if (out2_pre || out2_gate) tma_prefetch_desc(&p.tmC2);
        if (stage_x) {
            tma_prefetch_desc(&p.tmX);
            mbar_init(&x_bar[0], 1);
            mbar_init(&x_bar[1], 1);
        }
        fence_mbar_init();
    }
    __syncthreads();
    if (PAIR) cluster_sync_all();  // both CTAs' barriers exist before any multicast or remote arrive
    griddep_wait();  // everything above touched only shared memory and kernel parameters

    const int kb_per_split = (p.kb_main + p.splits - 1) / p.splits;
    // work items: cooperative PAIR -> (pair of M tiles, n tile, batch) per cluster; ping-pong PAIR -> (m tile, pair of
    // N tiles, batch) per cluster; else (m tile, n tile, split, batch) per CTA
    const int m_pairs = (p.m_tiles + 1) / 2;
    const int n_pairs = (p.n_tiles + 1) / 2;
    const int n_items = MC_A ? p.m_tiles * n_pairs * p.batch : PAIR ? m_pairs * p.n_tiles * p.batch : p.total_work;
    const int first = PAIR ? (int)blockIdx.x / 2 : (int)blockIdx.x;
    const int stride = PAIR ? (int)gridDim.x / 2 : (int)gridDim.x;
    auto decode = [&](int w, int& mt, int& nt, int& sp, int& z) {
        if (MC_A) {
            mt = w % p.m_tiles;
            const int t = w / p.m_tiles;
            nt = 2 * (t % n_pairs) + rank;
            z = t / n_pairs;
            sp = 0;
        } else if (PAIR) {
            mt = 2 * (w % m_pairs) + rank;
            const int t = w / m_pairs;
            nt = t % p.n_tiles;
            z = t / p.n_tiles;
            sp = 0;
        } else {
            mt = w % p.m_tiles;
            int t = w / p.m_tiles;
            nt = t % p.n_tiles;
            t /= p.n_tiles;
            sp = t % p.splits;
            z = t / p.splits;
        }
    };
    // k-blocks of split sp: n_main of the main operands from kb_begin on, then (split 0 only) the extension's
    auto kblocks = [&](int sp, int& kb_begin, int& n_main) {
        kb_begin = sp * kb_per_split;
        n_main = min(p.kb_main, kb_begin + kb_per_split) - kb_begin;
        return n_main + ((sp == 0) ? p.kb_ext : 0);
    };

    if (warp < 4) {
        // ============================== TMA producer ==============================
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            // B: the whole tile (single CTA, ping-pong pair), or this CTA's half multicast to both CTAs of a cooperative
            // pair (K-major: BN/2 rows at a 1024-byte aligned offset, so the two halves form the same swizzled tile as
            // one BN-row box; MN-major: every other 64-column box)
            auto load_b = [&](const CUtensorMap* m, uint8_t* sB, uint64_t* bar, int n0, int kcoord, int ncoord_off) {
                if (B_MN == 0) {
                    if (MC_B)
                        tma_load_2d_mc(sB + rank * (BN / 2) * 128, m, bar, kcoord, n0 + rank * (BN / 2) + ncoord_off, 0x3);
                    else
                        tma_load_2d(sB, m, bar, kcoord, n0 + ncoord_off);
                } else {
#pragma unroll
                    for (int j = 0; j < (BN + 63) / 64; ++j) {
                        if (MC_B) {
                            if ((j & 1) == rank) tma_load_2d_mc(sB + j * 8192, m, bar, n0 + 64 * j + ncoord_off, kcoord, 0x3);
                        } else {
                            tma_load_2d(sB + j * 8192, m, bar, n0 + 64 * j + ncoord_off, kcoord);
                        }
                    }
                }
            };
            B2D_TRACE_ONLY(int t = 0;)
            for (int w = first; w < n_items; w += stride) {
                int mt, nt, sp, z;
                decode(w, mt, nt, sp, z);
                const int m0 = mt * BLOCK_M, n0 = nt * BN;
                int kb_begin, n_main;
                const int nkb = kblocks(sp, kb_begin, n_main);
                B2D_TRACE_ONLY(unsigned long long* trec = t < g_gemm_trace.max_tiles - 1 ? trace_rec(t, 2) : nullptr;
                               ++t; unsigned long long waited = 0;)
                for (int i = 0; i < nkb; ++i) {
                    B2D_TRACE_ONLY(const unsigned long long t0 = gtimer();)
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    B2D_TRACE_ONLY(if (trec != nullptr) {
                        const unsigned long long t1 = gtimer();
                        waited += t1 - t0;
                        if (i == 0) trec[TR_TURN] = t1;
                        if (i == nkb - 1) {
                            trec[TR_END] = t1;
                            trec[TR_TURN_WAIT] = waited;
                            trec[TR_SM] = sm_id();
                            trec[TR_MT] = mt;
                            trec[TR_NT] = nt;
                            trec[TR_KIND] = 1;
                        }
                    })
                    uint8_t* sA = smem + stage * Cfg::STAGE_BYTES;
                    uint8_t* sB = sA + A_STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);  // A + the whole B tile, in either mode
                    if (i < n_main) {
                        const int k0 = (kb_begin + i) * BLOCK_K;
                        if (MC_A) {  // this CTA's 64 rows of A (8 KB, 1024-byte aligned), into both CTAs of the pair
                            tma_load_2d_mc(sA + rank * 8192, &p.tmA, &full_bar[stage], k0 + z * p.a_bcol,
                                           m0 + rank * 64 + z * p.a_brow, 0x3);
                        } else if (A_MN == 0) {
                            tma_load_2d(sA, &p.tmA, &full_bar[stage], k0 + z * p.a_bcol, m0 + z * p.a_brow);
                        } else {
#pragma unroll
                            for (int j = 0; j < BLOCK_M / 64; ++j)
                                tma_load_2d(sA + j * 8192, &p.tmA, &full_bar[stage], m0 + 64 * j + z * p.a_bcol,
                                            k0 + z * p.a_brow);
                        }
                        if (B_MN == 0)
                            load_b(&p.tmB, sB, &full_bar[stage], n0, k0 + z * p.b_bcol, z * p.b_brow);
                        else
                            load_b(&p.tmB, sB, &full_bar[stage], n0, k0 + z * p.b_brow, z * p.b_bcol);
                    } else {
                        const int k2 = (i - n_main) * BLOCK_K;
                        // a ping-pong pair's two N tiles lie in one A2 group: take it from the pair's first tile, which
                        // exists even when the second lies past N
                        const int a2off = p.a2_group_n > 0 ? ((n0 - (MC_A ? rank * BN : 0)) / p.a2_group_n) * p.K2 : 0;
                        // A2 is always K-major [M, *]; B2 follows B's majorness
                        if (MC_A)
                            tma_load_2d_mc(sA + rank * 8192, &p.tmA2, &full_bar[stage], k2 + a2off,
                                           m0 + rank * 64 + z * p.a2_brow, 0x3);
                        else
                            tma_load_2d(sA, &p.tmA2, &full_bar[stage], k2 + a2off, m0 + z * p.a2_brow);
                        if (B_MN == 0)
                            load_b(&p.tmB2, sB, &full_bar[stage], n0, k2, z * p.b2_brow);
                        else
                            load_b(&p.tmB2, sB, &full_bar[stage], n0, k2 + z * p.b2_brow, 0);
                    }
                    if (++stage == Cfg::STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else {
        // ============================== math warpgroups ==============================
        setmaxnreg_inc<232>();
        const int cw = (warp >> 2) - 1;  // ping-pong: which tiles of the work list; cooperative: which 64-row half
        const int wq = warp & 3;
        float acc[HALVES][BN / 2];
        int stage = 0;
        uint32_t phase = 0;
        auto release = [&](int s) {
            mbar_arrive(&empty_bar[s]);
            if (PAIR) mbar_arrive_cluster(&empty_bar[s], rank ^ 1);
        };
        // Ping-pong turns: warpgroup 0 issues the main loop of the CTA's tiles 0, 2, 4, ..., warpgroup 1 of tiles 1, 3,
        // ...; a warpgroup starts its main loop once the other has issued all of its previous tile's MMAs (named barrier
        // 1 + cw), and signals the other when it has issued its own.  Warpgroup 1's initial arrive stands in for a
        // tile -1, and the CTA's last tile signals nobody, so no arrival is left pending at exit.
        if (PP && cw == 1) named_bar_arrive(1, 256);
        uint8_t* x_tile = x_tiles + cw * Cfg::X_TILE_BYTES;
        uint8_t* g_tile = g_tiles + cw * Cfg::G_TILE_BYTES;  // [table | temb] slices, BN bf16 each
        uint32_t x_phase = 0;
        int t = 0;  // position of w in the CTA's work list
        for (int w = first; w < n_items; w += stride, ++t) {
            int mt, nt, sp, z;
            decode(w, mt, nt, sp, z);
            int kb_begin, n_main;
            const int nkb = kblocks(sp, kb_begin, n_main);
            if (PP && (t & 1) != cw) {  // the other warpgroup's tile: its k-blocks pass through the ring in between
                stage += nkb;
                phase ^= (stage / Cfg::STAGES) & 1;
                stage %= Cfg::STAGES;
                continue;
            }
            B2D_TRACE_ONLY(unsigned long long* trec = t < g_gemm_trace.max_tiles - 1 ? trace_rec(t, cw) : nullptr;
                           int pass = 0;)
            B2D_TSTAMP(TR_TURN_WAIT);
            if (PP) named_bar_sync(1 + cw, 256);
            B2D_TSTAMP(TR_TURN);
            const bool live = !MC_A || nt < p.n_tiles;  // not the empty second tile of a ping-pong pair
            // The warpgroup's previous epilogue has read its x tile (every thread passed the barrier above): refill it
            // for this tile's epilogue.  The rows of every batch are the same; ragged edges are zero-filled, not read.
            // The gate slices are clamped to the columns below N (a multiple of 8: whole 16-byte chunks).
            if (stage_x && live && threadIdx.x % 128 == 0) {
                const uint32_t g_bytes = stage_gate ? (uint32_t)min(BN, p.N - nt * BN) * 2 : 0u;
                fence_proxy_async_smem();
                mbar_expect_tx(&x_bar[cw], Cfg::X_TILE_BYTES + 2 * g_bytes);
#pragma unroll
                for (int j = 0; j < BN / 64; ++j)
                    tma_load_2d(x_tile + j * (BLOCK_M * 128), &p.tmX, &x_bar[cw], nt * BN + 64 * j, mt * BLOCK_M);
                if (stage_gate) {
                    const bool g1 = p.gate_table != nullptr;
                    const long long smp = (long long)(mt * BLOCK_M / p.rows_per_sample);
                    bulk_load_1d(g_tile, (g1 ? p.gate_table : p.gate2_table) + nt * BN, g_bytes, &x_bar[cw]);
                    bulk_load_1d(g_tile + BN * 2, (g1 ? p.gate_temb : p.gate2_temb) + smp * p.temb_stride + nt * BN,
                                 g_bytes, &x_bar[cw]);
                }
            }
            int prev = -1;
            for (int i = 0; i < nkb; ++i) {
                mbar_wait(&full_bar[stage], phase);
                // the warpgroup's rows of A: the whole tile (ping-pong) or its 64-row half
                const uint32_t sA = smem_u32(smem + stage * Cfg::STAGE_BYTES) + (PP ? 0 : cw * 8192);
                const uint32_t sB = smem_u32(smem + stage * Cfg::STAGE_BYTES) + A_STAGE_BYTES;
                const uint32_t blo = (B_MN != 0) ? sdesc_lo_mnmajor(sB) : sdesc_lo_kmajor(sB);
                constexpr uint32_t bstep = (B_MN != 0) ? SDESC_KSTEP_MNMAJOR : SDESC_KSTEP_KMAJOR;
                wgmma_fence();
                // An MN-major A has no extension k-blocks (b2d_gemm rejects K2 > 0 with it), so the A layout is fixed
                // for the whole loop: one wgmma variant, no runtime choice between two inside the pipeline.
                if constexpr (A_MN != 0)
                    gemm_kblock<BN, 1, B_MN>(acc, sdesc_lo_mnmajor(sA), blo, SDESC_KSTEP_MNMAJOR, bstep, i == 0);
                else
                    gemm_kblock<BN, 0, B_MN>(acc, sdesc_lo_kmajor(sA), blo, SDESC_KSTEP_KMAJOR, bstep, i == 0);
                wgmma_commit();
                if (prev >= 0) {  // the previous k-block's MMAs are done: hand its stage back to the producer(s)
                    wgmma_wait<1>();
                    release(prev);
                }
                prev = stage;
                if (++stage == Cfg::STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            B2D_TSTAMP(TR_LAST_MMA);
            if (PP && w + stride < n_items) named_bar_arrive(2 - cw, 256);
            wgmma_wait<0>();
#pragma unroll
            for (int h = 0; h < HALVES; ++h) wgmma_fence_regs(acc[h]);
            release(prev);
            B2D_TSTAMP(TR_DRAINED);
            B2D_TRACE_ONLY(if (trec != nullptr && threadIdx.x % 128 == 0) {
                trec[TR_SM] = sm_id();
                trec[TR_MT] = mt;
                trec[TR_NT] = nt;
                trec[TR_KIND] = 1;
            })
            if (!live) continue;
            if (stage_x) {
                mbar_wait(&x_bar[cw], x_phase);
                x_phase ^= 1;
            }
            B2D_TSTAMP(TR_X);
            // accumulator d[4j + 2h + e] = (row 16 wq + lane/4 + 8h, column 8j + 2 (lane%4) + e) of each 64-row block
            const int row0 = mt * BLOCK_M + (PP ? 0 : cw * 64) + wq * 16 + (lane >> 2), col0 = nt * BN + 2 * (lane & 3);
            const uint32_t xs = smem_u32(x_tile), gs = smem_u32(g_tile);
            // Every thread's shared-memory writes, then the warpgroup's, before the TMA reads the tile (and with
            // wait_read, the TMA's read of it before the next pass rewrites it).
            auto store_tile = [&](const CUtensorMap* m, bool wait_read) {
                fence_proxy_async_smem();
                named_bar_sync(3 + cw, 128);
                B2D_TSTAMP(pass ? TR_PASS2 : TR_PASS1);
                if (threadIdx.x % 128 == 0) {
#pragma unroll
                    for (int j = 0; j < BN / 64; ++j)
                        tma_store_3d(m, x_tile + j * (BLOCK_M * 128), nt * BN + 64 * j, mt * BLOCK_M, z);
                    tma_store_commit();
                    B2D_TSTAMP(pass ? TR_ST2_ISSUE : TR_ST1_ISSUE);
                    tma_store_wait_read<0>();
                    B2D_TSTAMP(pass ? TR_ST2_READ : TR_ST1_READ);
                }
                B2D_TRACE_ONLY(++pass;)
                if (wait_read) named_bar_sync(3 + cw, 128);
            };
            if constexpr (PP) {
                if (out2_pre) {
                    if (p.epi == B2D_EPI_GELU)
                        gemm_epilogue_tile<B2D_EPI_GELU, BN, HALVES, OUT2_PRE>(p, acc, row0, col0, z, xs, gs, mt * BLOCK_M, nt * BN);
                    else
                        gemm_epilogue_tile<B2D_EPI_SILU, BN, HALVES, OUT2_PRE>(p, acc, row0, col0, z, xs, gs, mt * BLOCK_M, nt * BN);
                    store_tile(&p.tmC2, true);
                }
            }
            gemm_epilogue<BN, HALVES>(p, acc, row0, col0, z, xs, gs, mt * BLOCK_M, nt * BN);
            if (smem_out) {
                // the buffer is refilled (x load) or rewritten only after the warpgroup's next turn barrier, which the
                // storing thread reaches once the store has read it
                store_tile(&p.tmC, out2_gate);
                if constexpr (PP) {
                    if (out2_gate) {
                        gemm_gate2_pass<BN>(p, row0, col0, xs, gs, mt * BLOCK_M, nt * BN);
                        store_tile(&p.tmC2, false);
                    }
                }
            }
            B2D_TSTAMP(TR_END);
        }
        if (smem_out && threadIdx.x % 128 == 0) tma_store_wait_all<0>();  // the last tile is in global memory
        B2D_TRACE_ONLY(if (threadIdx.x % 128 == 0) {
            if (unsigned long long* trec = trace_rec(g_gemm_trace.max_tiles - 1, cw)) {
                trec[TR_END] = gtimer();
                trec[TR_SM] = sm_id();
                trec[TR_KIND] = 2;
            }
        })
    }
    // a CTA of a pair exits only after its peer can no longer multicast into its shared memory or arrive on its barriers
    if (PAIR) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// grid = CTAs; PAIR launches grid / 2 clusters of two CTAs, at most as many as can be resident at once (a GPC with an
// odd number of free SMs leaves one of them out of every cluster)
template <int BN, int A_MN, int B_MN, bool PAIR = false, bool PP = false>
static int launch_gemm(const GemmKParams& kp, int grid, cudaStream_t stream) {
    using Cfg = GemmCfg<BN, B_MN, PP>;
    static bool attr_set[64] = {};
    static int max_clusters[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    auto kern = gemm_kernel<BN, A_MN, B_MN, PAIR, PP>;
    if (dev < 64 && !attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return set_error(B2D_ERR_CUDA, "cudaFuncSetAttribute(gemm): %s", cudaGetErrorString(e));
        if (PAIR) {
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3(2);
            cfg.blockDim = dim3(GEMM_THREADS);
            cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
            cudaLaunchAttribute at;
            at.id = cudaLaunchAttributeClusterDimension;
            at.val.clusterDim.x = 2;
            at.val.clusterDim.y = 1;
            at.val.clusterDim.z = 1;
            cfg.attrs = &at;
            cfg.numAttrs = 1;
            e = cudaOccupancyMaxActiveClusters(&max_clusters[dev], kern, &cfg);
            if (e != cudaSuccess || max_clusters[dev] <= 0)
                return set_error(B2D_ERR_CUDA, "cudaOccupancyMaxActiveClusters(gemm): %s", cudaGetErrorString(e));
        }
        attr_set[dev] = true;
    }
    if (PAIR && dev < 64 && grid > 2 * max_clusters[dev]) grid = 2 * max_clusters[dev];
    launch_kc(kern, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, PAIR ? 2 : 1, kp);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(B2D_ERR_CUDA, "gemm launch: %s", cudaGetErrorString(e));
    count_launch();
    return B2D_OK;
}

template <int BN, bool PP = false>
static int dispatch_major(const GemmKParams& kp, int a_mn, int b_mn, int grid, cudaStream_t s) {
    if constexpr (BN % 64 != 0) {  // 160: K-major A only
        if (b_mn) return launch_gemm<BN, 0, 1, false, PP>(kp, grid, s);
        return launch_gemm<BN, 0, 0, false, PP>(kp, grid, s);
    }
    if (!a_mn && !b_mn) return launch_gemm<BN, 0, 0, false, PP>(kp, grid, s);
    if (!a_mn && b_mn) return launch_gemm<BN, 0, 1, false, PP>(kp, grid, s);
    if (a_mn && b_mn) return launch_gemm<BN, 1, 1, false, PP>(kp, grid, s);
    return launch_gemm<BN, 1, 0, false, PP>(kp, grid, s);
}

// Tile choice: minimise (waves x per-wave tile time) over tile widths, one wave of 128 x bn tiles costing ~ (bn - 48)
// units: the fit of the kernel with the per-pair epilogue, whose per-wave time grew with its code size.  A sweep of
// bn in {64, 128, 192, 256} x {single CTA, CTA pair} on the ping-pong kernel (tools/gemm_bench.py, H100 80GB HBM3 at
// 400 W, the twelve step GEMMs at M = 2688) keeps 128: the ping-pong 128 tile is 2-16 % faster than 192 on the
// plain-store, GELU and GELU' launches (192 wins only QKV dX, by 7 %), 256 loses everywhere, 64 loses 24-40 % on its
// doubled A traffic; 192 was 13-42 % slower on the gate/residual launches.  Those launches now ping-pong too.  A
// re-sweep of bn in {64, 128} on them and FFN up (H100 80GB HBM3 at 700 W, DESIGN 4.2.1) keeps 128 on to_out, cross
// to_out, FFN down and FFN up (15-48 % faster than 64); only cross to_q dX (gate2 copy, two store passes per tile) is
// faster at 64, by 13 %.  The choice here sees the shape, not the epilogue, and the plain-store launches of that shape
// lose at 64, so it stays 128.
// The N = 2048 shapes keep their 2.55-wave tail (336 tiles on 132 SMs): about a third of a wave of idle SMs per
// launch.  64 only when no wider tile fits N.  MN-major A tiles are built from 64-column TMA boxes, so they need
// bn % 64 == 0.  The sweep above ran with CTA pairs whose remote empty-barrier arrivals fenced at cluster scope, which
// halved their main-loop rate; with that fixed, 128-wide ping-pong tiles run on 2-CTA clusters where they can (b2d_gemm,
// DESIGN 4.2.2), and the wider cooperative pairs have not been re-timed.
static int pick_tile(int M, int N, int nsm, int work_mult, int a_mn, int group_n) {
    const int cands[4] = {256, 192, 160, 128};
    int best = 64;
    double best_t = 1e30;
    const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
    for (int i = 0; i < 4; ++i) {
        const int bn = cands[i];
        if (a_mn && (bn % 64) != 0) continue;
        if (group_n > 0 && (group_n % bn) != 0) continue;
        if (bn > N) continue;
        const int n_tiles = (N + bn - 1) / bn;
        const long long tiles = (long long)m_tiles * n_tiles * work_mult;
        const long long waves = (tiles + nsm - 1) / nsm;
        const double t = (double)waves * (bn - 48);
        if (t < best_t - 1e-9) {
            best_t = t;
            best = bn;
        }
    }
    return best;
}

}  // namespace b2d

using namespace b2d;

#ifdef B2D_GEMM_TRACE
// Timeline buffer of the following gemm_kernel launches on the current device: grid x max_tiles x 3 records of
// GEMM_TRACE_SLOTS u64 (zeroed by the caller), or buf = null to stop tracing.
extern "C" int b2d_gemm_trace_set(void* buf, int max_tiles) {
    const GemmTrace tr = {reinterpret_cast<unsigned long long*>(buf), max_tiles};
    cudaError_t e = cudaMemcpyToSymbol(g_gemm_trace, &tr, sizeof(tr));
    if (e != cudaSuccess) return set_error(B2D_ERR_CUDA, "gemm trace: %s", cudaGetErrorString(e));
    return B2D_OK;
}
#endif

extern "C" int b2d_gemm(const b2d_gemm_desc* d, void* stream_v) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    if (d == nullptr) return set_error(B2D_ERR_ARG, "gemm: null descriptor");
    if (d->A == nullptr || d->B == nullptr || d->out == nullptr) return set_error(B2D_ERR_ARG, "gemm: null operand");
    B2D_BIND(d->A);
    if (d->M <= 0 || d->N <= 0 || d->K <= 0) return set_error(B2D_ERR_SHAPE, "gemm: M,N,K must be positive");
    if (d->N % 8 != 0) return set_error(B2D_ERR_SHAPE, "gemm: N %% 8 != 0 (N=%d)", d->N);
    if (d->K2 % 64 != 0) return set_error(B2D_ERR_SHAPE, "gemm: K2 %% 64 != 0");
    if ((d->lda % 8) || (d->ldb % 8)) return set_error(B2D_ERR_ALIGN, "gemm: lda/ldb must be multiples of 8 elements");
    if (((uintptr_t)d->A & 15) || ((uintptr_t)d->B & 15) || ((uintptr_t)d->out & 15))
        return set_error(B2D_ERR_ALIGN, "gemm: pointers must be 16-byte aligned");
    const int splits = d->splits > 0 ? d->splits : 1;
    const int batch = d->batch > 0 ? d->batch : 1;
    // The tensor maps of a batched launch span every batch (see below), so the k-block that runs past a ragged K reads
    // the next batch's elements instead of TMA zero fill wherever the batch offset moves along K.
    if (batch > 1 && d->K % BLOCK_K != 0 &&
        ((d->a_mn_major ? d->a_boff_row : d->a_boff_col) != 0 || (d->b_mn_major ? d->b_boff_row : d->b_boff_col) != 0))
        return set_error(B2D_ERR_SHAPE, "gemm: a batch offset along K needs K %% 64 == 0 (K=%d)", d->K);
    const bool f32_atomic = d->epi == B2D_EPI_F32_ATOMIC || d->epi == B2D_EPI_F32_ATOMIC_T;
    if (splits > 1 && !f32_atomic) return set_error(B2D_ERR_ARG, "gemm: split-K needs an atomic fp32 epilogue");
    if (splits > 1 && d->K2 > 0) return set_error(B2D_ERR_ARG, "gemm: split-K with extension operands unsupported");
    if (d->epi == B2D_EPI_GATE_RES && d->res == nullptr) return set_error(B2D_ERR_ARG, "gemm: GATE_RES needs res");
    if (d->epi == B2D_EPI_MUL_DGELU && d->aux == nullptr) return set_error(B2D_ERR_ARG, "gemm: MUL_DGELU needs aux");
    if (d->gate_table != nullptr && (d->gate_temb == nullptr || d->rows_per_sample <= 0))
        return set_error(B2D_ERR_ARG, "gemm: gate needs temb + rows_per_sample");
    if (d->gate2_table != nullptr && (d->gate2_temb == nullptr || d->rows_per_sample <= 0 || d->out2 == nullptr))
        return set_error(B2D_ERR_ARG, "gemm: gate2 needs gate2_temb, rows_per_sample and out2");
    if (d->K2 > 0 && d->a_mn_major) return set_error(B2D_ERR_ARG, "gemm: extension operands need K-major A");
    // epilogue operands: 16-byte aligned pointers, and leading dimensions / batch offsets that keep every row 16-byte
    // aligned (in elements of the output type: fp32 for the F32 epilogues, bf16 otherwise)
    {
        const bool f32_out = d->epi == B2D_EPI_F32_ATOMIC || d->epi == B2D_EPI_F32_ATOMIC_T || d->epi == B2D_EPI_F32_STORE;
        const int64_t out_vec = f32_out ? 4 : 8;
        const void* ptrs[] = {d->out2, d->bias, d->res, d->aux, d->gate_table, d->gate_temb, d->gate2_table, d->gate2_temb};
        for (const void* q : ptrs)
            if ((uintptr_t)q & 15) return set_error(B2D_ERR_ALIGN, "gemm: epilogue pointers must be 16-byte aligned");
        if ((d->ldc % out_vec) || (d->c_boff % out_vec) || (d->out2 != nullptr && (d->ldc2 % 8)) ||
            (d->res != nullptr && (d->ldres % 8)) || (d->aux != nullptr && (d->ldaux % 8)) ||
            ((d->gate_table != nullptr || d->gate2_table != nullptr) && (d->temb_stride % 8)))
            return set_error(B2D_ERR_ALIGN, "gemm: ldc, ldc2, ldres, ldaux, temb_stride and c_boff must keep rows 16-byte aligned");
    }

    int nsm = device_sm_count();
    if (nsm <= 0) return B2D_ERR_CUDA;
    int max_ctas = d->max_ctas > 0 ? d->max_ctas : nsm;
    if (d->cta_pair < 0 || d->cta_pair > 2) return set_error(B2D_ERR_ARG, "gemm: cta_pair must be 0 (auto), 1 or 2");
    // CTA pairs need a K-major A operand, no split-K, at least one full pair of M tiles and two SMs
    const bool pair_ok = !d->a_mn_major && splits == 1 && d->M > BLOCK_M && max_ctas >= 2;
    if (d->cta_pair == 2 && !pair_ok)
        return set_error(B2D_ERR_ARG, "gemm: cta_pair = 2 needs K-major A, splits = 1, M > 128 and max_ctas >= 2");
    const int bn = d->block_n > 0 ? d->block_n : pick_tile(d->M, d->N, max_ctas, splits * batch, d->a_mn_major, d->a2_group_n);
    if (bn != 64 && bn != 128 && bn != 160 && bn != 192 && bn != 256) return set_error(B2D_ERR_ARG, "gemm: bad block_n %d", bn);
    if (d->cta_pair == 2 && bn == 64) return set_error(B2D_ERR_ARG, "gemm: CTA pairs need block_n >= 128");
    if ((bn % 64) && d->a_mn_major) return set_error(B2D_ERR_ARG, "gemm: block_n 160 needs a K-major A operand");
    if (d->a2_group_n > 0 && (d->a2_group_n % bn) != 0)
        return set_error(B2D_ERR_ARG, "gemm: a2_group_n (%d) must be a multiple of block_n (%d)", d->a2_group_n, bn);
    const long long m_tiles = (d->M + BLOCK_M - 1) / BLOCK_M, n_tiles = (d->N + bn - 1) / bn;
    const long long total = m_tiles * n_tiles * splits * batch;
    if (total > 0x7fffffffLL) return set_error(B2D_ERR_SHAPE, "gemm: too many tiles");
    const int grid = (int)(total < max_ctas ? total : max_ctas);
    // Ping-pong where a CTA gets more than one tile and both accumulators fit.  With one tile per CTA the second
    // warpgroup would idle, and the cooperative schedule splits the tile between both.  A gate/residual tile brings its
    // gate into shared memory with its residual tile, as one vector over its columns, so that its one-warpgroup
    // epilogue reads no global memory (loading the gates per column group and row from there, the exposed last tile of
    // the N = 2048 shapes made such launches 1.2-1.55x slower than cooperative on an H100).  That needs every tile
    // inside one sample, and room for one gate only: launches whose samples do not start on 128-row tile boundaries,
    // or that have both gate and gate2, stay cooperative.  The step has neither.  Ping-pong bf16 out tiles leave by
    // TMA store, batch z at z * c_boff: a batch stride the TMA can take (16-byte multiples by the alignment rule
    // above) unless it is 0, every batch writing the same window.
    const bool gated = d->epi == B2D_EPI_GATE_RES && (d->gate_table != nullptr || d->gate2_table != nullptr);
    const bool gate_pp = !gated || ((d->gate_table == nullptr || d->gate2_table == nullptr) &&
                                    (d->rows_per_sample % BLOCK_M == 0 || d->rows_per_sample >= d->M));
    const bool pp_able = bn <= 128 && gate_pp && (!gemm_bf16_out(d->epi) || batch == 1 || d->c_boff > 0);
    // Ping-pong on CTA pairs: N-pairs of 128-wide tiles that share (multicast) their A tile, with more pair items than
    // clusters.  Both tiles of a pair must read the same LoRA A2 slice.  N-pairs rather than M-pairs: every N of the
    // step is a multiple of 256, while its M = 2688 is 21 tiles, so M-pairs would leave one CTA of every column's last
    // pair on zero-filled rows (4.5 % of the MMAs) and add pair items on the N = 2048 shapes' last wave.
    const long long n_pair_items = m_tiles * ((n_tiles + 1) / 2) * batch;
    const bool pp_pair_able = pair_ok && pp_able && bn == 128 && n_pair_items > max_ctas / 2 &&
                              (d->a2_group_n == 0 || d->a2_group_n % (2 * bn) == 0);
    // cta_pair 0 takes ping-pong pairs only on launches of the kind they were measured on, the twelve step GEMMs
    // (M = 2688, N in {2048, 6144, 8192}, K in {2048, 6144, 8192}): one batch, an even number of N tiles (no CTA runs
    // a zero-filled tile) and more tiles than CTAs (single-CTA ping-pong's own condition).  There, on an H100 80GB HBM3
    // at 700 W (DESIGN 4.2.2, two rounds against the single-CTA build, median SM clock 1965 MHz, its 1890 / 1980 MHz),
    // the per-block sum of the twelve EPI_STORE launches fell from 1169 / 1160 to 1038 / 1038 us and of the fused
    // launches from 1258 / 1266 to 1204 / 1191 us; QKV, FFN up, FFN up dX and FFN down dX by 6-14 % under EPI_STORE,
    // the other eight by 2-9 %.  Batched launches (the block-batched LoRA and kv2
    // projections), launches with an odd N-tile count and launches with at most one tile per CTA keep their single-CTA
    // schedule: pairs were not measured on them, and an odd or single N tile leaves half of a cluster multiplying
    // zeros.  cta_pair 2: pairs, ping-pong where they can run and cooperative M-pairs elsewhere.
    const bool pair_auto = pp_pair_able && batch == 1 && n_tiles % 2 == 0 && total > grid;
    const bool pair = d->cta_pair == 2 || (d->cta_pair == 0 && pair_auto);
    const bool pp = pair ? pp_pair_able : pp_able && total > grid;
    const int a_box_rows = pair && pp ? 64 : d->a_mn_major ? 64 : BLOCK_M;  // A (and A2): rows of the box one CTA loads
    const int b_box_rows = pair && !pp ? bn / 2 : bn;                        // K-major B (and B2): the same

    GemmKParams kp;
    memset(&kp, 0, sizeof(kp));
    // ---- tensor maps. K-major operand [rows, K]: box {64, rows_tile}.  MN-major operand [K, cols]: box {64, 64}.
    int rc;
    // total extents seen by TMA: include batch offsets so every batch's window is in-bounds
    {
        long long rowsA = d->a_mn_major ? (long long)d->K + (batch - 1) * d->a_boff_row : (long long)d->M + (batch - 1) * d->a_boff_row;
        long long colsA = d->a_mn_major ? (long long)d->M + (batch - 1) * d->a_boff_col : (long long)d->K + (batch - 1) * d->a_boff_col;
        rc = make_tmap_2d(&kp.tmA, d->A, rowsA, colsA, d->lda, a_box_rows, 64);
        if (rc) return rc;
        long long rowsB = d->b_mn_major ? (long long)d->K + (batch - 1) * d->b_boff_row : (long long)d->N + (batch - 1) * d->b_boff_row;
        long long colsB = d->b_mn_major ? (long long)d->N + (batch - 1) * d->b_boff_col : (long long)d->K + (batch - 1) * d->b_boff_col;
        rc = make_tmap_2d(&kp.tmB, d->B, rowsB, colsB, d->ldb, d->b_mn_major ? 64 : b_box_rows, 64);
        if (rc) return rc;
        if (d->K2 > 0) {
            if (d->A2 == nullptr || d->B2 == nullptr) return set_error(B2D_ERR_ARG, "gemm: K2>0 needs A2,B2");
            int groups = d->a2_group_n > 0 ? (d->N + d->a2_group_n - 1) / d->a2_group_n : 1;
            rc = make_tmap_2d(&kp.tmA2, d->A2, (long long)d->M + (batch - 1) * d->a2_boff_row, (long long)d->K2 * groups,
                              d->lda2, a_box_rows, 64);
            if (rc) return rc;
            if (d->b_mn_major)
                rc = make_tmap_2d(&kp.tmB2, d->B2, (long long)d->K2 + (batch - 1) * d->b2_boff_row, d->N, d->ldb2, 64, 64);
            else
                rc = make_tmap_2d(&kp.tmB2, d->B2, (long long)d->N + (batch - 1) * d->b2_boff_row, d->K2, d->ldb2, b_box_rows, 64);
            if (rc) return rc;
        }
    }
    kp.M = d->M; kp.N = d->N; kp.K = d->K; kp.K2 = d->K2;
    kp.a2_group_n = d->a2_group_n;
    kp.splits = splits; kp.batch = batch;
    kp.a_brow = (int)d->a_boff_row; kp.a_bcol = (int)d->a_boff_col;
    kp.b_brow = (int)d->b_boff_row; kp.b_bcol = (int)d->b_boff_col;
    kp.c_boff = d->c_boff;
    kp.a2_brow = (int)d->a2_boff_row; kp.b2_brow = (int)d->b2_boff_row;
    kp.bias_boff = d->bias_boff;
    if (d->a2_boff_row < 0 || d->b2_boff_row < 0 || d->bias_boff < 0 || (d->bias_boff % 8) != 0)
        return set_error(B2D_ERR_ARG, "gemm: extension/bias batch offsets must be >= 0 (bias_boff a multiple of 8)");
    kp.epi = d->epi;
    kp.alpha = d->alpha;
    kp.out = d->out; kp.ldc = d->ldc;
    kp.out2 = d->out2; kp.ldc2 = d->ldc2;
    kp.bias = (const __nv_bfloat16*)d->bias;
    kp.res = (const __nv_bfloat16*)d->res; kp.ldres = d->ldres;
    kp.aux = (const __nv_bfloat16*)d->aux; kp.ldaux = d->ldaux;
    kp.gate_table = (const __nv_bfloat16*)d->gate_table;
    kp.gate_temb = (const __nv_bfloat16*)d->gate_temb;
    kp.gate2_table = (const __nv_bfloat16*)d->gate2_table;
    kp.gate2_temb = (const __nv_bfloat16*)d->gate2_temb;
    kp.temb_stride = d->temb_stride;
    kp.rows_per_sample = d->rows_per_sample;
    kp.m_tiles = (d->M + BLOCK_M - 1) / BLOCK_M;
    kp.n_tiles = (d->N + bn - 1) / bn;
    kp.kb_main = (d->K + BLOCK_K - 1) / BLOCK_K;
    kp.kb_ext = d->K2 / BLOCK_K;
    if (splits > kp.kb_main) return set_error(B2D_ERR_ARG, "gemm: splits > k-blocks");
    // every split must own at least one k-block
    {
        int per = (kp.kb_main + splits - 1) / splits;
        if ((splits - 1) * per >= kp.kb_main) return set_error(B2D_ERR_ARG, "gemm: empty split (K=%d splits=%d)", d->K, splits);
    }
    kp.total_work = (int)total;
    if (pp && (d->epi == B2D_EPI_GATE_RES || d->epi == B2D_EPI_MUL_DGELU)) {  // ping-pong x tiles
        const bool res = d->epi == B2D_EPI_GATE_RES;
        rc = make_tmap_2d(&kp.tmX, res ? d->res : d->aux, d->M, d->N, res ? d->ldres : d->ldaux, BLOCK_M, 64);
        if (rc) return rc;
    }
    // ping-pong out (and out2) tiles
    const bool out2_tiles = d->out2 != nullptr && (d->epi == B2D_EPI_GELU || d->epi == B2D_EPI_SILU ||
                                                   (d->epi == B2D_EPI_GATE_RES && d->gate2_table != nullptr));
    for (int o = 0; o < (out2_tiles ? 2 : 1) && pp && gemm_bf16_out(d->epi); ++o) {
        const long long ld = o ? d->ldc2 : d->ldc;
        const uint64_t dims[3] = {(uint64_t)d->N, (uint64_t)d->M, (uint64_t)batch};
        const uint64_t strides[2] = {(uint64_t)ld * 2, (uint64_t)(batch > 1 ? d->c_boff : d->M * ld) * 2};
        const uint32_t box[3] = {64, BLOCK_M, 1};
        rc = make_tmap_nd(o ? &kp.tmC2 : &kp.tmC, o ? d->out2 : d->out, 3, dims, strides, box, 2, 1);
        if (rc) return rc;
    }
    if (pair) {
        const long long pairs = pp ? n_pair_items : ((m_tiles + 1) / 2) * n_tiles * batch;
        const int clusters = (int)(pairs < max_ctas / 2 ? pairs : max_ctas / 2);
        if (pp)
            return d->b_mn_major ? launch_gemm<128, 0, 1, true, true>(kp, 2 * clusters, stream)
                                 : launch_gemm<128, 0, 0, true, true>(kp, 2 * clusters, stream);
        switch (bn) {
            case 128: return d->b_mn_major ? launch_gemm<128, 0, 1, true>(kp, 2 * clusters, stream) : launch_gemm<128, 0, 0, true>(kp, 2 * clusters, stream);
            case 160: return d->b_mn_major ? launch_gemm<160, 0, 1, true>(kp, 2 * clusters, stream) : launch_gemm<160, 0, 0, true>(kp, 2 * clusters, stream);
            case 192: return d->b_mn_major ? launch_gemm<192, 0, 1, true>(kp, 2 * clusters, stream) : launch_gemm<192, 0, 0, true>(kp, 2 * clusters, stream);
            default: return d->b_mn_major ? launch_gemm<256, 0, 1, true>(kp, 2 * clusters, stream) : launch_gemm<256, 0, 0, true>(kp, 2 * clusters, stream);
        }
    }
    switch (bn) {
        case 64: return pp ? dispatch_major<64, true>(kp, d->a_mn_major, d->b_mn_major, grid, stream)
                           : dispatch_major<64>(kp, d->a_mn_major, d->b_mn_major, grid, stream);
        case 128: return pp ? dispatch_major<128, true>(kp, d->a_mn_major, d->b_mn_major, grid, stream)
                            : dispatch_major<128>(kp, d->a_mn_major, d->b_mn_major, grid, stream);
        case 160: return dispatch_major<160>(kp, d->a_mn_major, d->b_mn_major, grid, stream);
        case 192: return dispatch_major<192>(kp, d->a_mn_major, d->b_mn_major, grid, stream);
        default: return dispatch_major<256>(kp, d->a_mn_major, d->b_mn_major, grid, stream);
    }
}
