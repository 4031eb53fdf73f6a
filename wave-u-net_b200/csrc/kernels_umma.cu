// kernels_umma.cu - tensor-core plane convolution and weight gradient for sm_90a (Hopper wgmma).
//
// One kernel serves the forward conv blocks and their dgrads (both are "plane convolutions", launch.h):
//     out_cls[b, m, n] = epi( sum_terms  plane[b, m + d, :] . W_term[:, n] )
// mapped onto wgmma as a shifted-tap implicit GEMM:
//   * A operand: the CTA stages a SLAB of input rows once per 16-channel chunk in shared memory, as bf16
//     "channel-atom planes"  [hi a0|hi a1|lo a0|lo a1][row][16 B]  (K-major, no-swizzle canonical layout: 8 rows x 16 B
//     core matrices, SBO = 128 B between 8-row groups, LBO = atom-plane stride between the two K atoms of one k16 MMA).
//     A conv tap is then just a descriptor START-ADDRESS shift of d*16 B - the slab is read by every tap without being
//     re-loaded or re-converted.  Decimation ([:, ::2, :], UnetAudioSeparator.py:100), the skip crop (:122), zero padding
//     and the linear / learned upsampling (:109-118, InterpolationLayer.py:19-39) all happen in the fp32 -> bf16
//     conversion that fills the slab, so none of those tensors ever exists in HBM.
//   * fp32-level accuracy: every fp32 operand x is split x = hi + lo (two bf16), and each K step issues three MMAs
//     lo*hi + hi*lo + hi*hi into the same fp32 accumulator (error ~2^-17 per operand; single-pass bf16 / tf32 miss the
//     1e-4 parity bar - BASELINE.md section 6).
//   * B operand (weights): pre-packed once per optimizer step into the exact K-step streaming order, hi/lo bf16, core-matrix
//     layout (umma_pack_kernel); streamed with cp.async.bulk through an mbarrier ring.
//   * a CTA is two warpgroups over a 128-row tile; each holds 64 rows x NPAD fp32 accumulators in registers.  The MMAs of a
//     step are asynchronous (wgmma.mma_async): while they run, the same threads convert the next slab.  Epilogue: registers
//     -> bias / LeakyReLU (fwd) -> a shared-memory staging tile -> coalesced global stores, with the LeakyReLU-slope /
//     accumulate read-back of the dgrad.
// Kernels in this file:
//   plane_conv_umma_kernel<NPAD, DG>          the conv (forward: DG = false, dgrad: DG = true)
//   split_views_kernel, wgrad_umma_bulk_kernel<NT>   hi/lo split arrays of a layer's wgrad operands (+ bias column sums) and
//                                            the bulk-copy-fed wgrad;  wgrad_umma_kernel<NT>: the converter-fed form, for layers
//                                            whose operand views do not fit one split pass
//   umma_pack_kernel                         fp32 weights -> hi/lo bf16 blocks in K-step streaming order (pair-merged classes: two
//                                            taps side by side per row shift)
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "kernels_umma.h"

namespace wun {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must become a trap (reported error), never a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) asm volatile("trap;");
    }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// mbar_arrive_expect_tx + bulk_g2s of `bytes`, issued by the thread with tid == 0 only.  The predicate lives inside the asm, so
// the code has no branch on the thread index: between MMAs still in flight and the next ones, such a branch makes ptxas
// serialise the MMAs (C7520).
__device__ __forceinline__ void bulk_g2s_thread0(uint32_t tid, uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.eq.u32 p, %0, 0;\n\t"
                 "@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%1], %2;\n\t"
                 "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%3], [%4], %2, [%1];\n\t}"
                 ::"r"(tid), "r"(bar), "r"(bytes), "r"(dst), "l"(src)
                 : "memory");
}

// No-swizzle shared-memory matrix descriptor of wgmma: start address, leading / stride byte offsets (all >> 4).
//   K-major operand:  LBO = bytes between the two 8-element K groups of a k16 step, SBO = bytes between 8-row M/N groups.
//   MN-major operand: LBO = bytes between 8-row K groups, SBO = bytes between 8-element M/N groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// waits until at most N committed MMA groups of this warpgroup are still running
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// After wgmma_wait<0>(): the accumulator registers are only now final.  The empty asm "redefines" each of them, so that
// no read of an accumulator is scheduled above the wait.
template <int N>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// One m64nNk16 MMA for every N the kernels use (16..128 in steps of 16), from one asm template: the N/2 accumulators are
// read-write operands %0 .. %(N/2 - 1) (WUN_ACC<N> lists them, WUN_D<N> binds them) and the two descriptors are the input
// operands that follow (WUN_DESC<N>).
#define WUN_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define WUN_ACC16 "%0, %1, %2, %3, %4, %5, %6, %7"
#define WUN_ACC32 WUN_ACC16 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define WUN_ACC48 WUN_ACC32 ", %16, %17, %18, %19, %20, %21, %22, %23"
#define WUN_ACC64 WUN_ACC48 ", %24, %25, %26, %27, %28, %29, %30, %31"
#define WUN_ACC80 WUN_ACC64 ", %32, %33, %34, %35, %36, %37, %38, %39"
#define WUN_ACC96 WUN_ACC80 ", %40, %41, %42, %43, %44, %45, %46, %47"
#define WUN_ACC112 WUN_ACC96 ", %48, %49, %50, %51, %52, %53, %54, %55"
#define WUN_ACC128 WUN_ACC112 ", %56, %57, %58, %59, %60, %61, %62, %63"
#define WUN_D16 WUN_F8(0)
#define WUN_D32 WUN_D16, WUN_F8(8)
#define WUN_D48 WUN_D32, WUN_F8(16)
#define WUN_D64 WUN_D48, WUN_F8(24)
#define WUN_D80 WUN_D64, WUN_F8(32)
#define WUN_D96 WUN_D80, WUN_F8(40)
#define WUN_D112 WUN_D96, WUN_F8(48)
#define WUN_D128 WUN_D112, WUN_F8(56)
#define WUN_DESC16 "%8, %9"
#define WUN_DESC32 "%16, %17"
#define WUN_DESC48 "%24, %25"
#define WUN_DESC64 "%32, %33"
#define WUN_DESC80 "%40, %41"
#define WUN_DESC96 "%48, %49"
#define WUN_DESC112 "%56, %57"
#define WUN_DESC128 "%64, %65"
#define WUN_WGMMA(N, T)                                                                                                     \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"                                                           \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 {" WUN_ACC##N "}, " WUN_DESC##N ", p, 1, 1, " T ", " T ";\n\t}" \
                 : WUN_D##N                                                                                             \
                 : "l"(da), "l"(db))
#define WUN_WGMMA_ANY_N(T)                                                                                                  \
    if constexpr (N == 16) WUN_WGMMA(16, T);                                                                                \
    else if constexpr (N == 32) WUN_WGMMA(32, T);                                                                           \
    else if constexpr (N == 48) WUN_WGMMA(48, T);                                                                           \
    else if constexpr (N == 64) WUN_WGMMA(64, T);                                                                           \
    else if constexpr (N == 80) WUN_WGMMA(80, T);                                                                           \
    else if constexpr (N == 96) WUN_WGMMA(96, T);                                                                           \
    else if constexpr (N == 112) WUN_WGMMA(112, T);                                                                         \
    else WUN_WGMMA(128, T);

// D[64 x N] += A[64 x 16] * B[16 x N], bf16 -> fp32, as ONE wgmma (A is read from shared memory once per k16 step).  MN = 1:
// both operands are MN-major, else both K-major.  Accumulator register i of a thread holds column (i/4)*8 + (lane%4)*2 + i%2 and
// row 16*(warp%4) + lane/4 + 8*((i/2)%2) of the warpgroup's 64 x N tile.
template <int N, int MN>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t da, uint64_t db) {
    static_assert(N % 16 == 0 && N >= 16 && N <= 128, "m64nNk16: N = 16..128 in steps of 16");
    if constexpr (MN) { WUN_WGMMA_ANY_N("1") }
    else { WUN_WGMMA_ANY_N("0") }
}
#undef WUN_WGMMA_ANY_N
#undef WUN_WGMMA
#undef WUN_F8
__device__ __forceinline__ int acc_col(int i, int lane) { return (i >> 2) * 8 + (lane & 3) * 2 + (i & 1); }
__device__ __forceinline__ int acc_row(int i, int warp, int lane) { return 16 * (warp & 3) + (lane >> 2) + 8 * ((i >> 1) & 1); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo_elem, float hi_elem) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo_elem, hi_elem);   // .x = first (low address)
    return *reinterpret_cast<uint32_t*>(&t);
}
// 16 fp32 values -> 8 words of bf16 hi parts and 8 words of bf16 remainders (x = hi + lo to ~2^-17)
__device__ __forceinline__ void split_hi_lo(const float* x, uint32_t* hi, uint32_t* lo) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const __nv_bfloat16 h0 = __float2bfloat16_rn(x[2 * i]), h1 = __float2bfloat16_rn(x[2 * i + 1]);
        hi[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        lo[i] = pack_bf16x2(x[2 * i] - __bfloat162float(h0), x[2 * i + 1] - __bfloat162float(h1));
    }
}

// ------------------------------------------------------------------------------------------------
// slab fill helpers
// ------------------------------------------------------------------------------------------------
// Interpolated row of a MID plane from row x and its successor nx (channels [c0, c0 + nv)): learned or linear upsampling.
__device__ __forceinline__ void mid_blend(const PlaneView& P, int c0, int nv, float* x, const float* nx) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        if (i < nv) {
            if (P.blend) { const float w = __ldg(P.blend + c0 + i); x[i] = w * x[i] + (1.f - w) * nx[i]; }
            else x[i] = x[i] + (nx[i] - x[i]) * 0.5f;
        }
    }
}

// 16 channels [c0, c0+16) of plane row r of batch b, fp32, zero where invalid.
__device__ __forceinline__ void load_row16(const PlaneView& P, int b, int r, int c0, float* x) {
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] = 0.f;
    if (r < P.r_lo || r >= P.r_hi) return;
    const float* p = P.base + (long long)b * P.bstride + (long long)r * P.rstride + c0;
    const int nv = min(16, P.C - c0);      // multiple of 8 (eligibility)
    if (nv >= 16) {
        const float4* q = reinterpret_cast<const float4*>(p);
#pragma unroll
        for (int i = 0; i < 4; ++i) { float4 t = __ldg(q + i); x[4 * i] = t.x; x[4 * i + 1] = t.y; x[4 * i + 2] = t.z; x[4 * i + 3] = t.w; }
    } else if (nv >= 8) {
        const float4* q = reinterpret_cast<const float4*>(p);
#pragma unroll
        for (int i = 0; i < 2; ++i) { float4 t = __ldg(q + i); x[4 * i] = t.x; x[4 * i + 1] = t.y; x[4 * i + 2] = t.z; x[4 * i + 3] = t.w; }
    }
    if (P.kind == PLANE_MID) {
        float nx[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) nx[i] = 0.f;
        const bool has_next = (P.mid_mode == MID_VALID) || (r + 1 < P.xrows);
        if (has_next) {
            const float4* q = reinterpret_cast<const float4*>(p + P.rstride);
            const int n4 = (nv >= 16) ? 4 : 2;
            for (int i = 0; i < n4; ++i) { float4 t = __ldg(q + i); nx[4 * i] = t.x; nx[4 * i + 1] = t.y; nx[4 * i + 2] = t.z; nx[4 * i + 3] = t.w; }
        } else if (P.mid_mode == MID_CLAMP) {
#pragma unroll
            for (int i = 0; i < 16; ++i) nx[i] = x[i];
        }
        mid_blend(P, c0, nv, x, nx);
    }
}

// A (plane, tile) pair whose slab would hold nothing but zero rows - the tile's rows plus the group's tap span lie
// entirely outside the plane's valid rows - contributes nothing: the K loop skips the group and its packed weights.  This
// is what the dgrad of a down block looks like outside the skip window: the gradient of the odd rows (g_odd) is zero there.
__device__ __forceinline__ bool group_is_empty(const UmmaLaunch& L, const UmmaGroup& G, int m_base) {
    const PlaneView& P = L.planes[G.plane];
    const int lo = m_base + G.dmin;
    return lo + L.rows_alloc <= P.r_lo || lo >= P.r_hi;
}

// ------------------------------------------------------------------------------------------------
// conv epilogue: staged rows -> global memory
// ------------------------------------------------------------------------------------------------
// Per half (pair-merged classes have two, launch.h OutView::pairC) one base pointer that already contains the batch item and
// the block's first column; an item then costs one 32-bit multiply-add.
struct EpiHalf {
    float* dst;            // + m * rstride + 4 * (quad within the half)
    const float* saved;    // same geometry (null: no slope)
    int rstride, lo, hi, acc_lo, acc_hi;
};
struct EpiBlock {
    EpiHalf h[2];
    int qsplit;            // quads [0, qsplit) of the staged block belong to half 0, the rest to half 1
};
template <bool PAIR>
__device__ __forceinline__ EpiBlock epi_block(const OutView& O, int b, int col0, int Q, bool slope) {
    EpiBlock B;
    const bool pair = PAIR && O.pairC > 0;
    const int c1 = pair ? max(col0, O.pairC) : 0;           // first launch column of half 1 inside / after this block
    B.qsplit = pair ? min(Q, max(0, (O.pairC - col0) >> 2)) : Q;
    B.h[0].dst = O.base + (long long)b * O.bstride + col0;
    B.h[0].saved = (slope && O.saved) ? O.saved + (long long)b * O.bstride + col0 : nullptr;
    B.h[0].rstride = O.rstride;
    B.h[0].lo = pair ? O.lo_h[0] : O.m_lo; B.h[0].hi = pair ? O.hi_h[0] : O.m_hi;
    B.h[0].acc_lo = O.acc_lo; B.h[0].acc_hi = O.acc_hi;
    if (pair) {
        // quad q >= qsplit sits at launch column col0 + 4q = half-1 column (col0 + 4q - pairC): fold (c1 - pairC) - 4 * qsplit into the base
        const long long adj = (long long)b * O.bstride2 + (c1 - O.pairC) - 4 * B.qsplit;
        B.h[1].dst = O.base2 + adj;
        B.h[1].saved = (slope && O.saved2) ? O.saved2 + adj : nullptr;
        B.h[1].rstride = O.rstride2;
        B.h[1].lo = O.lo_h[1]; B.h[1].hi = O.hi_h[1];
        B.h[1].acc_lo = O.acc_lo2; B.h[1].acc_hi = O.acc_hi2;
    } else {
        B.h[1] = B.h[0];
    }
    return B;
}

// One warp writes out 32 staged rows (row r0 + 0..31 of the tile), lanes running over (row, 4-column quad) pairs so that narrow
// layers (N = 24..48) still use every lane and a warp store covers several consecutive rows.  Forward form: nothing to read back.
__device__ __forceinline__ void epi_write_rows_simple(const float* __restrict__ stage, int SW, int r0, int lane, int Q, int m0,
                                                      const EpiBlock& B) {
    const int dr = 32 / Q, dq = 32 - dr * Q;
    int rl = lane / Q, q = lane - rl * Q;
    for (; rl < 32; rl += dr, q += dq) {
        if (q >= Q) { q -= Q; ++rl; if (rl >= 32) break; }
        const EpiHalf& H = (q < B.qsplit) ? B.h[0] : B.h[1];
        const int m = m0 + rl;
        if (m < H.lo || m >= H.hi) continue;
        const float4 o = *reinterpret_cast<const float4*>(stage + (size_t)(r0 + rl) * SW + 4 * q);
        *reinterpret_cast<float4*>(H.dst + m * H.rstride + 4 * q) = o;
    }
}
// dgrad form: the LeakyReLU-slope read of the saved activation and the accumulate read of the destination are issued for
// kEpiBatch items BEFORE any of them is used (memory-level parallelism: otherwise the store loop is a chain of dependent loads).
constexpr int kEpiBatch = 2;
__device__ __forceinline__ void epi_write_rows_vec(const float* __restrict__ stage, int SW, int r0, int lane, int Q, int m0,
                                                   const EpiBlock& B) {
    const int dr = 32 / Q, dq = 32 - dr * Q;
    int rl = lane / Q, q = lane - rl * Q;
    while (rl < 32) {
        float4 o[kEpiBatch], sv[kEpiBatch], old[kEpiBatch];
        float* dst[kEpiBatch];
        unsigned flags = 0;           // per item: bit u = valid, bit 8+u = slope, bit 16+u = accumulate
#pragma unroll
        for (int u = 0; u < kEpiBatch; ++u) {
            if (q >= Q) { q -= Q; ++rl; }
            if (rl < 32) {
                const EpiHalf& H = (q < B.qsplit) ? B.h[0] : B.h[1];
                const int m = m0 + rl;
                if (m >= H.lo && m < H.hi) {
                    const int off = m * H.rstride + 4 * q;
                    dst[u] = H.dst + off;
                    o[u] = *reinterpret_cast<const float4*>(stage + (size_t)(r0 + rl) * SW + 4 * q);
                    flags |= 1u << u;
                    if (H.saved) { sv[u] = __ldg(reinterpret_cast<const float4*>(H.saved + off)); flags |= 0x100u << u; }
                    if (m >= H.acc_lo && m < H.acc_hi) { old[u] = *reinterpret_cast<const float4*>(dst[u]); flags |= 0x10000u << u; }
                }
            }
            rl += dr; q += dq;
        }
#pragma unroll
        for (int u = 0; u < kEpiBatch; ++u) {
            if (!(flags & (1u << u))) continue;
            float4 v = o[u];
            if (flags & (0x100u << u)) {
                v.x *= (sv[u].x > 0.f) ? 1.f : 0.2f; v.y *= (sv[u].y > 0.f) ? 1.f : 0.2f;
                v.z *= (sv[u].z > 0.f) ? 1.f : 0.2f; v.w *= (sv[u].w > 0.f) ? 1.f : 0.2f;
            }
            if (flags & (0x10000u << u)) { v.x += old[u].x; v.y += old[u].y; v.z += old[u].z; v.w += old[u].w; }
            *reinterpret_cast<float4*>(dst[u]) = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// the conv kernel
// ------------------------------------------------------------------------------------------------
constexpr int kConvThreads = 256;      // two warpgroups: rows [0, 64) and [64, 128) of the tile
constexpr int kBStagesMax = 6;         // weight ring: L.nbs stages of up to L.TB taps

// One step of a CTA's K loop = one weight-ring stage: taps [t0, t0 + nt) (relative to the group) of 16-channel chunk c of
// group g; blk = index of its first packed weight block (pack order: group, chunk, term).
struct ConvStep {
    int g, c, t0, nt, blk;
};
// Moves s to the next step (from g = -1: to the first one), skipping groups whose slab would be all zeros together with
// their packed blocks.  false = the K loop is done.
__device__ __forceinline__ bool next_step(const UmmaLaunch& L, const UmmaClass& K, int m_base, ConvStep& s) {
    if (s.g >= 0) {
        const UmmaGroup& G = K.groups[s.g];
        const int nterm = G.term_end - G.term_begin;
        s.blk += s.nt;
        s.t0 += s.nt;
        if (s.t0 < nterm) { s.nt = min(L.TB, nterm - s.t0); return true; }
        s.t0 = 0;
        if (++s.c < ((L.planes[G.plane].C + 15) >> 4)) { s.nt = min(L.TB, nterm); return true; }
    }
    for (++s.g; s.g < K.ngroups; ++s.g) {
        const UmmaGroup& G = K.groups[s.g];
        const int nterm = G.term_end - G.term_begin;
        if (!group_is_empty(L, G, m_base)) { s.c = 0; s.t0 = 0; s.nt = min(L.TB, nterm); return true; }
        s.blk += ((L.planes[G.plane].C + 15) >> 4) * nterm;
    }
    return false;
}

// Moves s from any step of its (group, chunk) to the first step of the next non-empty (group, chunk).  false = none left.
__device__ __forceinline__ bool next_chunk(const UmmaLaunch& L, const UmmaClass& K, int m_base, ConvStep& s) {
    const UmmaGroup& G = K.groups[s.g];
    s.nt = (G.term_end - G.term_begin) - s.t0;      // as if this step ran to the chunk's last tap
    return next_step(L, K, m_base, s);
}

// The slab of (group, chunk) holds plane rows m_base + dmin + [0, rows_alloc), 16 channels, as hi / lo atom planes.  Each thread
// owns one slab row (rows_alloc <= 152 < kConvThreads; threads past the slab redo its last row: the same bits to the same
// address), and nothing branches on the thread index: a row outside the plane's valid rows has its loads predicated off and is
// zeroed by a select.  slab_load only issues the global loads and slab_store converts and stores them, so that a step can keep
// the next chunk's loads in flight while it waits for its previous step's MMAs.
struct SlabRow {
    float x[16], nx[16];       // the row, and (MID planes) its successor
    bool valid, has_next;
};
// 4 floats at q if ld, else zeros: a predicated load (no branch; rows outside the plane cost no memory traffic)
__device__ __forceinline__ void ldg4_if(bool ld, const float* q, float* x) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t"
                 "mov.b32 %0, 0;\n\tmov.b32 %1, 0;\n\tmov.b32 %2, 0;\n\tmov.b32 %3, 0;\n\t"
                 "@p ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];\n\t}"
                 : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3])
                 : "l"(q), "r"((int)ld));
}
__device__ __forceinline__ void load16(bool ld, const float* p, int nv, float* x) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (i < 2 || nv >= 16) ldg4_if(ld, p + 4 * i, x + 4 * i);
        else { x[4 * i] = 0.f; x[4 * i + 1] = 0.f; x[4 * i + 2] = 0.f; x[4 * i + 3] = 0.f; }
    }
}
__device__ __forceinline__ void slab_load(const PlaneView& P, int b, int r, int c0, SlabRow& R) {
    const int nv = min(16, P.C - c0);      // 8 or 16 (eligibility: C % 8 == 0)
    R.valid = r >= P.r_lo && r < P.r_hi;
    const int rc = min(max(r, P.r_lo), P.r_hi - 1);      // a group's slab has a valid row (group_is_empty)
    const float* p = P.base + (long long)b * P.bstride + (long long)rc * P.rstride + c0;
    load16(R.valid, p, nv, R.x);
    if (P.kind == PLANE_MID) {
        R.has_next = (P.mid_mode == MID_VALID) || (rc + 1 < P.xrows);
        load16(R.valid && R.has_next, p + P.rstride, nv, R.nx);
    }
}
__device__ __forceinline__ void slab_store(const PlaneView& P, int c0, SlabRow& R, uint8_t* S, uint32_t atom, int rr) {
    const int nv = min(16, P.C - c0);
    if (P.kind == PLANE_MID) {
#pragma unroll
        for (int i = 0; i < 16; ++i) R.nx[i] = R.has_next ? R.nx[i] : (P.mid_mode == MID_CLAMP ? R.x[i] : 0.f);
        mid_blend(P, c0, nv, R.x, R.nx);
    }
    uint32_t hi[8], lo[8];
#pragma unroll
    for (int i = 0; i < 16; ++i) R.x[i] = R.valid ? R.x[i] : 0.f;
    split_hi_lo(R.x, hi, lo);
    *reinterpret_cast<uint4*>(S + 16u * rr) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(S + atom + 16u * rr) = make_uint4(hi[4], hi[5], hi[6], hi[7]);
    *reinterpret_cast<uint4*>(S + 2 * atom + 16u * rr) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    *reinterpret_cast<uint4*>(S + 3 * atom + 16u * rr) = make_uint4(lo[4], lo[5], lo[6], lo[7]);
}

// Taps per weight-ring stage: ~16 KB of packed weights, 1..4 taps.  A function of NPAD alone, so that the kernel's tap loop has a
// trip count fixed at compile time; the planner reports the same value.
constexpr __host__ __device__ int conv_stage_taps(int NPAD) {
    return 16384 / (64 * NPAD) > 4 ? 4 : (16384 / (64 * NPAD) < 1 ? 1 : 16384 / (64 * NPAD));
}

// The MMAs of one K step, nt taps (1 <= nt <= NT) with row shifts d[0 .. nt), committed as one group.  Every tap count gets its
// own straight-line sequence: ptxas closes an MMA group at the end of every basic block that issues MMAs, so taps behind a
// per-tap `if` would each be a group, and wait_group 1 after the step would then retire all but the last of them.
template <int NPAD, int NT>
__device__ __forceinline__ void conv_step_mmas(int nt, float* acc, uint32_t sa, uint32_t sb, uint32_t atom, const int* d, int dmin) {
    if constexpr (NT > 1) {
        if (nt < NT) { conv_step_mmas<NPAD, NT - 1>(nt, acc, sa, sb, atom, d, dmin); return; }
    }
    constexpr uint32_t blk_bytes = 64u * NPAD;
#pragma unroll
    for (int tt = 0; tt < NT; ++tt) {
        const uint32_t a = sa + 16u * (uint32_t)(d[tt] - dmin);
        const uint32_t bb = sb + tt * blk_bytes;
        const uint64_t a_hi = gmma_desc(a, atom, 128), a_lo = gmma_desc(a + 2 * atom, atom, 128);
        const uint64_t b_hi = gmma_desc(bb, 32u * NPAD, 128), b_lo = gmma_desc(bb + 16u * NPAD, 32u * NPAD, 128);
        wgmma_tile<NPAD, 0>(acc, a_lo, b_hi);
        wgmma_tile<NPAD, 0>(acc, a_hi, b_lo);
        wgmma_tile<NPAD, 0>(acc, a_hi, b_hi);
    }
    wgmma_commit();
}

static __host__ __device__ size_t conv_smem_bytes(int NPAD, int rows_alloc, int TB, int nbs) {
    const size_t pipe = 2 * 64 * (size_t)rows_alloc + (size_t)nbs * TB * 64 * NPAD;
    const size_t epi = 128 * ((size_t)NPAD + 4) * 4;
    return ((pipe > epi ? pipe : epi) + 127) / 128 * 128 + kBStagesMax * 8 + 4 * (size_t)NPAD;
}

// grid = (row tiles of 128, output-channel splits, batch * classes).  Shared memory: two slabs, the weight ring, the ring's
// mbarriers, this split's bias; the epilogue re-uses the slabs + ring as a 128 x (NPAD + 4) fp32 staging tile.
template <int NPAD, bool DG>
__global__ void __launch_bounds__(kConvThreads, 2) plane_conv_umma_kernel(const __grid_constant__ UmmaLaunch L) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // warp-uniform for the compiler: an MMA operand it thinks may diverge makes it serialize the MMAs
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
    const int cls = blockIdx.z % L.ncls, b = blockIdx.z / L.ncls;
    const UmmaClass& K = L.cls[cls];
    const int split = blockIdx.y;
    const int m_base = K.out.m_lo + blockIdx.x * 128;
    if (m_base >= K.out.m_hi) return;

    const uint32_t atom = 16u * L.rows_alloc;
    const uint32_t slab_bytes = 4u * atom;
    constexpr uint32_t blk_bytes = 64u * NPAD;               // [hi a0|hi a1|lo a0|lo a1] x NPAD rows x 16 B ... see umma_pack_kernel
    constexpr int TB = conv_stage_taps(NPAD);                // == L.TB (launch_plane_conv_umma checks)
    constexpr uint32_t stage_bytes = blk_bytes * TB;
    uint8_t* ring = smem + 2 * slab_bytes;
    const size_t pipe = 2 * (size_t)slab_bytes + (size_t)L.nbs * stage_bytes, epi = 128u * (NPAD + 4) * 4u;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ((pipe > epi ? pipe : epi) + 127) / 128 * 128);
    float* bias_s = reinterpret_cast<float*>(bars + kBStagesMax);
    const uint32_t bar0 = smem_u32(bars);
    for (int i = tid; i < NPAD; i += kConvThreads) {
        const int n = split * NPAD + i;
        bias_s[i] = (L.bias && n < L.N) ? __ldg(L.bias + ((L.pairC > 0 && n >= L.pairC) ? n - L.pairC : n)) : 0.f;
    }
    if (tid == 0) {
        for (int i = 0; i < L.nbs; ++i) mbar_init(bar0 + 8u * i, 1);
        fence_barrier_init();
    }
    __syncthreads();

    // Everything the K loop branches on (cur, ld, the fill target) depends only on L, blockIdx and the step counter.
    const uint8_t* wsrc = K.wpack[split];
    ConvStep cur = {-1, 0, 0, 0, 0};
    bool more = next_step(L, K, m_base, cur);
    ConvStep ld = cur;                  // the next step whose weights are still to be loaded
    bool ld_more = more;
    for (int i = 0; i < L.nbs && ld_more; ++i) {
        bulk_g2s_thread0(tid, smem_u32(ring + i * stage_bytes), wsrc + (size_t)ld.blk * blk_bytes, blk_bytes * ld.nt, bar0 + 8u * i);
        ld_more = next_step(L, K, m_base, ld);
    }
    const int row = min(tid, L.rows_alloc - 1);       // this thread's slab row
    SlabRow R;
    if (more) {
        const UmmaGroup& G = K.groups[cur.g];
        slab_load(L.planes[G.plane], b, m_base + G.dmin + row, cur.c * 16, R);
        slab_store(L.planes[G.plane], cur.c * 16, R, smem, atom, row);
    }
    fence_proxy_async();                // generic-proxy slab writes -> visible to the tensor core (async proxy)
    __syncthreads();

    // Step s = one ring stage: TB taps (fewer at the end of a group) of one chunk, 3 MMAs per tap.  The MMAs of step s stay in
    // flight until step s + 1 has issued its own: wait_group 1 retires step s - 1 only, and after the block barrier that follows
    // it, step s - 1's ring stage takes the weights of step s - 1 + nbs.  The first step of a chunk issues the loads of the
    // next chunk's slab rows before that wait and converts them into the other slab after the barrier, once the previous
    // chunk's last step (its last reader) has retired in both warpgroups.
    float acc[NPAD / 2];
#pragma unroll
    for (int i = 0; i < NPAD / 2; ++i) acc[i] = 0.f;
    int slab = 0, st = 0, phase = 0, st_prev = -1;     // ring stage of step s, its mbarrier phase, the stage of step s - 1
    for (int s = 0; more; ++s) {
        mbar_wait(bar0 + 8u * st, phase);
        const UmmaGroup& G = K.groups[cur.g];
        const uint32_t sa = smem_u32(smem + slab * slab_bytes) + 64u * 16u * wg;
        const uint32_t sb = smem_u32(ring + st * stage_bytes);
        wgmma_fence();
        conv_step_mmas<NPAD, TB>(cur.nt, acc, sa, sb, atom, L.d + G.term_begin + cur.t0, G.dmin);
        ConvStep fc = cur;              // the chunk whose slab this step fills
        const bool fill = cur.t0 == 0 && next_chunk(L, K, m_base, fc);
        const PlaneView& FP = L.planes[K.groups[fc.g].plane];
        if (fill) slab_load(FP, b, m_base + K.groups[fc.g].dmin + row, fc.c * 16, R);
        // the bookkeeping of this step runs while the MMAs do
        ConvStep nx = cur;
        more = next_step(L, K, m_base, nx);
        const bool new_slab = more && nx.t0 == 0;
        const bool refill = st_prev >= 0 && ld_more;
        const ConvStep lw = ld;
        if (refill) ld_more = next_step(L, K, m_base, ld);
        wgmma_wait<1>();
        __syncthreads();
        if (refill)
            bulk_g2s_thread0(tid, smem_u32(ring + st_prev * stage_bytes), wsrc + (size_t)lw.blk * blk_bytes, blk_bytes * lw.nt,
                             bar0 + 8u * st_prev);
        st_prev = st;
        if (++st == L.nbs) { st = 0; phase ^= 1; }
        if (fill) {
            slab_store(FP, fc.c * 16, R, smem + (slab ^ 1) * slab_bytes, atom, row);
            fence_proxy_async();
            if (new_slab) __syncthreads();      // read by the very next step (otherwise the next step's barrier orders it)
        }
        if (new_slab) slab ^= 1;
        cur = nx;
    }
    wgmma_wait<0>();
    acc_fence<NPAD / 2>(acc);
    __syncthreads();

    // ===================== epilogue =====================
    // every MMA has retired and every weight copy has landed: the pipeline memory becomes the staging tile
    float* stage = reinterpret_cast<float*>(smem);
    constexpr int SW = NPAD + 4;                             // padded row stride (floats)
#pragma unroll
    for (int i = 0; i < NPAD / 2; i += 2) {
        const int col = acc_col(i, lane), row = 64 * wg + acc_row(i, warp, lane);
        float v0 = acc[i], v1 = acc[i + 1];
        if (L.epilogue == EPI_BIAS_LRELU) {
            v0 += bias_s[col]; v1 += bias_s[col + 1];
            v0 = fmaxf(0.2f * v0, v0); v1 = fmaxf(0.2f * v1, v1);
        }
        *reinterpret_cast<float2*>(stage + row * SW + col) = make_float2(v0, v1);
    }
    __syncthreads();
    const int n0 = split * NPAD;
    const int ncols = min(NPAD, L.N - n0);
    if (ncols <= 0) return;
    const bool vec = (ncols % 4 == 0) && (K.out.rstride % 4 == 0) && ((reinterpret_cast<uintptr_t>(K.out.base) & 15) == 0) &&
                     ((K.out.bstride & 3) == 0);
    if (vec) {      // (pair-merged classes always take this path: the planner checks both views)
        // warp w writes rows 32 (w % 4) + [0, 32) of one half of the column quads
        const int Q = ncols >> 2, Qa = (Q + 1) >> 1;
        const int q0 = (warp >= 4) ? Qa : 0, nq = (warp >= 4) ? Q - Qa : Qa;
        if (nq <= 0) return;
        const EpiBlock EB = epi_block<true>(K.out, b, n0 + 4 * q0, nq, L.epilogue == EPI_SLOPE);
        if (DG) epi_write_rows_vec(stage + 4 * q0, SW, (warp & 3) * 32, lane, nq, m_base + (warp & 3) * 32, EB);
        else epi_write_rows_simple(stage + 4 * q0, SW, (warp & 3) * 32, lane, nq, m_base + (warp & 3) * 32, EB);
    } else {
        const long long tile_off = (long long)b * K.out.bstride + n0;
        for (int it = tid; it < 128 * ncols; it += kConvThreads) {
            const int r = it / ncols, j = it - r * ncols;
            const int m = m_base + r;
            if (m >= K.out.m_hi) continue;
            const long long roff = tile_off + (long long)m * K.out.rstride;
            float o = stage[r * SW + j];
            if (L.epilogue == EPI_SLOPE && K.out.saved) o *= (__ldg(K.out.saved + roff + j) > 0.f) ? 1.f : 0.2f;
            float* dst = K.out.base + roff + j;
            if (m >= K.out.acc_lo && m < K.out.acc_hi) o += *dst;
            *dst = o;
        }
    }
}

size_t umma_smem_bytes(const UmmaLaunch& L) { return conv_smem_bytes(L.NPAD, L.rows_alloc, L.TB, L.nbs); }
size_t umma_choice_smem_bytes(const UmmaChoice& ch) { return conv_smem_bytes(ch.NPAD, ch.rows_alloc, ch.TB, ch.nbs); }

// The output layer stays in its own kernels (kernels_simt.cu): the conv epilogue holds 64 x NPAD accumulators per warpgroup in
// registers, which leaves no room for the output convs, the loss and their gradients.
bool umma_output_fusable(const ConvLaunch&, const UmmaChoice&, const OutputLaunch&) { return false; }

constexpr int kConvSmemMax = 200 * 1024;      // opt-in limit set for every conv instantiation (the planner stays far below)

template <int NPAD>
static cudaError_t launch_conv_npad(const UmmaLaunch& L, dim3 grid, size_t smem, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(plane_conv_umma_kernel<NPAD, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvSmemMax);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(plane_conv_umma_kernel<NPAD, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvSmemMax);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    // dgrad (EPI_SLOPE / EPI_PLAIN): batched read-back epilogue with the accumulate ranges (separate instantiation)
    if (L.epilogue != EPI_BIAS_LRELU) plane_conv_umma_kernel<NPAD, true><<<grid, kConvThreads, smem, stream>>>(L);
    else plane_conv_umma_kernel<NPAD, false><<<grid, kConvThreads, smem, stream>>>(L);
    return cudaGetLastError();
}

cudaError_t launch_plane_conv_umma(const UmmaLaunch& L, cudaStream_t stream, const OutputFuse* fuse) {
    if (fuse) return cudaErrorInvalidValue;
    int max_tiles = 0;
    for (int q = 0; q < L.ncls; ++q) max_tiles = max(max_tiles, (L.cls[q].out.m_hi - L.cls[q].out.m_lo + 127) / 128);
    if (max_tiles <= 0) return cudaSuccess;
    const size_t smem = umma_smem_bytes(L);
    if (smem > (size_t)kConvSmemMax || L.nbs < 2 || L.nbs > kBStagesMax || L.MT != 1 || L.TB != conv_stage_taps(L.NPAD))
        return cudaErrorInvalidValue;
    const dim3 grid(max_tiles, L.nsplit, L.batch * L.ncls);
    switch (L.NPAD) {
        case 16: return launch_conv_npad<16>(L, grid, smem, stream);
        case 32: return launch_conv_npad<32>(L, grid, smem, stream);
        case 48: return launch_conv_npad<48>(L, grid, smem, stream);
        case 64: return launch_conv_npad<64>(L, grid, smem, stream);
        case 80: return launch_conv_npad<80>(L, grid, smem, stream);
        case 96: return launch_conv_npad<96>(L, grid, smem, stream);
        case 112: return launch_conv_npad<112>(L, grid, smem, stream);
        case 128: return launch_conv_npad<128>(L, grid, smem, stream);
        default: return cudaErrorInvalidValue;
    }
}

// ------------------------------------------------------------------------------------------------
// wgrad kernels (MN-major operands: K = rows).  Stage layout per side: [hi|lo][atom (8 ch)][row][16 B]; for an MN-major
// no-swizzle operand the 8x8 core matrix is 8 rows (K) x 16 B, K groups LBO = 128 B apart, channel atoms SBO = atom-plane
// stride apart.  A tap is again a start-address shift (d rows * 16 B) of the P side.
// grid = (batch * chunks_per_batch / chunks_per_cta, n_mtiles * n_ntiles, tap sets of all groups).  Warps 0-7: two
// warpgroups, each owning one 64-channel M block of the 128-channel tile and a subset of the CTA's taps (wgrad_body),
// accumulators taps x NT in registers; warps 8..: the stage producer.
// ------------------------------------------------------------------------------------------------
constexpr int kWgRK = 64;          // rows per pipeline stage
constexpr int kWgSpan = 16;        // extra P rows per stage (max tap shift span)
constexpr int kWgStagesMax = 3;    // pipeline stages: as many as fit in shared memory (L.nstages)
constexpr int kWgMmaThreads = 256;
constexpr int kWgAccCols = 256;    // accumulator columns (taps x NT) per warpgroup: 128 fp32 registers per thread
constexpr int kWgConvThreads = 128;                 // converter-fed kernel: 4 converter warps
constexpr int kWgSmemMax = 200 * 1024;
constexpr int kWgSlotFloats = 128 * kWgAccCols;     // one CTA's partial tile: [tap][128 M rows][NT]

// Taps one CTA (and so one warpgroup) holds accumulators for: as many NT-column tiles as 128 registers per thread take, at most
// a group's kWgMaxTaps.
constexpr __host__ __device__ int wgrad_max_taps(int NT) { return kWgAccCols / NT < kWgMaxTaps ? kWgAccCols / NT : kWgMaxTaps; }

// The MMAs of one 64-row chunk for one warpgroup: nt taps (0 <= nt <= T), 4 k16 steps x 3 MMAs per tap, committed as one group.
// As in conv_step_mmas, every tap count gets its own straight-line sequence, so that wait_group 1 after the chunk really keeps
// this chunk in flight instead of retiring all its taps but the last.  offA / offB: per tap, the byte shift of each operand.
template <int NT, int T>
__device__ __forceinline__ void wgrad_chunk_mmas(int nt, float* acc, uint32_t sa, uint32_t sb, uint32_t planeA, uint32_t planeB,
                                                 const uint32_t* offA, const uint32_t* offB) {
    if constexpr (T > 0) {
        if (nt < T) { wgrad_chunk_mmas<NT, T - 1>(nt, acc, sa, sb, planeA, planeB, offA, offB); return; }
    }
    constexpr uint32_t atomsA = 16, atomsB = NT / 8;
#pragma unroll
    for (int t = 0; t < T; ++t) {
#pragma unroll
        for (int ks = 0; ks < kWgRK / 16; ++ks) {
            const uint32_t a = sa + offA[t] + 256u * ks, bb = sb + offB[t] + 256u * ks;
            const uint64_t a_hi = gmma_desc(a, 128, planeA), a_lo = gmma_desc(a + atomsA * planeA, 128, planeA);
            const uint64_t b_hi = gmma_desc(bb, 128, planeB), b_lo = gmma_desc(bb + atomsB * planeB, 128, planeB);
            wgmma_tile<NT, 1>(acc + t * (NT / 2), a_lo, b_hi);
            wgmma_tile<NT, 1>(acc + t * (NT / 2), a_hi, b_lo);
            wgmma_tile<NT, 1>(acc + t * (NT / 2), a_hi, b_hi);
        }
    }
    wgmma_commit();
}

template <bool BULK, int NT>
__device__ __forceinline__ void wgrad_body(const UmmaWgradLaunch& L, const WgSplit* S) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // group / tap set of this CTA
    int gi = 0;
    while (gi + 1 < L.ngroups && (int)blockIdx.z >= L.grp[gi + 1].z0) ++gi;
    const WgGroup& Gp = L.grp[gi];
    const int tapset = blockIdx.z - Gp.z0;
    if ((int)blockIdx.x >= Gp.n_ctas_x || (int)blockIdx.y >= Gp.n_mtiles * Gp.n_ntiles || Gp.NT != NT) return;
    const int total_chunks = L.batch * Gp.chunks_per_batch;
    const int g0 = blockIdx.x * Gp.chunks_per_cta;
    const int g1 = min(g0 + Gp.chunks_per_cta, total_chunks);
    if (g0 >= g1) return;
    const int mtile = blockIdx.y / Gp.n_ntiles, ntile = blockIdx.y % Gp.n_ntiles;
    const int tap0 = tapset * Gp.taps_per_cta;
    const int ntap = min(Gp.taps_per_cta, Gp.ntaps - tap0);
    const int swap = Gp.swap;
    const PlaneView& SA = swap ? Gp.G : Gp.P;       // M side (128-channel tile)
    const PlaneView& SB = swap ? Gp.P : Gp.G;       // N side (NT-channel tile)
    const int ca0 = mtile * 128, cb0 = ntile * NT;
    const int rowsA = swap ? kWgRK : kWgRK + kWgSpan;
    const int rowsB = swap ? kWgRK + kWgSpan : kWgRK;
    const uint32_t planeA = 16u * rowsA, planeB = 16u * rowsB;           // atom-plane strides
    constexpr int atomsA = 16, atomsB = NT / 8;
    const uint32_t bytesA = 2u * atomsA * planeA, bytesB = 2u * atomsB * planeB;
    const uint32_t stage_bytes = bytesA + bytesB;
    int dmin = Gp.d[tap0];
    for (int t = 1; t < ntap; ++t) dmin = min(dmin, Gp.d[tap0 + t]);

    const int nst = L.nstages;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + nst * stage_bytes);
    const uint32_t bar0 = smem_u32(bars);
    auto BAR = [&](int i) { return bar0 + 8u * i; };
    const int FULL = 0, EMPTY = kWgStagesMax;
    if (tid == 0) {
        for (int i = 0; i < kWgStagesMax; ++i) { mbar_init(BAR(FULL + i), BULK ? 1 : kWgConvThreads); mbar_init(BAR(EMPTY + i), kWgMmaThreads); }
        fence_barrier_init();
    }
    // channel chunks the tensors really have inside this tile; the bulk copies leave the rest of the operand tile zero
    const int chunksA = max(0, min(8, (SA.C - ca0 + 15) / 16)), chunksB = max(0, min(NT / 16, (SB.C - cb0 + 15) / 16));
    if (BULK) {
        for (uint32_t i = tid; i < (uint32_t)nst * stage_bytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
        fence_proxy_async();
    }
    __syncthreads();
    const int nchunks = g1 - g0;

    if (warp >= kWgMmaThreads / 32) {
        // ===================== producer =====================
        if (BULK) {
            if (warp == kWgMmaThreads / 32 && lane == 0) {
                const uint8_t* baseA = swap ? S->G[gi] : S->P[gi];
                const uint8_t* baseB = swap ? S->P[gi] : S->G[gi];
                const long long a_ps = swap ? S->g_pstride[gi] : S->p_pstride[gi], b_ps = swap ? S->p_pstride[gi] : S->g_pstride[gi];
                const long long a_cs = 4 * a_ps, b_cs = 4 * b_ps;
                const long long a_bs = (swap ? S->g_nchunk[gi] : S->p_nchunk[gi]) * a_cs, b_bs = (swap ? S->p_nchunk[gi] : S->g_nchunk[gi]) * b_cs;
                const int a_row0 = swap ? S->g_row0[gi] : S->p_row0[gi], b_row0 = swap ? S->p_row0[gi] : S->g_row0[gi];
                const uint32_t tx = (uint32_t)(chunksA * 4) * planeA + (uint32_t)(chunksB * 4) * planeB;
                for (int ci = 0; ci < nchunks; ++ci) {
                    const int st = ci % nst;
                    const int gch = g0 + ci;
                    const int b = gch / Gp.chunks_per_batch;
                    const int rc = Gp.m_lo + (gch % Gp.chunks_per_batch) * kWgRK;      // first G row of the chunk
                    const int rowA = (swap ? rc : rc + dmin) - a_row0, rowB = (swap ? rc + dmin : rc) - b_row0;   // array indices
                    mbar_wait(BAR(EMPTY + st), ((ci / nst) & 1) ^ 1);
                    mbar_arrive_expect_tx(BAR(FULL + st), tx);
                    const uint32_t sa = smem_u32(smem + st * stage_bytes), sb = sa + bytesA;
                    for (int g = 0; g < chunksA; ++g) {
                        const uint8_t* src = baseA + (long long)b * a_bs + (long long)(ca0 / 16 + g) * a_cs + (long long)rowA * 16;
                        bulk_g2s(sa + (uint32_t)(2 * g) * planeA, src, planeA, BAR(FULL + st));                               // hi atom 2g
                        bulk_g2s(sa + (uint32_t)(2 * g + 1) * planeA, src + a_ps, planeA, BAR(FULL + st));                    // hi atom 2g+1
                        bulk_g2s(sa + (uint32_t)(atomsA + 2 * g) * planeA, src + 2 * a_ps, planeA, BAR(FULL + st));           // lo atom 2g
                        bulk_g2s(sa + (uint32_t)(atomsA + 2 * g + 1) * planeA, src + 3 * a_ps, planeA, BAR(FULL + st));       // lo atom 2g+1
                    }
                    for (int g = 0; g < chunksB; ++g) {
                        const uint8_t* src = baseB + (long long)b * b_bs + (long long)(cb0 / 16 + g) * b_cs + (long long)rowB * 16;
                        bulk_g2s(sb + (uint32_t)(2 * g) * planeB, src, planeB, BAR(FULL + st));
                        bulk_g2s(sb + (uint32_t)(2 * g + 1) * planeB, src + b_ps, planeB, BAR(FULL + st));
                        bulk_g2s(sb + (uint32_t)(atomsB + 2 * g) * planeB, src + 2 * b_ps, planeB, BAR(FULL + st));
                        bulk_g2s(sb + (uint32_t)(atomsB + 2 * g + 1) * planeB, src + 3 * b_ps, planeB, BAR(FULL + st));
                    }
                }
            }
        } else {
            // items of a chunk: (side, row, 16-channel group); A side = 8 groups (128 channels), B side = NT/16 groups
            const int ctid = tid - kWgMmaThreads;
            const int gA = 8, gB = NT / 16;
            const int itemsA = rowsA * gA, items = itemsA + rowsB * gB;
            for (int ci = 0; ci < nchunks; ++ci) {
                const int st = ci % nst;
                uint8_t* Sm = smem + st * stage_bytes;
                const int gch = g0 + ci;                              // batch-folded chunk index
                const int b = gch / Gp.chunks_per_batch;
                const int rc = Gp.m_lo + (gch % Gp.chunks_per_batch) * kWgRK;   // first G row of this chunk
                const int rend = min(rc + kWgRK, Gp.m_hi);
                mbar_wait(BAR(EMPTY + st), ((ci / nst) & 1) ^ 1);
                for (int it = ctid; it < items; it += kWgConvThreads) {
                    const bool isA = it < itemsA;
                    const int k = isA ? it : it - itemsA;
                    const int nr = isA ? rowsA : rowsB;        // consecutive threads -> consecutive rows (conflict-free st.shared)
                    const int g = k / nr, rr = k - g * nr;
                    const bool isP = isA != (swap != 0);
                    const PlaneView& V = isA ? SA : SB;
                    const int c0 = (isA ? ca0 : cb0) + g * 16;
                    const int row = isP ? (rc + dmin + rr) : (rc + rr);
                    float x[16];
                    if (c0 < V.C && (isP || row < rend)) load_row16(V, b, row, c0, x);    // G rows beyond the chunk / class contribute 0
                    else {
#pragma unroll
                        for (int i = 0; i < 16; ++i) x[i] = 0.f;
                    }
                    uint32_t hi[8], lo[8];
                    split_hi_lo(x, hi, lo);
                    const uint32_t plane = isA ? planeA : planeB;
                    uint8_t* base = Sm + (isA ? 0u : bytesA) + (uint32_t)(2 * g) * plane + 16u * rr;
                    const uint32_t lo_off = (isA ? atomsA : atomsB) * plane;
                    *reinterpret_cast<uint4*>(base) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                    *reinterpret_cast<uint4*>(base + lo_off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                    *reinterpret_cast<uint4*>(base + plane) = make_uint4(hi[4], hi[5], hi[6], hi[7]);
                    *reinterpret_cast<uint4*>(base + plane + lo_off) = make_uint4(lo[4], lo[5], lo[6], lo[7]);
                }
                fence_proxy_async();
                mbar_arrive(BAR(FULL + st));
            }
        }
        return;
    }

    // ===================== MMA warpgroups =====================
    constexpr int TMAX = wgrad_max_taps(NT);     // >= taps_per_cta (umma_plan_wgrad)
    constexpr int NACC = TMAX * NT / 2;
    // warp-uniform for the compiler: an MMA operand it thinks may diverge makes it serialize the MMAs
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
    // What this warpgroup owns: a tile whose two 64-channel M blocks both hold real channels gives block wg to warpgroup wg, with
    // all the CTA's taps; a tile with one such block (an M side of <= 64 channels, or the last block of a 144-channel side) gives
    // that block to both warpgroups and splits the taps between them.  No warpgroup multiplies a block of padding.
    const bool tsplit = SA.C - ca0 <= 64;
    const int th = (ntap + 1) >> 1;
    const int wt0 = (tsplit && wg) ? th : 0;                  // first of this warpgroup's taps, relative to tap0
    const int wnt = tsplit ? (wg ? ntap - th : th) : ntap;   // its tap count (0 for warpgroup 1 of a one-tap tile split)
    const int mrow0 = tsplit ? 0 : 64 * wg;                  // its first M row in the tile
    uint32_t offA[TMAX], offB[TMAX];                         // per tap: the row shift (16 B per row) of the P side's operand
#pragma unroll
    for (int t = 0; t < TMAX; ++t) {
        const uint32_t shift = t < wnt ? 16u * (uint32_t)(Gp.d[tap0 + wt0 + t] - dmin) : 0u;
        offA[t] = swap ? 0u : shift;
        offB[t] = swap ? shift : 0u;
    }
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    for (int ci = 0; ci < nchunks; ++ci) {
        const int st = ci % nst;
        mbar_wait(BAR(FULL + st), (ci / nst) & 1);
        const uint32_t sa = smem_u32(smem + st * stage_bytes) + (uint32_t)(mrow0 / 8) * planeA, sb = smem_u32(smem + st * stage_bytes) + bytesA;
        wgmma_fence();
        wgrad_chunk_mmas<NT, TMAX>(wnt, acc, sa, sb, planeA, planeB, offA, offB);
        // chunk ci stays in flight while the next stage is awaited: only chunk ci - 1 has surely finished reading its stage
        wgmma_wait<1>();
        if (ci > 0) mbar_arrive(BAR(EMPTY + (ci - 1) % nst));
    }
    wgmma_wait<0>();
    acc_fence<NACC>(acc);
    // ===================== epilogue: accumulators -> partial tile (or reductions into dW) =====================
    // A tap-split tile leaves rows [64, 128) of its slot unwritten: they are channels >= SA.C, which the reduction skips.
    if (L.partial) {
        const int tiles = Gp.n_mtiles * Gp.n_ntiles;
        float* part = L.partial + (size_t)(Gp.slot0 + (tapset * tiles + (int)blockIdx.y) * Gp.n_ctas_x + (int)blockIdx.x) * kWgSlotFloats;
#pragma unroll
        for (int t = 0; t < TMAX; ++t) {
            if (t >= wnt) break;
#pragma unroll
            for (int i = 0; i < NT / 2; i += 2) {
                const int row = mrow0 + acc_row(i, warp, lane), col = acc_col(i, lane);
                *reinterpret_cast<float2*>(part + (size_t)((wt0 + t) * 128 + row) * NT + col) =
                    make_float2(acc[t * (NT / 2) + i] * L.scale, acc[t * (NT / 2) + i + 1] * L.scale);
            }
        }
        return;
    }
    const int sM = swap ? L.w_sg : L.w_sp, sN = swap ? L.w_sp : L.w_sg;
#pragma unroll
    for (int t = 0; t < TMAX; ++t) {
        if (t >= wnt) break;
        float* dst_t = L.dW + Gp.woff[tap0 + wt0 + t];
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) {
            const int m = ca0 + mrow0 + acc_row(i, warp, lane), n = cb0 + acc_col(i, lane);
            if (m < SA.C && n < SB.C) atomicAdd(dst_t + (long long)m * sM + (long long)n * sN, acc[t * (NT / 2) + i] * L.scale);
        }
    }
}

template <int NT>
__global__ void __launch_bounds__(kWgMmaThreads + 32, 1) wgrad_umma_bulk_kernel(const __grid_constant__ UmmaWgradLaunch L,
                                                                                 const __grid_constant__ WgSplit S) {
    wgrad_body<true, NT>(L, &S);
}
template <int NT>
__global__ void __launch_bounds__(kWgMmaThreads + kWgConvThreads, 1) wgrad_umma_kernel(const __grid_constant__ UmmaWgradLaunch L) {
    wgrad_body<false, NT>(L, nullptr);
}

static size_t wgrad_stage_bytes(int swap, int NT) {
    const int rowsA = swap ? kWgRK : kWgRK + kWgSpan, rowsB = swap ? kWgRK + kWgSpan : kWgRK;
    return 2u * 16 * 16 * rowsA + 2u * (NT / 8) * 16 * rowsB;
}

static size_t wgrad_smem_bytes(const UmmaWgradLaunch& L) {
    size_t stage = 0;
    for (int g = 0; g < L.ngroups; ++g) stage = max(stage, wgrad_stage_bytes(L.grp[g].swap, L.grp[g].NT));
    return L.nstages * stage + 2 * kWgStagesMax * 8;
}

size_t umma_wgrad_smem_bytes(const UmmaWgradLaunch& L) { return wgrad_smem_bytes(L); }

// N tiles of an N side of Cn channels: at most 128 wide, 16-multiples
static void wgrad_ntiles(int Cn, int* nt, int* ntiles) {
    *nt = (Cn + 15) / 16 * 16;
    *ntiles = 1;
    while (*nt > 128) { *ntiles *= 2; *nt = ((Cn + *ntiles - 1) / *ntiles + 15) / 16 * 16; }
}

long long umma_wgrad_issued_macs(const WgGroup& G, int batch) {
    const int Cm = G.swap ? G.G.C : G.P.C;
    return (long long)batch * G.chunks_per_batch * kWgRK * G.ntaps * (64LL * ((Cm + 63) / 64)) * G.NT * G.n_ntiles;
}

bool umma_plan_wgrad(UmmaWgradLaunch* L) {
    if (L->ngroups < 1 || L->ngroups > kWgMaxGroups) return false;
    for (int gi = 0; gi < L->ngroups; ++gi) {
        WgGroup& G = L->grp[gi];
        const int Cp = G.P.C, Cg = G.G.C;
        if (Cp % 8 || Cg % 8 || Cp < 16 || Cg < 16 || G.ntaps < 1 || G.ntaps > kWgMaxTaps) return false;
        if (G.P.rstride % 4 || G.G.rstride % 4 || G.P.bstride % 4 || G.G.bstride % 4) return false;
        if ((reinterpret_cast<uintptr_t>(G.P.base) & 15) || (reinterpret_cast<uintptr_t>(G.G.base) & 15)) return false;
        int dmin = G.d[0], dmax = G.d[0];
        for (int t = 1; t < G.ntaps; ++t) { dmin = min(dmin, G.d[t]); dmax = max(dmax, G.d[t]); }
        if (dmax - dmin > kWgSpan) return false;
        if (G.m_hi <= G.m_lo) return false;
        G.chunks_per_batch = (G.m_hi - G.m_lo + kWgRK - 1) / kWgRK;
    }
    // The wider side fills M.  Putting the narrower side on M when that issues fewer MMAs (down2: Cp 48 on one M block, Cg 72
    // in N tiles of 80) measured slower on H100: the wider NT leaves room for fewer taps per CTA, so more tap sets re-stage the
    // same rows (down2's wgrad kernel 393 -> 454 us).
    int NT = 16;               // one N-tile width for all groups: one kernel instantiation per launch
    for (int gi = 0; gi < L->ngroups; ++gi) {
        WgGroup& G = L->grp[gi];
        G.swap = (G.G.C > G.P.C) ? 1 : 0;
        const int Cm = G.swap ? G.G.C : G.P.C, Cn = G.swap ? G.P.C : G.G.C;
        G.n_mtiles = (Cm + 127) / 128;
        int nt;
        wgrad_ntiles(Cn, &nt, &G.n_ntiles);
        NT = max(NT, nt);
    }
    long long work = 0;        // ~MMA work units of the launch, to size the K ranges
    for (int gi = 0; gi < L->ngroups; ++gi) {
        WgGroup& G = L->grp[gi];
        G.NT = NT;
        int tpc = wgrad_max_taps(NT);                     // the accumulators of all taps of a CTA live in registers
        if (tpc > G.ntaps) tpc = G.ntaps;
        G.n_tapsets = (G.ntaps + tpc - 1) / tpc;
        tpc = (G.ntaps + G.n_tapsets - 1) / G.n_tapsets;   // balance
        G.taps_per_cta = tpc;
        work += (long long)L->batch * G.chunks_per_batch * G.n_tapsets * G.n_mtiles * G.n_ntiles;
    }
    // K range per CTA: the launch should be ONE full wave (1 CTA per SM): every CTA runs concurrently and pays the dW
    // reduction once.  Start from work/SMs and grow until the (per-group rounded) CTA count fits.
    const int kSMs = 132;
    long long per = (work + kSMs - 1) / kSMs, most = 1;
    if (per < 2) per = 2;
    for (int gi = 0; gi < L->ngroups; ++gi) most = max(most, (long long)L->batch * L->grp[gi].chunks_per_batch);
    int z = 0, gx = 0, gy = 0, slots = 0;
    for (;;) {              // ends with <= kSMs CTAs, or with one CTA per (group, tile, tap set): umma_wgrad_partial_bytes
        long long ctas = 0;
        for (int gi = 0; gi < L->ngroups; ++gi) {
            const WgGroup& G = L->grp[gi];
            const long long total = (long long)L->batch * G.chunks_per_batch;
            const long long c = min(per, total);
            ctas += ((total + c - 1) / c) * G.n_tapsets * G.n_mtiles * G.n_ntiles;
        }
        if (ctas <= kSMs || per >= most) break;
        per = min(most, per + (per + 15) / 16);
    }
    for (int gi = 0; gi < L->ngroups; ++gi) {
        WgGroup& G = L->grp[gi];
        const long long total = (long long)L->batch * G.chunks_per_batch;
        G.chunks_per_cta = (int)min(per, total);
        G.n_ctas_x = (int)((total + G.chunks_per_cta - 1) / G.chunks_per_cta);
        G.z0 = z;
        z += G.n_tapsets;
        G.slot0 = slots;
        slots += G.n_tapsets * G.n_mtiles * G.n_ntiles * G.n_ctas_x;
        gx = max(gx, G.n_ctas_x);
        gy = max(gy, G.n_mtiles * G.n_ntiles);
    }
    L->grid_x = gx; L->grid_y = gy; L->grid_z = z;
    L->nstages = kWgStagesMax;
    while (L->nstages > 2 && wgrad_smem_bytes(*L) > kWgSmemMax) --L->nstages;
    return wgrad_smem_bytes(*L) <= kWgSmemMax;
}

// the instantiation of the launch's N-tile width (umma_plan_wgrad gives every group the same one)
template <bool BULK>
static cudaError_t launch_wgrad_any(const UmmaWgradLaunch& L, const WgSplit* S, cudaStream_t stream) {
    const dim3 grid(L.grid_x, L.grid_y, L.grid_z);
    const size_t smem = wgrad_smem_bytes(L);
    const int threads = kWgMmaThreads + (BULK ? 32 : kWgConvThreads);
    {
        const int NT = L.grp[0].NT;
        cudaError_t e = cudaSuccess;
#define WUN_WG_CASE(W)                                                                                                      \
    case W:                                                                                                                 \
        if (BULK) {                                                                                                         \
            static bool set = false;                                                                                        \
            if (!set) { e = cudaFuncSetAttribute(wgrad_umma_bulk_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmemMax); set = e == cudaSuccess; } \
            if (e == cudaSuccess) wgrad_umma_bulk_kernel<W><<<grid, threads, smem, stream>>>(L, *S);                       \
        } else {                                                                                                            \
            static bool set = false;                                                                                        \
            if (!set) { e = cudaFuncSetAttribute(wgrad_umma_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmemMax); set = e == cudaSuccess; } \
            if (e == cudaSuccess) wgrad_umma_kernel<W><<<grid, threads, smem, stream>>>(L);                                 \
        }                                                                                                                   \
        break;
        switch (NT) {
            WUN_WG_CASE(16) WUN_WG_CASE(32) WUN_WG_CASE(48) WUN_WG_CASE(64)
            WUN_WG_CASE(80) WUN_WG_CASE(96) WUN_WG_CASE(112) WUN_WG_CASE(128)
            default: return cudaErrorInvalidValue;
        }
#undef WUN_WG_CASE
        if (e != cudaSuccess) return e;
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_wgrad_umma(const UmmaWgradLaunch& L, cudaStream_t stream) { return launch_wgrad_any<false>(L, nullptr, stream); }

// ------------------------------------------------------------------------------------------------
// Bulk-copy-fed wgrad (default).  A batched "split pass" materialises every plane view the layer's wgrad groups read
// (activation planes incl. interpolated MID planes, and the class gradients) as hi/lo bf16 atom planes
// [batch][16-ch chunk][hi a0|hi a1|lo a0|lo a1][row][16 B] with zero rows around the valid range; the wgrad kernel then fills
// its stages with cp.async.bulk issued by ONE thread instead of re-converting the same rows in every (class, plane, tap-set) CTA.
// ------------------------------------------------------------------------------------------------
constexpr int kSplitRB = 2048;     // rows of one (item, 16-channel chunk) a CTA of the split pass covers (8 per thread)

// blockIdx.y = job, blockIdx.x = (item, chunk, row block).  Thread t converts rows rb + t, rb + t + 256, ...; for a class-gradient
// view (job.colsum != null) it also keeps the 16 column sums of its rows, the CTA reduces them (shuffles + shared memory)
// and adds scale * sum to the bias gradient - the layer's bias gradient costs no launch and no extra pass over dPre.
__global__ void __launch_bounds__(256) split_views_kernel(const __grid_constant__ SplitJobs J) {
    const SplitJob& job = J.job[blockIdx.y];
    const int nrb = (job.rows + kSplitRB - 1) / kSplitRB;
    const int total = J.batch * job.nchunk * nrb;
    if ((int)blockIdx.x >= total) return;
    const int rbi = blockIdx.x % nrb, c = (blockIdx.x / nrb) % job.nchunk, b = blockIdx.x / (nrb * job.nchunk);
    const int r_end = min(job.rows, (rbi + 1) * kSplitRB);
    const long long ps = (long long)job.rows * 16;
    uint8_t* obase = job.out + (((long long)b * job.nchunk + c) * 4) * ps;
    float acc[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[k] = 0.f;
    for (int r = rbi * kSplitRB + threadIdx.x; r < r_end; r += 256) {
        float x[16];
        load_row16(job.V, b, job.row0 + r, c * 16, x);      // zero outside the valid rows / channels; MID planes blended here
        uint32_t hi[8], lo[8];
        split_hi_lo(x, hi, lo);
        uint8_t* o = obase + (long long)r * 16;
        *reinterpret_cast<uint4*>(o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        *reinterpret_cast<uint4*>(o + ps) = make_uint4(hi[4], hi[5], hi[6], hi[7]);
        *reinterpret_cast<uint4*>(o + 2 * ps) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        *reinterpret_cast<uint4*>(o + 3 * ps) = make_uint4(lo[4], lo[5], lo[6], lo[7]);
        if (job.colsum) {
#pragma unroll
            for (int k = 0; k < 16; ++k) acc[k] += x[k];
        }
    }
    if (job.colsum) {                                        // uniform per CTA
        __shared__ float red[8][16];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            float v = acc[k];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane == 0) red[warp][k] = v;
        }
        __syncthreads();
        if (threadIdx.x < 16 && c * 16 + (int)threadIdx.x < job.V.C) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x];
            if (job.colsum_part) job.colsum_part[(((long long)b * job.nchunk + c) * nrb + rbi) * 16 + threadIdx.x] = t;
            else atomicAdd(job.colsum + c * 16 + threadIdx.x, t * J.colsum_scale);
        }
    }
}

cudaError_t launch_split_views(const SplitJobs& J, cudaStream_t stream) {
    if (J.njobs <= 0) return cudaSuccess;
    long long most = 0;
    for (int j = 0; j < J.njobs; ++j)
        most = max(most, (long long)J.batch * J.job[j].nchunk * ((J.job[j].rows + kSplitRB - 1) / kSplitRB));
    if (most < 1) return cudaSuccess;
    if (most > 0x7fffffffLL) return cudaErrorInvalidValue;
    split_views_kernel<<<dim3((unsigned)most, J.njobs), 256, 0, stream>>>(J);
    return cudaGetLastError();
}

// Split arena of one layer's bulk-fed wgrad: one array per DISTINCT plane view the groups read (activation planes are shared
// by the classes, class gradients by the planes), covering the union of the row ranges the CTAs touch.  Returns the bytes
// needed at `batch` (arrays 256-B aligned); fills the jobs / operand table when `arena` is not null.
size_t umma_plan_wgrad_split(const UmmaWgradLaunch& U, int batch, uint8_t* arena, WgSplit* S, SplitJobs* J) {
    struct Slot { PlaneView V; int lo, hi; size_t off; };
    std::vector<Slot> slots;
    int p_slot[kWgMaxGroups], g_slot[kWgMaxGroups];
    auto find = [&](const PlaneView& V, int lo, int hi) {
        for (size_t i = 0; i < slots.size(); ++i)
            if (memcmp(&slots[i].V, &V, sizeof(PlaneView)) == 0) {
                slots[i].lo = min(slots[i].lo, lo); slots[i].hi = max(slots[i].hi, hi);
                return (int)i;
            }
        slots.push_back({V, lo, hi, 0});
        return (int)slots.size() - 1;
    };
    for (int g = 0; g < U.ngroups; ++g) {
        const WgGroup& G = U.grp[g];
        int dmin = G.d[0], dmax = G.d[0];
        for (int t = 1; t < G.ntaps; ++t) { dmin = min(dmin, G.d[t]); dmax = max(dmax, G.d[t]); }
        p_slot[g] = find(G.P, G.m_lo + dmin, G.m_hi + dmax + kWgOverreachP);
        g_slot[g] = find(G.G, G.m_lo, G.m_hi + kWgOverreachG);
    }
    if ((int)slots.size() > kSplitMaxJobs) return 0;
    size_t cur = 0;
    for (auto& sl : slots) {
        const int nchunk = (sl.V.C + 15) / 16, rows = (sl.hi - sl.lo + 7) / 8 * 8;
        cur = (cur + 255) / 256 * 256;
        sl.off = cur;
        cur += (size_t)batch * nchunk * 4 * rows * 16;
    }
    std::vector<size_t> part_off(slots.size());       // per-CTA column sums of the views that turn out to be class gradients
    for (size_t i = 0; i < slots.size(); ++i) {
        const int nchunk = (slots[i].V.C + 15) / 16, rows = (slots[i].hi - slots[i].lo + 7) / 8 * 8;
        cur = (cur + 255) / 256 * 256;
        part_off[i] = cur;
        cur += (size_t)batch * nchunk * ((rows + kSplitRB - 1) / kSplitRB) * 16 * sizeof(float);
    }
    if (arena) {
        memset(S, 0, sizeof(*S));
        memset(J, 0, sizeof(*J));
        J->batch = batch; J->njobs = (int)slots.size();
        for (size_t i = 0; i < slots.size(); ++i) {
            SplitJob& job = J->job[i];
            job.V = slots[i].V; job.out = arena + slots[i].off;
            job.nchunk = (slots[i].V.C + 15) / 16; job.rows = (slots[i].hi - slots[i].lo + 7) / 8 * 8; job.row0 = slots[i].lo;
            job.colsum_part = reinterpret_cast<float*>(arena + part_off[i]);
        }
        for (int g = 0; g < U.ngroups; ++g) {
            const SplitJob& jp = J->job[p_slot[g]];
            const SplitJob& jg = J->job[g_slot[g]];
            S->P[g] = jp.out; S->p_pstride[g] = (long long)jp.rows * 16; S->p_nchunk[g] = jp.nchunk; S->p_row0[g] = jp.row0;
            S->G[g] = jg.out; S->g_pstride[g] = (long long)jg.rows * 16; S->g_nchunk[g] = jg.nchunk; S->g_row0[g] = jg.row0;
        }
    }
    return cur + 256;
}

cudaError_t launch_wgrad_umma_bulk(const UmmaWgradLaunch& L, const WgSplit& S, cudaStream_t stream) {
    return launch_wgrad_any<true>(L, &S, stream);
}

bool umma_wgrad_bulk_setup(UmmaWgradLaunch* U, int batch, uint8_t* arena, const PlaneView* class_dpre, int ncls, float* db,
                           float colsum_scale, WgSplit* S, SplitJobs* J) {
    const size_t used = umma_plan_wgrad_split(*U, batch, arena, S, J);
    U->partial = reinterpret_cast<float*>(arena + (used + 255) / 256 * 256);     // behind the split arrays
    J->colsum_scale = colsum_scale;
    int matched = 0;
    for (int j = 0; j < J->njobs; ++j)
        for (int q = 0; q < ncls; ++q)
            if (memcmp(&J->job[j].V, &class_dpre[q], sizeof(PlaneView)) == 0) { J->job[j].colsum = db; ++matched; break; }
    return matched == ncls;
}

size_t umma_wgrad_partial_bytes(const UmmaWgradLaunch& U) {
    long long tiles = 0;                // umma_plan_wgrad: <= kSMs CTAs, or one per (group, tile, tap set)
    for (int g = 0; g < U.ngroups; ++g) tiles += (long long)U.grp[g].n_tapsets * U.grp[g].n_mtiles * U.grp[g].n_ntiles;
    return (size_t)max(tiles, 132LL) * kWgSlotFloats * sizeof(float) + 256;
}

// blockIdx.y < ngroups: the weight gradient of group y, one element of its tap-set tiles per thread iteration, the partial
// tiles of its CTAs along x added in x order; blockIdx.y == ngroups: the bias gradients of the split jobs, their CTAs' column
// sums added in (item, row block) order.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const __grid_constant__ UmmaWgradLaunch L, const __grid_constant__ SplitJobs J) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if ((int)blockIdx.y < L.ngroups) {
        if (!L.partial) return;
        const WgGroup& G = L.grp[blockIdx.y];
        const int NT = G.NT, tpc = G.taps_per_cta, tiles = G.n_mtiles * G.n_ntiles;
        const PlaneView& SA = G.swap ? G.G : G.P;
        const PlaneView& SB = G.swap ? G.P : G.G;
        const int sM = G.swap ? L.w_sg : L.w_sp, sN = G.swap ? L.w_sp : L.w_sg;
        const long long total = (long long)G.n_tapsets * tiles * tpc * 128 * NT;
        for (long long e = i0; e < total; e += stride) {
            long long r = e;
            const int n = (int)(r % NT); r /= NT;
            const int mrow = (int)(r % 128); r /= 128;
            const int t = (int)(r % tpc); r /= tpc;
            const int y = (int)(r % tiles), tapset = (int)(r / tiles);
            const int tap = tapset * tpc + t;
            const int m = (y / G.n_ntiles) * 128 + mrow, nn = (y % G.n_ntiles) * NT + n;
            if (tap >= G.ntaps || m >= SA.C || nn >= SB.C) continue;
            const float* p = L.partial + (size_t)(G.slot0 + (tapset * tiles + y) * G.n_ctas_x) * kWgSlotFloats + (size_t)(t * 128 + mrow) * NT + n;
            float sum = 0.f;
            for (int x = 0; x < G.n_ctas_x; ++x) sum += p[(size_t)x * kWgSlotFloats];
            atomicAdd(L.dW + G.woff[tap] + (long long)m * sM + (long long)nn * sN, sum);
        }
        return;
    }
    long long total = 0;
    for (int j = 0; j < J.njobs; ++j) if (J.job[j].colsum) total += J.job[j].V.C;
    for (long long e = i0; e < total; e += stride) {
        int j = 0;
        long long c = e;
        for (;; ++j) {
            if (!J.job[j].colsum) continue;
            if (c < J.job[j].V.C) break;
            c -= J.job[j].V.C;
        }
        const SplitJob& job = J.job[j];
        const int nrb = (job.rows + kSplitRB - 1) / kSplitRB;
        float sum = 0.f;
        for (int b = 0; b < J.batch; ++b)
            for (int rb = 0; rb < nrb; ++rb) sum += job.colsum_part[(((long long)b * job.nchunk + c / 16) * nrb + rb) * 16 + c % 16];
        atomicAdd(job.colsum + c, sum * J.colsum_scale);
    }
}

cudaError_t launch_wgrad_reduce(const UmmaWgradLaunch& U, const SplitJobs& J, cudaStream_t stream) {
    wgrad_reduce_kernel<<<dim3(132 * 2, U.ngroups + 1), 256, 0, stream>>>(U, J);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// weight pre-pack: fp32 W -> hi/lo bf16 blocks in K-step streaming order.  blockIdx.y = job (class, split).
// Block bi = ((group, chunk), term) in the kernel's loop order; element (a, n, kk) of the hi half sits at byte
// a*32*NPAD + (n/8)*128 + (n%8)*16 + kk*2, the lo half 16*NPAD bytes later: per K atom the block is a K-major
// [hi rows 0..NPAD) | lo rows NPAD..2*NPAD) matrix.
// One thread per (block, K atom, n): 8 k-values -> one 16-byte hi store and one 16-byte lo store (consecutive n = consecutive
// 16 B: coalesced); the fp32 reads are coalesced along n (forward: w_sn = 1) or 32 B contiguous per thread (dgrad: w_sk = 1).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) umma_pack_kernel(const __grid_constant__ UmmaPackLaunch PL) {
    const UmmaPackJob& J = PL.jobs[blockIdx.y];
    const long long total = (long long)J.nblocks * PL.NPAD * 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i % PL.NPAD);
        const int a = (int)((i / PL.NPAD) & 1);
        const int bi = (int)(i / (2LL * PL.NPAD));
        int g = 0, base = 0;
        while (g < J.ngroups - 1 && bi >= base + J.g_nchunk[g] * J.g_nterm[g]) { base += J.g_nchunk[g] * J.g_nterm[g]; ++g; }
        const int rel = bi - base;
        const int chunk = rel / J.g_nterm[g], term = J.g_term_begin[g] + rel % J.g_nterm[g];
        const int k0 = chunk * 16 + a * 8;            // first of this thread's 8 channels within the plane
        const int nn = J.n0 + n;
        float w[8];
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) w[kk] = 0.f;
        if (nn < PL.N) {
            // pair-merged launch: columns [pairC, 2*pairC) are the second class's weights (its own tap of the same row shift)
            const bool h2 = PL.pairC > 0 && nn >= PL.pairC;
            const int wo = h2 ? PL.woff2[term] : PL.woff[term];
            if (wo >= 0 || PL.pairC == 0) {
                const float* src = PL.W + (long long)wo + (long long)k0 * PL.w_sk + (long long)(h2 ? nn - PL.pairC : nn) * PL.w_sn;
#pragma unroll
                for (int kk = 0; kk < 8; ++kk)
                    if (k0 + kk < J.g_C[g]) w[kk] = __ldg(src + (long long)kk * PL.w_sk);
            }
        }
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const __nv_bfloat16 h0 = __float2bfloat16_rn(w[2 * q]), h1 = __float2bfloat16_rn(w[2 * q + 1]);
            hi[q] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
            lo[q] = pack_bf16x2(w[2 * q] - __bfloat162float(h0), w[2 * q + 1] - __bfloat162float(h1));
        }
        uint8_t* blk = J.out + (size_t)bi * 64u * PL.NPAD;
        const size_t off = (size_t)a * 32u * PL.NPAD + (size_t)(n >> 3) * 128u + (size_t)(n & 7) * 16u;
        *reinterpret_cast<uint4*>(blk + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        *reinterpret_cast<uint4*>(blk + 16u * PL.NPAD + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
}

cudaError_t launch_umma_pack(const UmmaPackLaunch& PL, cudaStream_t stream) {
    int maxblk = 0;
    for (int j = 0; j < PL.njobs; ++j) maxblk = max(maxblk, PL.jobs[j].nblocks);
    const long long total = (long long)maxblk * PL.NPAD * 2;
    if (total <= 0 || PL.njobs <= 0) return cudaSuccess;
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 4) blocks = 132 * 4;
    dim3 grid((unsigned)blocks, PL.njobs);
    umma_pack_kernel<<<grid, 256, 0, stream>>>(PL);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// host: turn a generic plane-convolution launch (launch.h ConvLaunch) into a tensor-core launch
// ------------------------------------------------------------------------------------------------
constexpr int kNpadMax = 128;      // accumulator columns per CTA: 64 fp32 registers per thread of each warpgroup
constexpr int kSMs = 132;

// output-channel splits of a launch: enough for NPAD <= kNpadMax, doubled once when the row tiles alone leave SMs idle (each
// CTA then runs cheaper MMAs; the K loop of a tile is the critical path of those latency-bound launches)
static int conv_nsplit(int N, long long tiles128) {
    const int npad_total = (N + 15) / 16 * 16;
    int s = (npad_total + kNpadMax - 1) / kNpadMax;
    if (s * 2 <= kUmmaMaxSplit && tiles128 * s * 2 <= kSMs && (N + s * 2 - 1) / (s * 2) >= 48) s *= 2;
    return s;
}
static int conv_npad(int N, int nsplit) { return ((N + nsplit - 1) / nsplit + 15) / 16 * 16; }

bool umma_plan_from_conv(const ConvLaunch& L, UmmaChoice* ch) {
    memset(ch, 0, sizeof(*ch));
    if (L.N < 16 || L.ncls < 1 || L.ncls > kMaxClasses) return false;
    if (L.pairC > 0) {       // pair-merged classes: both views must satisfy what the vectorised epilogue assumes
        if (L.pairC % 4 != 0 || L.N != 2 * L.pairC) return false;
        for (int q = 0; q < L.ncls; ++q) {
            const OutView& O = L.cls[q];
            if (O.pairC != L.pairC) return false;
            if (O.rstride % 4 || O.bstride % 4 || O.rstride2 % 4 || O.bstride2 % 4) return false;
            if ((reinterpret_cast<uintptr_t>(O.base) & 15) || (reinterpret_cast<uintptr_t>(O.base2) & 15) ||
                (reinterpret_cast<uintptr_t>(O.saved) & 15) || (reinterpret_cast<uintptr_t>(O.saved2) & 15)) return false;
        }
    }
    for (int p = 0; p < L.nplanes; ++p) {
        const PlaneView& P = L.planes[p];
        if (P.C % 8 != 0 || P.C < 8) return false;
        if (P.rstride % 4 != 0 || P.bstride % 4 != 0 || (reinterpret_cast<uintptr_t>(P.base) & 15) != 0) return false;
    }
    if ((L.N + 15) / 16 * 16 > kUmmaMaxSplit * kNpadMax) return false;
    long long tiles128 = 0;
    for (int q = 0; q < L.ncls; ++q) tiles128 += (long long)((L.cls[q].m_hi - L.cls[q].m_lo + 127) / 128) * L.batch;
    ch->nsplit = conv_nsplit(L.N, tiles128);
    ch->NPAD = conv_npad(L.N, ch->nsplit);
    int maxspan = 0, max_rows = 0;
    size_t bytes = 0;
    // packed-weight columns reserved per block: independent of the batch-dependent split above (the arena is sized by a
    // batch-1 dry run), i.e. the widest of the two split counts conv_nsplit can choose
    const int s0 = conv_nsplit(L.N, 1LL << 40);
    const int pack_cols = (s0 * 2 <= kUmmaMaxSplit) ? max(s0 * conv_npad(L.N, s0), 2 * s0 * conv_npad(L.N, 2 * s0)) : s0 * conv_npad(L.N, s0);
    for (int q = 0; q < L.ncls; ++q) {
        const OutView& O = L.cls[q];
        max_rows = max(max_rows, O.m_hi - O.m_lo);
        int ngroups = 0, t = O.term_begin;
        while (t < O.term_end) {
            const int p = L.terms[t].plane;
            int t1 = t, dmin = L.terms[t].d, dmax = dmin;
            while (t1 < O.term_end && L.terms[t1].plane == p) { dmin = min(dmin, L.terms[t1].d); dmax = max(dmax, L.terms[t1].d); ++t1; }
            if (dmax - dmin > 24) return false;
            maxspan = max(maxspan, dmax - dmin);
            bytes += (size_t)((L.planes[p].C + 15) / 16) * (t1 - t) * 64u * pack_cols;
            ++ngroups; t = t1;
        }
        if (ngroups > kUmmaMaxGroups) return false;
    }
    if (max_rows <= 0) return false;
    ch->pack_bytes = (bytes + 255) / 256 * 256;
    ch->MT = 1;
    ch->rows_alloc = 128 + (maxspan + 7) / 8 * 8;
    // weight ring: stages of TB taps (~16 KB) and ~64 KB in all, so that two CTAs share an SM (one hides the other's epilogue
    // and slab conversion)
    const int blk = 64 * ch->NPAD;
    ch->TB = conv_stage_taps(ch->NPAD);
    ch->nbs = min(kBStagesMax, max(2, 65536 / (ch->TB * blk)));
    return true;
}

cudaError_t umma_run_conv(const ConvLaunch& L, const UmmaChoice& ch, uint8_t* arena, cudaStream_t stream) {
    UmmaLaunch U;
    UmmaPackLaunch PL;
    cudaError_t e = umma_build(L, ch, arena, &U, &PL);
    if (e != cudaSuccess) return e;
    e = launch_umma_pack(PL, stream);
    if (e != cudaSuccess) return e;
    return launch_plane_conv_umma(U, stream);
}

cudaError_t umma_build(const ConvLaunch& L, const UmmaChoice& ch, uint8_t* arena, UmmaLaunch* Up, UmmaPackLaunch* PLp) {
    UmmaLaunch& U = *Up;
    UmmaPackLaunch& PL = *PLp;
    memset(&U, 0, sizeof(U));
    memset(&PL, 0, sizeof(PL));
    for (int p = 0; p < L.nplanes; ++p) U.planes[p] = L.planes[p];
    U.ncls = L.ncls; U.N = L.N; U.NPAD = ch.NPAD; U.nsplit = ch.nsplit; U.MT = ch.MT; U.rows_alloc = ch.rows_alloc;
    U.TB = ch.TB; U.nbs = ch.nbs; U.bias = L.bias; U.epilogue = L.epilogue; U.batch = L.batch;
    PL.W = L.W; PL.w_sk = L.w_sk; PL.w_sn = L.w_sn; PL.N = L.N; PL.NPAD = ch.NPAD;
    int nterm_total = 0;
    for (int q = 0; q < L.ncls; ++q) nterm_total = max(nterm_total, L.cls[q].term_end);
    for (int t = 0; t < nterm_total; ++t) { U.d[t] = L.terms[t].d; PL.woff[t] = L.terms[t].woff; PL.woff2[t] = L.terms[t].woff2; }
    PL.pairC = L.pairC; U.pairC = L.pairC;
    uint8_t* cur = arena;
    for (int q = 0; q < L.ncls; ++q) {
        UmmaClass& K = U.cls[q];
        K.out = L.cls[q];
        K.ngroups = 0;
        int t = K.out.term_begin;
        int nblocks = 0;
        UmmaPackJob J0;
        memset(&J0, 0, sizeof(J0));
        while (t < K.out.term_end) {
            const int p = L.terms[t].plane;
            UmmaGroup G;
            G.plane = p; G.term_begin = t; G.dmin = L.terms[t].d;
            int t1 = t;
            while (t1 < K.out.term_end && L.terms[t1].plane == p) { G.dmin = min(G.dmin, L.terms[t1].d); ++t1; }
            G.term_end = t1;
            const int g = K.ngroups++;
            K.groups[g] = G;
            J0.g_nchunk[g] = (L.planes[p].C + 15) / 16; J0.g_nterm[g] = t1 - t; J0.g_term_begin[g] = t; J0.g_C[g] = L.planes[p].C;
            nblocks += J0.g_nchunk[g] * J0.g_nterm[g];
            t = t1;
        }
        J0.ngroups = K.ngroups; J0.nblocks = nblocks;
        for (int sp = 0; sp < ch.nsplit; ++sp) {
            UmmaPackJob J = J0;
            J.n0 = sp * ch.NPAD; J.out = cur;
            K.wpack[sp] = cur;
            cur += (size_t)nblocks * 64u * ch.NPAD;
            if (PL.njobs >= kUmmaMaxPackJobs) return cudaErrorInvalidValue;
            PL.jobs[PL.njobs++] = J;
        }
    }
    return cudaSuccess;
}

}  // namespace wun
