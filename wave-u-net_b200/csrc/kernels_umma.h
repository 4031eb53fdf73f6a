// kernels_umma.h - parameter blocks and launchers of the tensor-core (wgmma) plane-convolution and wgrad kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "launch.h"

namespace wun {

constexpr int kUmmaMaxGroups = 4;
constexpr int kUmmaMaxSplit = 4;

struct UmmaGroup {          // all terms of one class that read the same plane (consecutive row shifts)
    int plane;
    int term_begin, term_end;   // indices into UmmaLaunch::d
    int dmin;
};

struct UmmaClass {
    OutView out;
    UmmaGroup groups[kUmmaMaxGroups];
    int ngroups;
    const uint8_t* wpack[kUmmaMaxSplit];   // packed weights of this class, per output-channel split
};

struct UmmaLaunch {
    PlaneView planes[kMaxPlanes];
    UmmaClass cls[kMaxClasses];
    int d[kMaxTerms];       // row shift of every term (grouped per class/plane)
    int ncls;
    int N;                  // real output channels
    int NPAD;               // channels handled per split, multiple of 16, <= 128
    int nsplit;             // output-channel splits (N > 128, or to spread sparse launches over more SMs)
    int MT;                 // 128-row tiles per CTA (1)
    int rows_alloc;         // slab rows  (>= MT*128 + max row-shift span)
    int TB, nbs;            // weight ring: nbs stages of TB taps
    const float* bias;
    int epilogue;
    int batch;
    int pairC;              // > 0: pair-merged classes (launch.h OutView::pairC); the bias repeats with this period
};

#ifndef __CUDACC__
inline int min(int a, int b) { return a < b ? a : b; }      // host compilers lack CUDA's min(int, int)
#endif

// The conv kernel's K-loop walk, here so that host code (the kernel test harness) walks the very same steps.
//
// A (plane, tile) pair whose slab would hold nothing but zero rows - the tile's rows plus the group's tap span lie
// entirely outside the plane's valid rows - contributes nothing: the K loop skips the group and its packed weights.  This
// is what the dgrad of a down block looks like outside the skip window: the gradient of the odd rows (g_odd) is zero there.
__host__ __device__ __forceinline__ bool group_is_empty(const UmmaLaunch& L, const UmmaGroup& G, int m_base) {
    const PlaneView& P = L.planes[G.plane];
    const int lo = m_base + G.dmin;
    return lo + L.rows_alloc <= P.r_lo || lo >= P.r_hi;
}

// One step of a CTA's K loop = one weight-ring stage: taps [t0, t0 + nt) (relative to the group) of 16-channel chunk c of
// group g; blk = index of its first packed weight block (pack order: group, chunk, term).
struct ConvStep {
    int g, c, t0, nt, blk;
};
// Moves s to the next step (from g = -1: to the first one), skipping groups whose slab would be all zeros together with
// their packed blocks.  false = the K loop is done.
__host__ __device__ __forceinline__ bool next_step(const UmmaLaunch& L, const UmmaClass& K, int m_base, ConvStep& s) {
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
__host__ __device__ __forceinline__ bool next_chunk(const UmmaLaunch& L, const UmmaClass& K, int m_base, ConvStep& s) {
    const UmmaGroup& G = K.groups[s.g];
    s.nt = (G.term_end - G.term_begin) - s.t0;      // as if this step ran to the chunk's last tap
    return next_step(L, K, m_base, s);
}

constexpr int kUmmaMaxPackJobs = kMaxClasses * kUmmaMaxSplit;

struct UmmaPackJob {        // one (class, split) weight pack
    uint8_t* out;
    int ngroups;
    int g_nchunk[kUmmaMaxGroups], g_nterm[kUmmaMaxGroups], g_term_begin[kUmmaMaxGroups], g_C[kUmmaMaxGroups];
    int n0;
    int nblocks;
};

struct UmmaPackLaunch {
    const float* W;
    int woff[kMaxTerms];
    int woff2[kMaxTerms];   // pair-merged launches (pairC > 0): weight offset of columns [pairC, 2*pairC); -1 = zeros
    int pairC;
    int w_sk, w_sn;
    int N, NPAD;
    int njobs;
    UmmaPackJob jobs[kUmmaMaxPackJobs];
};

struct UmmaChoice {         // tiling decisions for one ConvLaunch
    int NPAD, nsplit, MT, rows_alloc, TB, nbs;
    size_t pack_bytes;      // arena bytes the packed weights of this launch need
};

// wgrad on tensor cores: for every group (one forward class x one input plane)
//   dW[woff_t + cp*w_sp + cg*w_sg] += scale * sum_{b, m in [m_lo,m_hi)} P[b, m+d_t, cp] * G[b, m, cg]
// A GEMM with the ROWS as the reduction dimension: both operands are MN-major (channels contiguous).
constexpr int kWgMaxGroups = 8;
constexpr int kWgMaxTaps = 8;

struct WgGroup {
    PlaneView P;            // activation side (tap-shifted; may be a MID plane)
    PlaneView G;            // gradient side (pre-activation gradient), rows m
    int m_lo, m_hi;
    int ntaps;
    int d[kWgMaxTaps];
    int woff[kWgMaxTaps];
    // tiling (filled by umma_plan_wgrad)
    int swap;               // 0: A (M side) = P, B (N side) = G;  1: A = G, B = P
    int NT;                 // N-tile width (multiple of 16, <= 128; the same for every group of a launch)
    int n_mtiles, n_ntiles; // tiles of 128 / NT channels (a CTA's M tile: two 64-channel blocks, one per warpgroup)
    int taps_per_cta, n_tapsets;
    int chunks_per_batch;   // 64-row chunks per batch element
    int chunks_per_cta;     // consecutive (batch-folded) chunks one CTA reduces
    int n_ctas_x;           // ceil(batch*chunks_per_batch / chunks_per_cta)
    int z0;                 // first blockIdx.z of this group (one z per tap set)
    int slot0;              // first partial-tile slot of this group (UmmaWgradLaunch::partial)
};

struct UmmaWgradLaunch {
    WgGroup grp[kWgMaxGroups];
    int ngroups;
    int batch;
    float* dW;
    // not null: every CTA stores its scaled 128 x (taps x NT) tile at slot (slot0 + (tapset * tiles + y) * n_ctas_x + x) and
    //   launch_wgrad_reduce adds the slots in a fixed order (a run-to-run reproducible dW); null: CTAs add into dW atomically
    float* partial;
    int w_sp, w_sg;         // element strides of dW along the P-channel / G-channel index
    float scale;
    int grid_x, grid_y, grid_z;
    int nstages;            // shared-memory pipeline stages (2 or 3)
};

// converter-fed wgrad: for layers whose operand views do not fit one split pass (umma_plan_wgrad_split returns 0)
cudaError_t launch_wgrad_umma(const UmmaWgradLaunch& L, cudaStream_t stream);
// ---- bulk-copy-fed wgrad (default) ------------------------------------------------------------------------------------
constexpr int kSplitMaxJobs = 2 * kWgMaxGroups;

struct SplitJob {           // materialise plane rows [row0, row0 + rows) of V as hi/lo bf16 atom planes at `out`
    PlaneView V;
    uint8_t* out;           // [batch][nchunk][4][rows][16 B]
    int nchunk, rows, row0;
    float* colsum;          // class-gradient views: bias gradient [V.C] that receives colsum_scale * column sums (else null)
    float* colsum_part;     // the per-CTA column sums [batch][nchunk][row blocks][16]; launch_wgrad_reduce adds them into colsum
};

struct SplitJobs {
    SplitJob job[kSplitMaxJobs];
    int njobs, batch;
    float colsum_scale;
};

struct WgSplit {            // where the wgrad groups find their operands (filled next to the SplitJobs)
    const uint8_t* P[kWgMaxGroups];
    const uint8_t* G[kWgMaxGroups];
    long long p_pstride[kWgMaxGroups], g_pstride[kWgMaxGroups];   // bytes between the 4 sub-planes of a chunk (= rows * 16)
    int p_nchunk[kWgMaxGroups], g_nchunk[kWgMaxGroups];
    int p_row0[kWgMaxGroups], g_row0[kWgMaxGroups];               // plane row stored at array index 0
};

// Split arena of one layer's wgrad at `batch`: bytes needed (0 = too many distinct views); fills the jobs / operand table
// when `arena` (256-B aligned, that many bytes) is given.
size_t umma_plan_wgrad_split(const UmmaWgradLaunch& U, int batch, uint8_t* arena, WgSplit* S, SplitJobs* J);
cudaError_t launch_split_views(const SplitJobs& J, cudaStream_t stream);
// Bytes of the partial tiles of a bulk-fed wgrad launch (U.partial), at any batch.
size_t umma_wgrad_partial_bytes(const UmmaWgradLaunch& U);
// The fixed-order sums of a layer's weight gradient (U.partial) and bias gradient (the colsum jobs of J) into dW / colsum:
// float atomics would add the CTAs' contributions in a different order on every run.  A dW or bias element receives one sum
// per forward class (<= 2 in every launch the engine plans), and two float additions onto zero commute, so the result is the
// same bits on every run.
cudaError_t launch_wgrad_reduce(const UmmaWgradLaunch& U, const SplitJobs& J, cudaStream_t stream);
cudaError_t launch_wgrad_umma_bulk(const UmmaWgradLaunch& L, const WgSplit& S, cudaStream_t stream);
// Everything a bulk-fed wgrad launch needs before the split pass / wgrad / reduce launches: the split arena at `arena` (256-B
// aligned; umma_plan_wgrad_split(*U, batch, ...) bytes, rounded up to 256, then umma_wgrad_partial_bytes(*U)), U->partial behind
// it, and the bias gradient `db` (scaled by colsum_scale) on the jobs that split one of the layer's class-gradient views
// class_dpre[0..ncls) - `db` null: no fused column sums.  false: a class-gradient view is not among the split jobs.
bool umma_wgrad_bulk_setup(UmmaWgradLaunch* U, int batch, uint8_t* arena, const PlaneView* class_dpre, int ncls, float* db,
                           float colsum_scale, WgSplit* S, SplitJobs* J);
// rows one wgrad CTA can read past the last valid row of a group: G side / P side (chunk rounding + tap span)
constexpr int kWgOverreachG = 64, kWgOverreachP = 64 + 16;

// fills the tiling fields (groups' P, G, taps and the common fields already set); false = not eligible
bool umma_plan_wgrad(UmmaWgradLaunch* L);
// MACs a planned group issues at `batch` (every 64-row chunk, tap, 64-channel M block with a real channel and N tile)
long long umma_wgrad_issued_macs(const WgGroup& G, int batch);

// Output layer fused into the epilogue of the last up block's forward conv: the 1x1 output convs over [crop(mix) || features]
// (OutputLayer.py:8,15), the activation, the difference source (:17-22), the test-time clip, the MSE loss (Training.py:50-63) and
// their gradients.  The wgmma conv kernel keeps its accumulators in registers and has no room for this epilogue, so
// umma_output_fusable() is false and the output layer runs in its own kernels; the block stays the engine's description of it.
constexpr int kOutFuseMaxCols = 8;    // nconv * C the fused epilogue supports (registers); wider heads use the separate kernels
struct OutputFuse {
    OutputLaunch O;
    float* gfeat;           // training: dPre of the last up block (gradient twin of O.feat, same geometry) or null
    float* grads;           // training: flat gradient buffer (O.w_off / O.b_off index it) or null
    float grad_scale;
    int t_step;             // output frame of (class q, row m, half h) = t0[q] + t_step * m + h
    int t0[kMaxClasses];
};
// whether the conv launch `ch` plans for L can carry the output layer described by O
bool umma_output_fusable(const ConvLaunch& L, const UmmaChoice& ch, const OutputLaunch& O);

size_t umma_smem_bytes(const UmmaLaunch& L);
// dynamic shared memory the kernel variant chosen in `ch` is launched with / of a planned wgrad launch (plan audit)
size_t umma_choice_smem_bytes(const UmmaChoice& ch);
size_t umma_wgrad_smem_bytes(const UmmaWgradLaunch& L);
cudaError_t launch_plane_conv_umma(const UmmaLaunch& L, cudaStream_t stream, const OutputFuse* fuse = nullptr);
cudaError_t launch_umma_pack(const UmmaPackLaunch& PL, cudaStream_t stream);
// Decide whether / how a generic plane-convolution launch runs on the tensor cores; false = not eligible (SIMT).
bool umma_plan_from_conv(const ConvLaunch& L, UmmaChoice* choice);
// Pack the weights into `arena` (choice.pack_bytes, 256-B aligned) and enqueue the tensor-core kernel.
cudaError_t umma_run_conv(const ConvLaunch& L, const UmmaChoice& choice, uint8_t* arena, cudaStream_t stream);
// The two parameter blocks umma_run_conv launches (exposed for the probe / per-kernel timing).
cudaError_t umma_build(const ConvLaunch& L, const UmmaChoice& choice, uint8_t* arena, UmmaLaunch* U, UmmaPackLaunch* PL);

}  // namespace wun
