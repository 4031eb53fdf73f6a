// kernels.h - host-callable launchers of every kernel of the engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "launch.h"


namespace wun {

// Output layer (OutputLayer.py:5-23) + loss (Training.py:50-63) parameter block.
struct OutputLaunch {
    const float* params;     // flat parameter buffer
    long long w_off[8];      // per output conv: kernel [ofs][C+F][C] offset
    long long b_off[8];
    const float* mix;        // [B, T_in, C]
    const float* feat;       // [B, Tf, F]  output of the last up block
    const float* targets;    // [K][B, T_out, C] or null
    float* outputs;          // [K][B, T_out, C] or null
    float* dpre;             // [B, T_out, nconv*C] (written when targets != null)
    float* loss;             // device scalar accumulator (pre-zeroed) or null
    float* loss_part;        // with loss: per-CTA loss sums (output_loss_partial_bytes); the last CTA adds them into *loss in a fixed order
    unsigned* loss_count;    // with loss: CTAs done; 0 before the launch, 0 again after it
    int batch, T_in, Tf, T_out, C, F;
    int nconv, K;            // number of output convs, number of sources
    int ofs, pad_left;
    int crop_feat;           // mix row of feature row 0        (Utils.crop, UnetAudioSeparator.py:127)
    int crop_out;            // mix row of output frame 0       (OutputLayer.py:20)
    int output_type;         // 0 direct, 1 difference
    int activation;          // 0 tanh, 1 linear(+clip at test time)
    int training;
    float inv_count;         // 1 / (B*T_out*C*K)
};

struct UpsampleBwdLaunch {
    const float* due;        // [B, N, C]   gradient wrt the even (copied) rows
    const float* dmid;       // [B, nmid, C] gradient wrt the interpolated rows
    const float* x;          // [B, N, C]   saved forward input of the upsampler (producer's output)
    float* gx;               // [B, N, C]   out: gradient wrt the producer's PRE-activation
    const float* blend;      // sigmoid(var) [C] or null (linear: 0.5)
    float* dvar;             // gradient of the interp variable [C] or null
    float* part;             // with dvar: per-CTA sums (upsample_dvar_partial_bytes); the last CTA adds them into dvar in a fixed order
    unsigned* count;         // with dvar: CTAs done; 0 before the launch, 0 again after it
    int batch, N, nmid, C;
    int mid_mode;
    float scale;
    int rows_per_cta;
};

// First down block (kernels_first.cu).  Class 0: full-rate rows a = 2m, m in [0, Td) -> dec[b][m][n];
// class 1: rows a = 2m+1, m in [mo_lo, mo_hi) -> odd[b][m - mo_lo][n].  x row of (row a, tap j) = a + j - pad_left.
struct FirstLayer {
    const float* x; long long x_bstride; int T;     // x[b][t][c], c < C
    int k, pad_left;                                // taps; 0 for valid (context) convs, (k-1)/2 for same
    float* dec; long long dec_bstride; int Td;
    float* odd; long long odd_bstride; int mo_lo, mo_hi;
    const float* W;                                 // [k][C][N]
    const float* bias;                              // [N]
    int batch;
};

struct FirstWgrad {
    FirstLayer L;                 // x, geometry; dec / odd here are the GRADIENT tensors g_dec / g_odd (read only)
    float* dW;                    // [k][C][N]
    float* db;                    // [N] or null
    float scale;
    int rows_per_cta;             // class rows one CTA reduces (multiple of 128; set by the launcher)
    int grid_x;                   // row blocks per (item, class) (set by the launcher)
    float* part;                  // per-CTA sums [class][item][row block][k*C*N + N], added up in a fixed order by a second kernel
};

void launch_plane_conv_simt(const ConvLaunch& L, cudaStream_t stream);
bool first_layer_supported(int C, int N, int k);
void launch_first_fwd(const FirstLayer& L, int C, int N, cudaStream_t stream);
void launch_first_wgrad(FirstWgrad P, int C, int N, cudaStream_t stream);
// bytes of FirstWgrad::part at `batch` (any supported C, N, k)
size_t first_wgrad_partial_bytes(int batch);
void launch_plane_wgrad_simt(WgradLaunch L, cudaStream_t stream);
void launch_colsum(const PlaneView& V, int batch, float scale, float* out, cudaStream_t stream);
// with targets and loss: the last CTA adds the per-CTA sums at L.loss_part into *loss in a fixed order (L.loss_count == 0)
void launch_output_fwd(const OutputLaunch& L, cudaStream_t stream);
size_t output_loss_partial_bytes(int batch, int T_out);
void launch_output_dgrad(const OutputLaunch& L, float* gfeat, cudaStream_t stream);
// part: the per-CTA sums (output_wgrad_partial_bytes), added into grads in a fixed order by a second kernel
void launch_output_wgrad(const OutputLaunch& L, float* grads, float* part, float scale, cudaStream_t stream);
size_t output_wgrad_partial_bytes(const OutputLaunch& L);
// with dvar: the last CTA adds the per-CTA sums at L.part into dvar in a fixed order (L.count == 0)
void launch_upsample_bwd(UpsampleBwdLaunch L, cudaStream_t stream);
// bytes of UpsampleBwdLaunch::part for C channels at `batch` (any N)
size_t upsample_dvar_partial_bytes(int batch, int C);
void launch_sigmoid(const float* x, float* y, int n, cudaStream_t stream);
void launch_adam(float* p, const float* g, float* m, float* v, long long n, float lr_t, float b1, float b2,
                 float eps, float* state, cudaStream_t stream);
void launch_gather_windows(const float* padded, long long n_padded, const long long* starts, int n_windows,
                           int T_in, int C, float* out, cudaStream_t stream);
void launch_scatter_windows(const float* outs, const long long* starts, int n_windows, int n_sources, int T_out,
                            int C, float* preds, long long n_frames, cudaStream_t stream);

// kernels_feed.cu: one training batch cut out of a device-resident track pool (random snippet, random_amplify, centre crop)
cudaError_t launch_feed_batch(const float* pool, long long total_frames, const long long* track_offset,
                              const long long* track_length, int n_tracks, int batch, int K, int C, int T_in, int T_out,
                              int augmentation, unsigned long long seed, long long* step_state, float* mix_out,
                              float* targets_out, long long* chosen, cudaStream_t stream);

}  // namespace wun
