// kernels.h - host-callable launchers of every kernel of the engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "launch.h"


namespace wun {

// Sets the message wun_last_error() returns and returns `code` (engine.cu).
int set_last_error(int code, const char* msg);

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

__host__ __device__ __forceinline__ uint64_t feed_mix64(uint64_t z) {       // splitmix64 finaliser
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// kernels_feed.cu: one training batch cut out of a device-resident track pool (random snippet, random_amplify, centre crop)
cudaError_t launch_feed_batch(const float* pool, long long total_frames, const long long* track_offset,
                              const long long* track_length, int n_tracks, int batch, int K, int C, int T_in, int T_out,
                              int augmentation, unsigned long long seed, long long* step_state, float* mix_out,
                              float* targets_out, long long* chosen, cudaStream_t stream);

// kernels_eval.cu: Test.test's per-batch loss and running mean - curr = sum_k mean(d_k) / K with d = (target - output)^2, or
// |target - output| with l1 - over slots of K * WUN_EVAL_LOSS_CTAS doubles (include/wun.h wun_eval_batch_loss)
void launch_eval_loss(const float* outputs, const float* targets, int K, long long n, double* state, double* batch_loss,
                      double* slots, bool l1, cudaStream_t stream);

// kernels_spec.cu: the spectrogram U-Net's inference graph (frame 1024, hop 768, 513 bins)
struct SpecStft {
    const float* signal;     // [signals][T]
    long long T;
    int n_frames;            // 1 + (T - 1024) / 768
    float* spec;             // [signals][n_frames][513] complex (float2), or null
    float* logmag;           // [signals][n_frames][512]: log1p(|X|) without the last bin, or null
    float* mag;              // [signals][n_frames][513]: |X|, or null
};
void launch_spec_stft(const SpecStft& P, int signals, cudaStream_t stream);

// A 5x5 stride-2 layer over NHWC tensors whose channels sit at a pitch: x[b][h][w][x_pitch] (channels [0, Ci)),
// y[b][h][w][y_pitch] (channels [y_off, y_off + Co)).  W is [5][5][Ci][Co] for the down conv, [5][5][Co][Ci] transposed.
struct SpecConv {
    const float* x; int Hi, Wi, Ci, x_pitch;
    float* y; int Ho, Wo, Co, y_pitch, y_off;
    const float* W; const float* bias;
    const float* beta; const float* mean; const float* var;      // inference batch norm (unused by the mask)
    int batch;
};
void launch_spec_down(const SpecConv& A, cudaStream_t stream);      // + bias, batch norm, LeakyReLU(0.2)
void launch_spec_up(const SpecConv& A, cudaStream_t stream);        // transposed + bias, batch norm, ReLU
// transposed to 1 channel + sigmoid, bin 512 = 0.5; out = mask * X (complex [B][n][513]) or mask * |X| with magnitude
void launch_spec_mask(const SpecConv& A, const float* X, float* out, int magnitude, cudaStream_t stream);
// irfft + inverse window per frame into frames [batch][n_frames][1024], then overlap-add into out [batch][T]
void launch_spec_istft(const float* Y, int n_frames, int batch, float* frames, float* out, long long T, cudaStream_t stream);

// kernels_spec_train.cu: the spectrogram U-Net's training step
// tf.layers.dropout(rate=0.5) keep bit of element i (flat NHWC index of the concatenation) of `level` in the U-Net of
// `source` at dropout step `step`; oracle/spectrogram_train_oracle.py restates it in numpy
__host__ __device__ __forceinline__ bool spec_dropout_keep(uint64_t seed, uint64_t step, int source, int level, uint64_t i) {
    const uint64_t key = (step << 16) ^ ((uint64_t)source << 8) ^ (uint64_t)level;
    const uint64_t stream = feed_mix64(seed ^ feed_mix64(key + 0x9E3779B97F4A7C15ull));
    return (feed_mix64(stream + i * 0x9E3779B97F4A7C15ull) >> 63) != 0;
}

// A 5x5 gather over NHWC tensors at channel pitches, in the stride-2 (output o reads input 2o + k - 1) or transposed
// (output o gathers input (o + 1 - k) / 2, o < 2 Hi) geometry.  Weight of (tap, output channel co, input channel ci) at
// W[tap * w_tap + co * w_co + ci * w_ci].  x_drop / y_drop: keep masks laid out like x / y (kept elements count twice).
struct SpecTrainConv {
    const float* x; int Hi, Wi, Ci, x_pitch; const uint8_t* x_drop;
    float* y; int Ho, Wo, Co, y_pitch, y_off; const uint8_t* y_drop; int accumulate;
    const float* W; long long w_tap, w_co, w_ci;
    const float* bias;                                            // or null
    int batch;
};
void launch_spec_train_conv(const SpecTrainConv& A, int up, cudaStream_t stream);

// Per-channel sums over the N rows of z [N][C] in fp64, in a fixed order, then per channel:
//   mode 0  batch mean and rstd = 1/sqrt(biased var + 1e-3) into stat; moving_mean / moving_var updated with decay 0.999
//   mode 1  dy = g * (a > 0 ? 1 : neg_slope) (g, a at `pitch`): out = sum dy (beta's gradient), coef = (mean dy, mean dy*xhat)
//   mode 2  out = sum z (a conv bias gradient)
struct SpecChanSum {
    int mode;
    const float* z; long long N; int C;
    const float* g; const float* a; int pitch; float neg_slope;
    float2* stat; float2* coef; float* out;
    float* moving_mean; float* moving_var;
    double2* part;                                                // [spec_chan_partials(N)][C]
    double2* local;                                               // modes 0, 1: this call's [C] (sum 1, sum 2)
    const double2* gathered;                                      // modes 0, 1: [world][C], every rank's local
    double n;                                                     // modes 0, 1: rows over all ranks
};
int spec_chan_partials(long long N);
// sums over this call's N rows: mode 2 writes out, modes 0 and 1 write local
void launch_spec_chan_sum(const SpecChanSum& S, cudaStream_t stream);
// modes 0 and 1, after the ranks' local sums are gathered
void launch_spec_chan_finish(const SpecChanSum& S, int world, cudaStream_t stream);
// (z - mean) * rstd + beta, then max(neg_slope * v, v), into y [N][y_pitch]
void launch_spec_bn_apply(const float* z, long long N, int C, const float2* stat, const float* beta, float neg_slope,
                          float* y, int y_pitch, cudaStream_t stream);
// in place: z [N][C] -> dz = rstd * (dy - coef.x - xhat * coef.y)
void launch_spec_bn_backward(float* z, long long N, int C, const float* g, const float* a, int pitch, float neg_slope,
                             const float2* stat, const float2* coef, cudaStream_t stream);
// keep[i] is the keep bit of element first + i
void launch_spec_dropout(uint8_t* keep, long long n, long long first, unsigned long long seed, const long long* step_state,
                         int source, int level, cudaStream_t stream);
// mask [frames][512]: logits in, sigmoid out; out = mask * X (complex [frames][513]) or mask * |X| with magnitude
void launch_spec_mask_apply(float* mask, long long frames, const float* X, float* out, int magnitude, cudaStream_t stream);
struct SpecMaskBwd {
    const float* X; const float* mask; float* dlogit;             // [B][n][513] complex, [B][n][512], [B][n][512]
    int n_frames; long long T;
    int raw_audio;
    const float* audio; const float* target;                      // U7: [B][T]
    const float* tmag;                                            // U7a: [B][n][513]
    float scale;                                                  // 1 / (B T K) or 1 / (B n 513 K)
};
void launch_spec_mask_backward(const SpecMaskBwd& M, int batch, cudaStream_t stream);
// dW[tap * w_tap + c_lo * w_lo + c_hi * w_hi] = sum over low-resolution positions p = (b, h, w) of
// lo[p][c_lo] * hi[b][2h + kh - 1][2w + kw - 1][c_hi]
struct SpecWgrad {
    const float* lo; int lo_pitch; const uint8_t* lo_drop; int Clo;
    const float* hi; int hi_pitch; int Chi;
    int Hl, Wl, batch;
    float* dW; long long w_tap, w_lo, w_hi;
    float* part;                                                  // [spec_wgrad_partials][25 Clo Chi] when that is > 1
};
int spec_wgrad_partials(const SpecWgrad& G);
void launch_spec_wgrad(const SpecWgrad& G, cudaStream_t stream);
void launch_spec_step_advance(long long* step_state, cudaStream_t stream);

}  // namespace wun
