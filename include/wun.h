/*
 * wun.h - C ABI of the Wave-U-Net forward/backward engine for H100 (libwun.so).
 *
 * The reference has no FFI layer; its boundary for this path is the Python duck type
 *     UnetAudioSeparator(model_config).get_padding(shape) / .get_output(mix, training, ...)
 * (the reference's Models/UnetAudioSeparator.py:15-144) plus the loss / Adam lines of
 * its Training.py:50-77.  Each entry point below names the reference lines it replaces.
 * The Python facade in wave-u-net_b200/Models/UnetAudioSeparator.py binds these with ctypes
 * (see INTEGRATION.md).
 *
 * Conventions
 *   - plain C types only; no torch / CUDA types in signatures (cudaStream_t travels as void*).
 *   - every device pointer is CALLER-OWNED (the facade hands in torch CUDA tensors' data_ptr()).
 *   - all tensors float32, channels-last [B, T, C] contiguous, like the reference (:88).
 *   - parameters / gradients / Adam slots are ONE contiguous float32 buffer each, laid out by
 *     wun_param_table() in TF variable-creation order (kernel [k, C_in, C_out], then bias, ...).
 *   - return value: 0 = ok, negative = error; wun_last_error() gives the message (thread-local).
 *     WUN_E_NOTIMPL mirrors the reference's NotImplementedError (:136, :144), WUN_E_SHAPE its
 *     AssertionError (:55, :121, Utils.py:114-117).
 *   - no hidden synchronisation, allocation or host<->device copy inside forward / backward / adam:
 *     everything is enqueued on `stream` - or, in wun_forward_backward, on internal streams of the handle that are forked
 *     from `stream` and joined back into it with events before the call returns (weight-gradient kernels, the split passes
 *     that feed them one layer ahead, the second launch of an up block's dgrad) - so a whole step can be captured in a
 *     CUDA graph.  The workspace pointers are baked into such a graph: keep the workspace alive as long as the graph.
 */
#ifndef WUN_H
#define WUN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WUN_OK           0
#define WUN_E_INVALID   -1   /* bad argument / null pointer */
#define WUN_E_NOTIMPL   -2   /* unknown upsampling / output_type / output_activation  */
#define WUN_E_SHAPE     -3   /* infeasible shape (reference AssertionError)            */
#define WUN_E_CUDA      -4   /* CUDA runtime error (message has the cudaError string)  */
#define WUN_E_NOGPU     -5   /* compute entry point called without a usable CUDA device */

#define WUN_MAX_SOURCES 8

/* model_config keys read by UnetAudioSeparator.__init__ (:20-32) + num_sources (Config.py:49).
 * upsampling: 0 = "linear", 1 = "learned".  output_type: 0 = "direct", 1 = "difference".
 * output_activation: 0 = "tanh", 1 = "linear".  Any other value -> WUN_E_NOTIMPL at create. */
typedef struct WunConfig {
    int32_t num_layers;
    int32_t num_initial_filters;
    int32_t filter_size;
    int32_t merge_filter_size;
    int32_t input_filter_size;
    int32_t output_filter_size;
    int32_t upsampling;
    int32_t output_type;
    int32_t context;          /* 0 = "same" padding, 1 = "valid" (context) */
    int32_t num_channels;     /* 1 if mono_downmix else 2 */
    int32_t num_sources;      /* len(source_names) */
    int32_t output_activation;
} WunConfig;

typedef struct WunParamInfo {
    char     name[64];        /* TF variable name, e.g. "separator/conv1d_3/kernel" */
    int32_t  ndim;
    int32_t  shape[3];        /* kernel: [k, C_in, C_out]; bias: [C_out]; interp: [F] */
    int64_t  offset;          /* element offset into the flat parameter buffer */
    int64_t  numel;
} WunParamInfo;

typedef struct WunHandle WunHandle;

/* --- pure host (usable without a GPU) ------------------------------------------------------- */

/* UnetAudioSeparator.get_padding (:34-83): desired output frames -> (T_in, T_out). */
int wun_get_padding(const WunConfig* cfg, int64_t num_frames, int64_t* t_in, int64_t* t_out);

/* UnetAudioSeparator.__init__ (:15-32) for a fixed window: validates the config, solves all layer
 * shapes for `num_frames` desired output frames and builds the launch plan.  No device work. */
int wun_create(const WunConfig* cfg, int64_t num_frames, WunHandle** out);
/* Same, but for a given INPUT window length (what get_output sees: mix.shape[1]). */
int wun_create_for_input(const WunConfig* cfg, int64_t input_frames, WunHandle** out);
int wun_destroy(WunHandle* h);

int64_t wun_input_frames(const WunHandle* h);     /* T_in  */
int64_t wun_output_frames(const WunHandle* h);    /* T_out */

/* Variables under scope "separator" (:92) in creation order; what Utils.getTrainableVariables
 * ("separator") (Utils.py:5-6) would list. */
int64_t wun_param_count(const WunHandle* h);                 /* number of tensors  */
int64_t wun_param_numel(const WunHandle* h);                 /* total float32 elements */
int wun_param_table(const WunHandle* h, WunParamInfo* out, int64_t capacity);

/* Bytes of scratch the engine needs for batch `batch` (activations kept for backward, gradients of
 * activations, reduction scratch).  `training` = 0 sizes it for forward only. */
int64_t wun_workspace_bytes(const WunHandle* h, int64_t batch, int training);

/* Algorithmic work of one forward pass at batch `batch` (live positions only, 2 FLOP per MAC) and
 * of forward+backward; used by bench.py for the roofline. */
double wun_forward_flops(const WunHandle* h, int64_t batch);
double wun_forward_backward_flops(const WunHandle* h, int64_t batch);

/* Number of kernels one call enqueues (for bench.py's gpu_launches claim). */
int64_t wun_launches_forward(const WunHandle* h);
int64_t wun_launches_forward_backward(const WunHandle* h);

/* --- device entry points ---------------------------------------------------------------------- */

/* get_output (:85-144): mix [B, T_in, C] -> sources, written to `outputs` as
 * [num_sources][B, T_out, C] contiguous in source_names order.  `training` = 0 applies AudioClip
 * (Utils.py:89-92) exactly where the reference does. */
int wun_forward(WunHandle* h, const float* params, const float* mix, int64_t batch, int training,
                float* outputs, void* workspace, int64_t workspace_bytes, void* stream);

/* One training-graph evaluation (Training.py:47-63 + the tf.gradients half of :77):
 * forward, MSE loss  sum_k mean((target_k - est_k)^2) / K  -> *loss (device scalar), and the
 * gradient of that loss wrt every parameter -> `grads` (flat, same layout as params; overwritten).
 * targets: [num_sources][B, T_out, C].  outputs may be NULL.  grad_scale multiplies the gradient
 * (1/world_size for data-parallel averaging; 1.0 otherwise). */
int wun_forward_backward(WunHandle* h, const float* params, const float* mix, const float* targets,
                         int64_t batch, float* outputs, float* loss, float* grads, float grad_scale,
                         void* workspace, int64_t workspace_bytes, void* stream);

/* tf.train.AdamOptimizer(lr).minimize update (Training.py:77), TF formulation:
 *   lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t);  m,v moments;  p -= lr_t * m / (sqrt(v) + eps).
 * `step` = t >= 1.  One fused pass over the flat buffers. */
int wun_adam_step(WunHandle* h, float* params, const float* grads, float* m, float* v, int64_t step,
                  float lr, float beta1, float beta2, float eps, void* stream);
/* The same update with the step-dependent part on the device, as TF keeps it (variables beta1_power / beta2_power):
 * `state` = DEVICE float[3] {beta1_power, beta2_power, step}, initialised by the caller to {beta1, beta2, 0};
 * lr_t = lr * sqrt(1 - state[1]) / (1 - state[0]) is computed inside the kernel and the accumulators advance
 * ({*beta1, *beta2, +1}) after the update.  Nothing step-dependent is a launch argument, so a captured CUDA graph of a
 * whole training step replays correctly (wun_adam_step would freeze lr_t at its capture-time value). */
int wun_adam_step_device(WunHandle* h, float* params, const float* grads, float* m, float* v, float* state,
                         float lr, float beta1, float beta2, float eps, void* stream);

/* Data-parallel overlap (the one collective of the path, SURVEY 8e): the gradient is produced from the END of the flat buffer
 * (output layer) towards offset 0 (first down block).  Declare n buckets by their first flat offset, strictly descending, the
 * last one 0; every later wun_forward_backward records an internal event per bucket as soon as all gradients at offsets >=
 * first_offset[k] are final, and wun_stream_wait_grad_bucket makes `stream` (the caller's communication stream) wait for it -
 * so bucket k's all-reduce runs while the rest of the backward pass still computes.  Works inside CUDA-graph capture (plain
 * event record / wait).  n = 0 removes the buckets. */
int wun_set_grad_buckets(WunHandle* h, int n, const int64_t* first_offset);
int wun_stream_wait_grad_bucket(WunHandle* h, int k, void* stream);

/* Evaluate.predict_track (Evaluate.py:117-143) device side: cut `n_windows` windows
 * [T_in, C] starting at frame positions `starts[i]` (DEVICE array, int64) out of the already padded mixture
 * `padded` [n_padded, C] (device) into `mix_batch` [n_windows, T_in, C]  (gather), and
 * scatter window outputs [num_sources][n_windows, T_out, C] back into `preds`
 * [num_sources][n_frames, C] at `starts[i]` (plain overwrite, later windows win). */
int wun_gather_windows(WunHandle* h, const float* padded, int64_t n_padded, const int64_t* starts,
                       int64_t n_windows, float* mix_batch, void* stream);
int wun_scatter_windows(WunHandle* h, const float* outputs, const int64_t* starts, int64_t n_windows,
                        float* preds, int64_t n_frames, void* stream);

/* Training-batch construction on the device: replaces the tf.data input pipeline of the reference for the training
 * partition (Datasets.py:16-19 take_random_snippets, :196-214 map / shuffle / batch; Utils.py:26-36 random_amplify,
 * :38-42 crop_sample) with ONE kernel over a track pool that is resident in HBM.
 *   pool          [num_sources + 1][total_frames][C] float32 (device): every source in source_names order, then the
 *                 recorded mixture; the tracks are laid end to end along the frame axis
 *   track_offset  [n_tracks] int64 (device): first pool frame of each track;  track_length [n_tracks]: its frames
 *   step_state    int64[1] (device): batch counter; read by the kernel, advanced by one by this call (on the stream), so
 *                 the call can sit inside a captured CUDA graph and still draw a new batch on every replay
 * Per example b: track = hash(seed, step, b, 0) mod n_tracks, start = hash(.., 1) mod (length - T_in) [tf.random_uniform
 * maxval is exclusive]; with `augmentation` every source is scaled by its own gain in [0.7, 1.0) and the mix is the sum of
 * the scaled sources in source order, otherwise the recorded mix is copied; the targets keep the centre T_out frames.
 * Outputs: mix_out [batch, T_in, C], targets_out [num_sources][batch, T_out, C] (the layout wun_forward_backward takes);
 * `chosen` (optional, int64 [batch][2]) receives (track, start) of every example.  Bit-exact against
 * oracle/feeder_oracle.py.  T_in / T_out / C / num_sources are the handle's. */
int wun_feed_batch(WunHandle* h, const float* pool, int64_t total_frames, const int64_t* track_offset,
                   const int64_t* track_length, int64_t n_tracks, int64_t batch, int augmentation, uint64_t seed,
                   int64_t* step_state, float* mix_out, float* targets_out, int64_t* chosen, void* stream);

/* --- separation scoring (no handle) -------------------------------------------------------------
 * BSS Eval v4 as museval 0.2.0 evaluate(references, estimates, win, hop, mode="v4") computes it - the "images"
 * decomposition with 512-tap distortion filters solved once over the whole track and applied frame by frame - in float64.
 * Replaces the museval.eval_mus_track call at the reference's Evaluate.py:71.
 *   references, estimates  DEVICE float32 [nsrc][nsampl][nchan] (estimate k is scored against reference k; pad or truncate
 *                          the estimates to nsampl first)
 *   metrics   DEVICE float64 [4][nsrc][nwin]: SDR, ISR, SIR, SAR per frame, nwin = floor((nsampl - win + hop) / hop) >= 0;
 *             NaN for frames where some reference or estimate is silent, +inf for a zero denominator
 *   filters   optional DEVICE float64: the filters for all sources, C[j][e][k][c][l] (target j, estimate channel e, reference
 *             source k and channel c, tap l < 512), then those for source j alone, Cj[j][e][c][l]; NULL skips the copy
 * 1 <= nsrc <= WUN_MAX_SOURCES, nchan 1 or 2, nsampl, win, hop >= 1, workspace 256-byte aligned and at least
 * wun_bss_eval_workspace_bytes(...) bytes; otherwise WUN_E_INVALID (and wun_bss_eval_workspace_bytes returns WUN_E_INVALID).
 * Enqueued on `stream`; no allocation, no synchronisation.  The same inputs give the same bits on every call.  These two
 * functions do not set wun_last_error(): the return code is the whole report. */
int64_t wun_bss_eval_workspace_bytes(int64_t nsrc, int64_t nchan, int64_t nsampl, int64_t win, int64_t hop);
int wun_bss_eval(const float* references, const float* estimates, int64_t nsrc, int64_t nchan, int64_t nsampl,
                 int64_t win, int64_t hop, double* metrics, double* filters, void* workspace, int64_t workspace_bytes,
                 void* stream);

/* BSS Eval v3 as museval 0.2.0 evaluate(..., mode="v3") computes it: the decomposition of wun_bss_eval with the filters
 * solved again for every frame from that frame's samples alone (G and D of the zero-extended slices), and only for frames
 * that are not silent.  Inputs, metrics, argument checks and return codes as wun_bss_eval.
 *   filters   optional DEVICE float64 [nwin][...]: frame t's C then Cj in wun_bss_eval's layout; NaN for silent frames
 * The workspace holds the frames of one pass: wun_bss_eval_v3_workspace_bytes(..., frames_per_pass) bytes hold
 * frames_per_pass of them (frames_per_pass >= 1; fewer when there are fewer frames).  wun_bss_eval_v3 fits as many frames per
 * pass as workspace_bytes holds, at least one; the results are the same bits whatever that number is. */
int64_t wun_bss_eval_v3_workspace_bytes(int64_t nsrc, int64_t nchan, int64_t nsampl, int64_t win, int64_t hop,
                                        int64_t frames_per_pass);
int wun_bss_eval_v3(const float* references, const float* estimates, int64_t nsrc, int64_t nchan, int64_t nsampl,
                    int64_t win, int64_t hop, double* metrics, double* filters, void* workspace, int64_t workspace_bytes,
                    void* stream);

/* museval 0.2.0 bss_eval(references, estimates, win, hop, compute_permutation, filters_len=512, framewise_filters,
 * bsseval_sources_version) with its three switches as flags (the function behind museval.metrics' bss_eval_sources /
 * bss_eval_images and their _framewise forms).  wun_bss_eval is flags 0, wun_bss_eval_v3 WUN_BSS_FRAMEWISE_FILTERS: the
 * same bits and workspace sizes.
 *   WUN_BSS_FRAMEWISE_FILTERS  the filters solved for every frame (v3); frames_per_pass as in wun_bss_eval_v3 (ignored
 *                              without this flag)
 *   WUN_BSS_PERMUTATION        every (reference jtrue, estimate jest) pair is scored; per frame the candidate of
 *                              itertools.permutations(range(nsrc)) with the largest mean pair SIR is kept (the first on a
 *                              tie, the identity for a silent frame)
 *   WUN_BSS_SOURCES            the "sources" decomposition: SDR = |P_j|^2 / |est - P_j|^2, ISR NaN; SIR and SAR unchanged
 *   metrics       DEVICE float64 [4][nsrc][nwin]; row j is estimate j (scored against reference perm[j][t])
 *   perm          DEVICE int64 [nsrc][nwin], required with WUN_BSS_PERMUTATION (when nwin > 0), NULL without it
 *   pair_metrics  optional DEVICE float64 [4][nsrc (jtrue)][nsrc (jest)][nwin] (WUN_BSS_PERMUTATION only, else NULL)
 *   filters       optional, as in wun_bss_eval / wun_bss_eval_v3; with WUN_BSS_PERMUTATION the Cj part holds every pair,
 *                 Cj[jtrue][jest][e][c][l]
 * An unknown flag bit is WUN_E_INVALID; other checks and return codes as wun_bss_eval. */
#define WUN_BSS_FRAMEWISE_FILTERS 1
#define WUN_BSS_PERMUTATION       2
#define WUN_BSS_SOURCES           4
int64_t wun_bss_eval_ex_workspace_bytes(int64_t nsrc, int64_t nchan, int64_t nsampl, int64_t win, int64_t hop, int flags,
                                        int64_t frames_per_pass);
int wun_bss_eval_ex(const float* references, const float* estimates, int64_t nsrc, int64_t nchan, int64_t nsampl,
                    int64_t win, int64_t hop, int flags, double* metrics, int64_t* perm, double* pair_metrics,
                    double* filters, void* workspace, int64_t workspace_bytes, void* stream);

/* --- resampling (no handle) ----------------------------------------------------------------------
 * librosa 0.6.2 resample(y, sr_in, sr_out) with res_type='kaiser_best', which the reference applies to every track before and
 * after separation (Evaluate.py:64,104, Utils.resample): resampy 0.2's resample_f bit for bit, then fix_length's zero
 * padding.  Frames t < floor(n_in * ratio), ratio = (double)sr_out / sr_in, are resampy's output; the frames from there up to
 * n_out are zero.
 *   x      DEVICE float32 [n_in][nchan]          y  DEVICE float32 [n_out][nchan], n_out = wun_resample_frames(...)
 *   win, delta  DEVICE float64 [nwin]: the half filter table, already multiplied by the ratio when downsampling (as
 *          resampy.resample scales it before calling resample_f), and its forward difference with a trailing zero;
 *   precision   table entries per zero crossing (512 for kaiser_best)
 * nchan 1 or 2, rates > 0, n_out == wun_resample_frames(n_in, sr_in, sr_out) and floor(n_in * ratio) >= 1 (resampy raises
 * ValueError there); otherwise WUN_E_INVALID (and wun_resample_frames returns WUN_E_INVALID for a rate <= 0 or n_in < 0).
 * Enqueued on `stream`; no allocation, no synchronisation.  The same inputs give the same bits on every call.  These two
 * functions do not set wun_last_error(). */
/* librosa.resample(y, sr_in, sr_out) output length: ceil(n_in * ((double)sr_out / sr_in)) */
int64_t wun_resample_frames(int64_t n_in, int64_t sr_in, int64_t sr_out);
int wun_resample(const float* x, int64_t n_in, int64_t nchan, int64_t sr_in, int64_t sr_out, const double* win,
                 const double* delta, int64_t nwin, int64_t precision, float* y, int64_t n_out, void* stream);

/* --- validation / test loss (no handle) -----------------------------------------------------------
 * The data path of the reference's Test.test (Test.py:57-79) over a partition pool laid out as wun_feed_batch's.
 *
 * wun_snippet_batch: one evaluation batch, no augmentation (Datasets.py:21-25 take_all_snippets, :207 crop_sample).
 *   pool         DEVICE float32 [num_sources + 1][total_frames][nchan]: sources in source_names order, then the mix
 *   positions    DEVICE int64 [n_positions]: absolute pool frame of every snippet start, n_positions a multiple of batch
 *   batch_state  DEVICE int64[1]: batch counter; batch i = counter mod (n_positions / batch) reads positions[i * batch ..];
 *                advanced by one by this call (on the stream), so the call can sit inside a captured CUDA graph
 *   mix_out      DEVICE float32 [batch][input_frames][nchan]: the recorded mix
 *   targets_out  DEVICE float32 [num_sources][batch][output_frames][nchan]: the centre output_frames of every source
 *                ((input_frames - output_frames) / 2 frames cut at the front), the layout wun_forward returns
 * Pure data movement: the outputs are copies of pool values, bit for bit.
 *
 * wun_eval_batch_loss: curr = sum_k mean((targets[k] - outputs[k])^2) / num_sources in float64, then the running mean
 * state[0] += (1 / state[1]') * (curr - state[0]) with state[1]' = state[1] + 1 (Test.py:76).
 *   outputs, targets  DEVICE float32 [num_sources][n]      state  DEVICE float64[2] {total, n}, {0, 0} before a partition
 *   batch_loss        optional DEVICE float64[1] receiving curr
 *   workspace         DEVICE, 8-byte aligned, >= num_sources * WUN_EVAL_LOSS_CTAS * 8 bytes (per-CTA partial sums)
 * The grid and every reduction order are fixed, so the same inputs give the same bits on every call and on every GPU.
 * Both functions: WUN_E_INVALID on a bad argument; enqueued on `stream`; no allocation, no synchronisation; they do not set
 * wun_last_error(). */
#define WUN_EVAL_LOSS_CTAS 264
int wun_snippet_batch(const float* pool, int64_t total_frames, int64_t num_sources, int64_t nchan, int64_t input_frames,
                      int64_t output_frames, const int64_t* positions, int64_t n_positions, int64_t batch,
                      int64_t* batch_state, float* mix_out, float* targets_out, void* stream);
int wun_eval_batch_loss(const float* outputs, const float* targets, int64_t num_sources, int64_t n, double* state,
                        double* batch_loss, void* workspace, int64_t workspace_bytes, void* stream);

/* --- spectrogram U-Net, inference ------------------------------------------------------------------
 * The Jansson et al. baselines of the reference's Models/UnetSpectrogramSeparator.py (presets unet_spectrogram / U7 and
 * unet_spectrogram_l1 / U7a), the graph get_output(mix, training=False, return_spectrogram) builds:
 *   STFT (frame 1024, hop 768, fft 1024, periodic Hann, no end padding): n = 1 + (T - 1024) / 768 frames of 513 bins;
 *   per source, in source_names order, one U-Net on log1p(|X|) without the last bin, NHWC [B, n, 512, 1]:
 *     L down layers: conv2d 5x5 stride 2 'same' (F * 2^i filters) + batch norm + LeakyReLU(0.2);
 *     L - 1 up layers: conv2d_transpose 5x5 stride 2 'same' (F * 2^(L-i-2) filters) + batch norm + ReLU, then
 *       concat([skip, up]) on channels;
 *     mask: conv2d_transpose to 1 channel + sigmoid, bin 512 = 0.5;
 *   magnitude output mask * |X| [K][B, n, 513], or audio output inverse_stft(mask * X) with
 *   inverse_stft_window_fn(768, hann): [K][B, T, 1].
 * Batch norm is the inference form (x - moving_mean) / sqrt(moving_variance + 1e-3) + beta (center, no scale).
 * Parameters: one flat float32 buffer in TF creation order under "separator" - per source and layer conv2d_<i>/kernel
 * [5, 5, C_in, C_out] (conv2d_transpose_<i>/kernel: [5, 5, C_out, C_in]), its bias, then BatchNorm_<j>/beta,
 * moving_mean, moving_variance; the suffixes continue across the two U-Nets as TF's name uniquification does.
 * Every reduction has a fixed order: a window's estimate has the same bits whatever batch holds it.  No allocation,
 * synchronisation or copy inside wun_spec_forward / wun_spec_l1_batch_loss: both can be captured in a CUDA graph.
 * Errors: WUN_E_SHAPE (the reference's AssertionError) for a stereo model, num_sources != 2, (T - 1024) % 768 != 0, or an
 * n or a bin count (512) not divisible by 2^num_layers; WUN_E_INVALID for other bad arguments. */
typedef struct WunSpecConfig {
    int32_t num_layers;
    int32_t num_initial_filters;
    int32_t num_channels;     /* must be 1 (mono_downmix) */
    int32_t num_sources;      /* must be 2 */
} WunSpecConfig;

typedef struct WunSpecParamInfo {
    char     name[64];        /* e.g. "separator/conv2d_6/kernel", "separator/BatchNorm_11/moving_variance" */
    int32_t  ndim;
    int32_t  shape[4];
    int64_t  offset;          /* element offset into the flat parameter buffer */
    int64_t  numel;
} WunSpecParamInfo;

typedef struct WunSpecHandle WunSpecHandle;

#define WUN_SPEC_BINS 513

/* pure host (usable without a GPU) */
int wun_spec_create(const WunSpecConfig* cfg, int64_t num_frames, WunSpecHandle** out);
int wun_spec_destroy(WunSpecHandle* h);
int64_t wun_spec_input_frames(const WunSpecHandle* h);      /* T (= num_frames) */
int64_t wun_spec_output_frames(const WunSpecHandle* h);     /* T */
int64_t wun_spec_stft_frames(const WunSpecHandle* h);       /* n */
int64_t wun_spec_param_count(const WunSpecHandle* h);
int64_t wun_spec_param_numel(const WunSpecHandle* h);
int wun_spec_param_table(const WunSpecHandle* h, WunSpecParamInfo* out, int64_t capacity);
/* scratch of wun_spec_forward and wun_spec_l1_batch_loss at `batch` (one workspace serves both) */
int64_t wun_spec_workspace_bytes(const WunSpecHandle* h, int64_t batch);
/* 2 FLOP per convolution MAC over all 25 taps (down: output positions, transposed: input positions) */
double wun_spec_forward_flops(const WunSpecHandle* h, int64_t batch);
int64_t wun_spec_launches_forward(const WunSpecHandle* h, int return_spectrogram);

/* get_output(mix, training=False, return_spectrogram): mix [B, T, 1] -> outputs [K][B, T, 1], or with return_spectrogram
 * [K][B, n, 513] magnitudes.  Workspace 256-byte aligned, at least wun_spec_workspace_bytes(h, batch). */
int wun_spec_forward(WunSpecHandle* h, const float* params, const float* mix, int64_t batch, int return_spectrogram,
                     float* outputs, void* workspace, int64_t workspace_bytes, void* stream);
/* Test.test's U7a loss (Test.py:57-71): curr = sum_k mean|STFTmag(targets[k]) - est_mags[k]| / K over [B, n, 513] in float64,
 * then the running mean of wun_eval_batch_loss on state = {total, n}.  est_mags [K][B, n, 513] (wun_spec_forward with
 * return_spectrogram), targets [K][B, T, 1]; batch_loss optional.  Same fixed-order reduction as wun_eval_batch_loss. */
int wun_spec_l1_batch_loss(WunSpecHandle* h, const float* est_mags, const float* targets, int64_t batch, double* state,
                           double* batch_loss, void* workspace, int64_t workspace_bytes, void* stream);
/* wun_gather_windows / wun_scatter_windows for this handle's window (T_in = T_out = T, one channel, K sources) */
int wun_spec_gather_windows(WunSpecHandle* h, const float* padded, int64_t n_padded, const int64_t* starts,
                            int64_t n_windows, float* mix_batch, void* stream);
int wun_spec_scatter_windows(WunSpecHandle* h, const float* outputs, const int64_t* starts, int64_t n_windows,
                             float* preds, int64_t n_frames, void* stream);

/* --- spectrogram U-Net, training ------------------------------------------------------------------
 * One step of the reference's Training.py (:47-77) for network="unet_spectrogram": get_output(mix, training=True,
 * return_spectrogram=not raw_audio_loss), the loss sum_k loss_k / K and its gradients, and the batch-norm UPDATE_OPS.
 *   U7  (raw_audio_loss = 1): loss_k = mean((target_k - audio_k)^2) over [B, T, 1], through the inverse STFT;
 *   U7a (raw_audio_loss = 0): loss_k = mean|STFTmag(target_k) - mask_k |X|| over [B, n, 513].
 * Training differs from inference in two layers:
 *   batch norm: normalised with the batch mean and biased variance over B*H*W per channel; moving_mean and moving_variance
 *     in `params` move by (moving - batch value) * (1 - 0.999), the variance Bessel-corrected (N / max(N - 1, 1));
 *   dropout(rate 0.5) on the concatenations of up steps 0, 1, 2 (levels L-2, L-3, L-4), kept elements times 2.  The keep
 *     bit of element i (flat NHWC index) of level d in the U-Net of source k is a splitmix64 hash of (seed, the dropout
 *     counter *step_state, k, d, i) (oracle/spectrogram_train_oracle.py restates it); the call advances the counter by one.
 * LeakyReLU's slope at 0 is 0.2 and ReLU's is 0, as TF's Maximum / Relu gradients have them.  The two U-Nets run one after
 * the other on one set of activation buffers.
 *   params  DEVICE float32 [param_numel]: read, and the moving statistics updated
 *   mix [B, T, 1], targets [K][B, T, 1]; grads DEVICE float32 [param_numel]: every variable's gradient (0 for the moving
 *   statistics); loss DEVICE float64[1]; step_state DEVICE int64[1].
 * Every sum has a fixed order and there are no atomics: the same inputs give the same bits.  No allocation, host
 * synchronisation or copy inside these calls: feed, forward_backward and Adam can be captured in one CUDA graph. */
int64_t wun_spec_train_workspace_bytes(const WunSpecHandle* h, int64_t batch);
/* forward + input-gradient + weight-gradient convolution FLOPs of one step (the first layer has no input gradient) */
double wun_spec_train_flops(const WunSpecHandle* h, int64_t batch);
int wun_spec_forward_backward(WunSpecHandle* h, float* params, const float* mix, const float* targets, int64_t batch,
                              int raw_audio_loss, uint64_t seed, int64_t* step_state, float* grads, double* loss,
                              void* workspace, int64_t workspace_bytes, void* stream);
/* Data parallel: one rank's shard of a batch of global_batch examples.  The step on every rank is the single-device step on
 * the whole batch, up to the order of floating-point sums:
 *   batch norm: each layer's per-channel fp64 sums of this shard ((z, z^2) forward, (dy, dy * xhat) backward) are gathered
 *     from every rank into gathered [world][C][2] by `gather`, then added in rank order from 0.0 over global_batch * H * W
 *     rows, so every rank computes the same statistics and moving averages without a broadcast.  beta's gradient stays
 *     this shard's sum of dy, as every other gradient does;
 *   the loss gradient is scaled by 1 / global_batch, so the SUM of the ranks' gradients is the whole batch's; the loss
 *     written is this shard's mean;
 *   dropout hashes element i of the shard as element sample_offset * (elements per example) + i of the batch, so a
 *     shard's masks are those of its examples in the single-device step.
 * `gather(ctx, local, gathered, count, stream)` must put every rank's `count` doubles at `local` into gathered[rank *
 * count ...] and only enqueue work on `stream` (so that a step stays capturable in a CUDA graph); it returns 0 on success.
 * `local` is overwritten by later work on `stream`.  `gathered`: DEVICE, at least world * 16 * num_initial_filters *
 * 2^(num_layers - 1) bytes (gathered_bytes).  With world = 1 the gather may be null; then the call is
 * wun_spec_forward_backward bit for bit.  About 2 gathers per batch-norm layer per source per step (4 L - 2 for each of the
 * K = 2 sources), each at most 16 * C bytes per rank. */
typedef int (*WunSpecGatherFn)(void* ctx, const double* local, double* gathered, int64_t count, void* stream);
typedef struct WunSpecShard {
    int32_t rank, world;
    int64_t global_batch, sample_offset;
    double* gathered;
    int64_t gathered_bytes;
    WunSpecGatherFn gather;
    void* ctx;
} WunSpecShard;
int wun_spec_forward_backward_dp(WunSpecHandle* h, float* params, const float* mix, const float* targets, int64_t batch,
                                 int raw_audio_loss, uint64_t seed, int64_t* step_state, float* grads, double* loss,
                                 void* workspace, int64_t workspace_bytes, void* stream, const WunSpecShard* shard);
/* tf.train.AdamOptimizer step on the trainable variables (kernels, biases, betas), as wun_adam_step_device: state = DEVICE
 * float32[3] {beta1_power, beta2_power, step}.  The moving statistics have zero gradients and zero slots, so they keep their
 * bits; only the trainables' slots are checkpointed. */
int wun_spec_adam_step_device(WunSpecHandle* h, float* params, const float* grads, float* m, float* v, float* state,
                              float lr, float beta1, float beta2, float eps, void* stream);
/* Tests: where concatenation level `level` ([B, H, W, C] NHWC: the down layer's LeakyReLU output, then the up layer's ReLU
 * output; the bottom level has only the former) lies in the training workspace at `batch`.  After wun_spec_forward_backward
 * it holds the last source's activations, whose signs are the slopes the backward used. */
int wun_spec_debug_train_level(const WunSpecHandle* h, int64_t batch, int level, int64_t* offset_bytes, int64_t* elems);
/* Tests: where a buffer of the training workspace at `batch` lies; after wun_spec_forward_backward it holds the last
 * source's.  what = 0: the keep mask (uint8 [B, H, W, C] like the level) of dropped level `index`; 1 / 2: the batch
 * statistics (float32 [C][2] mean, rstd) of down / up layer `index`. */
int wun_spec_debug_train_buffer(const WunSpecHandle* h, int64_t batch, int what, int index, int64_t* offset_bytes,
                                int64_t* elems);
/* wun_feed_batch for this handle: T_in = T_out = T, one channel, K sources */
int wun_spec_feed_batch(WunSpecHandle* h, const float* pool, int64_t total_frames, const int64_t* track_offset,
                        const int64_t* track_length, int64_t n_tracks, int64_t batch, int augmentation, uint64_t seed,
                        int64_t* step_state, float* mix_out, float* targets_out, int64_t* chosen, void* stream);

/* --- FLAC decoding (csrc/kernels_flac.cu, DESIGN.md §4.10) -----------------------------------------
 * The reference loads compressed audio through librosa 0.6 / audioread / ffmpeg (Utils.load); these decode FLAC streams on the
 * device.  The host parses the metadata blocks and passes STREAMINFO's bits per sample (4..24), channels (1..8), sample rate
 * and maximum block size (0: unknown); `buf` is the DEVICE copy of the frame area (everything after the metadata), `nbytes`
 * long.  wun.read_flac (wun/flac.py) drives the two calls and chains the frames between them. */
typedef struct {
    int64_t offset;      /* byte offset of the frame in buf */
    int64_t number;      /* the header's frame number (fixed block size) or first sample number (variable block size) */
    int64_t end;         /* offset just past the frame's CRC-16, or a negative status (flac_frame.h: truncated, bad header,
                            bad subframe, bad residual, CRC-16 mismatch) */
    int32_t block_size;
    int32_t variable;    /* the header's blocking-strategy bit */
} WunFlacFrame;
/* Every frame candidate: each byte offset with a sync code, a legal header agreeing with STREAMINFO and a matching CRC-8,
 * parsed to its end.  Candidates go to `frames` (DEVICE, `capacity` records) in no particular order; *count (DEVICE uint64,
 * zeroed by the call) receives how many there are, which may exceed `capacity` (then call again with more room). */
int wun_flac_find_frames(const uint8_t* buf, int64_t nbytes, int32_t bps, int32_t channels, int32_t rate, int32_t max_block,
                         WunFlacFrame* frames, int64_t capacity, uint64_t* count, void* stream);
/* Decode the chained frames: frame j starts at byte offsets[j] and its samples go to rows first_samples[j] .. + block size
 * of `out` (DEVICE int32 [total_samples][channels], samples at full depth, FLAC channel order).  status[j] (DEVICE int32)
 * receives 0, or a negative status when the frame does not decode or does not fit the output; nothing is written outside the
 * frame's own rows. */
int wun_flac_decode_frames(const uint8_t* buf, int64_t nbytes, int32_t bps, int32_t channels, int32_t rate,
                           int32_t max_block, const int64_t* offsets, const int64_t* first_samples, int64_t nframes,
                           int32_t* out, int64_t total_samples, int32_t* status, void* stream);

/* --- FLAC encoding (csrc/kernels_flac_encode.cu, DESIGN.md §4.11) --------------------------------
 * The frames of a FLAC stream inside the streamable subset: fixed blocking at block_size (16..4608; the last frame shorter),
 * LPC order <= 12 at rates <= 48 kHz (<= 32 above), 15-bit coefficients, shifts 0-15, Rice partition order <= 8, rate and
 * sample size codes in every header (depths other than 8, 12, 16, 20 and 24 have no size code and take it from STREAMINFO,
 * which leaves the subset).  Each frame's stereo mode, subframe types, predictors and Rice parameters are chosen by exact bit
 * count.  4..24 bits per sample, 1..8 channels, any rate a frame header can express.  The same input gives the same bytes on
 * every run.  wun.write_flac (wun/flac.py) adds the metadata. */
#define WUN_FLAC_INT32 0       /* samples at full depth, within [-2^(bps-1), 2^(bps-1) - 1] */
#define WUN_FLAC_FLOAT32 1     /* clamp(rint(x * 2^(bps-1)), -2^(bps-1), 2^(bps-1) - 1), ties to even, NaN -> 0 */
/* Bytes of the workspace for n samples of `channels` channels (-1: arguments out of range).  Host only. */
int64_t wun_flac_encode_workspace_bytes(int64_t n, int32_t channels, int32_t block_size);
/* Bytes `out` needs: the sum of the frames' bounds (header, VERBATIM subframes, CRC-16), a multiple of 4.  Host only. */
int64_t wun_flac_encode_capacity(int64_t n, int32_t channels, int32_t bps, int32_t block_size);
/* Encode `samples` (DEVICE [n][channels] interleaved, int32 or float32 by sample_type) into the frame area at `out` (DEVICE,
 * 4-byte aligned, out_capacity bytes; the bytes past the frames are zero).  frame_offsets (DEVICE int64, n_frames + 1):
 * frame j occupies out[frame_offsets[j] .. frame_offsets[j + 1]); the last entry is the frame area's length, or -1 when an
 * int32 sample lies outside the depth (then nothing is written).  workspace: DEVICE, 256-byte aligned. */
int wun_flac_encode_frames(const void* samples, int32_t sample_type, int64_t n, int32_t channels, int32_t bps, int32_t rate,
                           int32_t block_size, void* workspace, int64_t workspace_bytes, uint8_t* out, int64_t out_capacity,
                           int64_t* frame_offsets, void* stream);

/* --- diagnostics -------------------------------------------------------------------------------- */
const char* wun_last_error(void);
const char* wun_version(void);
/* Human-readable plan (layer shapes, live windows, kernel choice per layer) into buf; returns the
 * number of bytes that the full text needs. */
int64_t wun_describe(const WunHandle* h, char* buf, int64_t capacity);
/* Plan audit (host only, no GPU needed): one text line per tensor-core launch of a forward+backward at `batch` with the
 * tiling the planner picks (kernel variant, NPAD, tile height, TMEM columns, ring depth, dynamic shared memory, grid) -
 * tests/test_host.py checks every preset against the hardware limits.  Returns the bytes the full text needs. */
int64_t wun_debug_plan(const WunHandle* h, int64_t batch, char* buf, int64_t capacity);
/* The same dry run, but the FULL description of every plane-convolution launch (planes, classes incl. pair-merged halves, terms)
 * as text, with addresses relative to fake bases (workspace 1 << 40, parameters 1 << 41, mix 1 << 42).  Host-only; the numpy
 * interpreter of tests/test_launch_semantics.py checks the planner's launch algebra with it. */
int64_t wun_debug_launches(const WunHandle* h, int64_t batch, char* buf, int64_t capacity);
/* Where a saved activation / activation-gradient lives inside the caller's workspace (tests: per-layer parity).
 * Names: dec<i>, odd<i> (live even / odd rows of down block i), z (bottleneck), up<i>, and g_<name> twins. */
int wun_debug_tensor(const WunHandle* h, const char* name, int64_t batch, int training, int64_t* offset_floats,
                     int64_t* rows, int32_t* channels);
/* Benchmark hook: (re)pack the weights of conv layer `layer` (0..L-1 down, L bottleneck, L+1..2L up) once and enqueue its
 * FORWARD kernel `iters` times on `stream`, reading the activations a previous wun_forward_backward left in `workspace`.
 * *flops_per_launch receives the layer's algorithmic (live-position) FLOPs at this batch.  bench.py times it with CUDA
 * events for the dominant-kernel roofline. */
int wun_debug_run_conv(WunHandle* h, int layer, int iters, const float* params, const float* mix, int64_t batch,
                       void* workspace, int64_t workspace_bytes, void* stream, double* flops_per_launch);
/* The same for any pass of a conv layer: pass 0 = forward, 1 = dgrad (every launch of the layer's input-gradient step; needs the
 * activation gradients a previous wun_forward_backward left in `workspace`), 2 = wgrad + bias gradient (accumulated into
 * `grads_scratch`, a flat buffer laid out like the parameters).  Each iteration repeats the layer's launches for that pass,
 * weight packs included for pass 1.  *flops_per_launch = the layer's algorithmic FLOPs for that pass at this batch.
 * bench.py uses it for the per-layer / per-family roofline table. */
int wun_debug_run_layer(WunHandle* h, int layer, int pass, int iters, const float* params, const float* mix,
                        float* grads_scratch, int64_t batch, void* workspace, int64_t workspace_bytes, void* stream,
                        double* flops_per_launch);
/* Which kernel family a conv layer uses: "simt" or "umma".  layer: 0..L-1 down, L bottleneck,
 * L+1..2L up.  pass: 0 fwd, 1 dgrad, 2 wgrad. */
const char* wun_layer_kernel(const WunHandle* h, int layer, int pass);


/* --- checkpoint helper (host only, no GPU needed) --------------------------------------------------
 * CRC-32C (Castagnoli) of `n` bytes, continuing from `crc` (0 to start): the checksum TensorFlow's V2 checkpoint
 * format stores (masked) for every index block and tensor.  Used by TFCheckpoint.py, which replaces the
 * tf.train.Saver calls at Training.py:92-98,113 and Evaluate.py:55-57. */
uint32_t wun_crc32c(uint32_t crc, const void* data, uint64_t n);

#ifdef __cplusplus
}
#endif
#endif /* WUN_H */
