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
