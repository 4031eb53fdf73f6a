// spec.cu - C ABI (include/wun.h, "spectrogram U-Net, inference") of the spectrogram U-Net baselines: shapes, the parameter
// table in TF creation order, the workspace map and the launch sequence of get_output(training=False)
// (the reference's Models/UnetSpectrogramSeparator.py) over the kernels of kernels_spec.cu.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/wun.h"
#include "kernels.h"

using namespace wun;

namespace {

constexpr int kFrame = 1024, kHop = 768, kBins = WUN_SPEC_BINS, kFreq = kBins - 1;

struct Layer {
    int Hi, Wi, Ci, Ho, Wo, Co;
    int64_t w, b, beta, mean, var;      // parameter offsets (beta/mean/var: -1 for the mask)
};

struct Net {                            // one source's U-Net
    std::vector<Layer> down, up;
    Layer mask;
};

}  // namespace

struct WunSpecHandle {
    WunSpecConfig cfg;
    int64_t T;
    int n;                              // STFT frames
    std::vector<WunSpecParamInfo> params;
    int64_t numel = 0;
    std::vector<Net> nets;
};

namespace {

int fail(int code, const std::string& m) { return set_last_error(code, m.c_str()); }

int64_t add_param(WunSpecHandle* h, const std::string& name, std::vector<int> shape) {
    WunSpecParamInfo p;
    memset(&p, 0, sizeof(p));
    snprintf(p.name, sizeof(p.name), "%s", name.c_str());
    p.ndim = (int32_t)shape.size();
    p.numel = 1;
    for (size_t i = 0; i < shape.size(); ++i) {
        p.shape[i] = shape[i];
        p.numel *= shape[i];
    }
    p.offset = h->numel;
    h->numel += p.numel;
    h->params.push_back(p);
    return p.offset;
}

std::string suffixed(const char* base, int i) {
    return std::string("separator/") + base + (i == 0 ? std::string() : "_" + std::to_string(i));
}

// The variables of tf.layers.conv2d / conv2d_transpose and tf.contrib.layers.batch_norm(center=True, scale=False), with the
// scope counters (conv2d, conv2d_transpose, BatchNorm) running on across layers and sources.
void build_params(WunSpecHandle* h) {
    const int L = h->cfg.num_layers, F = h->cfg.num_initial_filters;
    int n_conv = 0, n_tconv = 0, n_bn = 0;
    auto bn = [&](Layer& l) {
        const std::string s = suffixed("BatchNorm", n_bn++);
        l.beta = add_param(h, s + "/beta", {l.Co});
        l.mean = add_param(h, s + "/moving_mean", {l.Co});
        l.var = add_param(h, s + "/moving_variance", {l.Co});
    };
    for (int k = 0; k < h->cfg.num_sources; ++k) {
        Net net;
        int H = h->n, W = kFreq, C = 1;
        for (int i = 0; i < L; ++i) {
            Layer l{H, W, C, H / 2, W / 2, F << i, 0, 0, 0, 0, 0};
            const std::string s = suffixed("conv2d", n_conv++);
            l.w = add_param(h, s + "/kernel", {5, 5, l.Ci, l.Co});
            l.b = add_param(h, s + "/bias", {l.Co});
            bn(l);
            net.down.push_back(l);
            H = l.Ho; W = l.Wo; C = l.Co;
        }
        for (int i = 0; i + 1 < L; ++i) {
            Layer l{H, W, C, 2 * H, 2 * W, F << (L - i - 2), 0, 0, 0, 0, 0};
            const std::string s = suffixed("conv2d_transpose", n_tconv++);
            l.w = add_param(h, s + "/kernel", {5, 5, l.Co, l.Ci});
            l.b = add_param(h, s + "/bias", {l.Co});
            bn(l);
            net.up.push_back(l);
            H = l.Ho; W = l.Wo; C = 2 * l.Co;                // concat([skip, up])
        }
        Layer m{H, W, C, 2 * H, 2 * W, 1, 0, 0, -1, -1, -1};
        const std::string s = suffixed("conv2d_transpose", n_tconv++);
        m.w = add_param(h, s + "/kernel", {5, 5, 1, m.Ci});
        m.b = add_param(h, s + "/bias", {1});
        net.mask = m;
        h->nets.push_back(net);
    }
}

int64_t align256(int64_t b) { return (b + 255) / 256 * 256; }

// Workspace map at `batch` (bytes): X (complex spectrum), the network input, one concatenation buffer per level d < L-1
// ([skip(d) | up(d)], 2 * F * 2^d channels) and the bottom layer's output, the masked spectrum, the iSTFT frames, and the
// L1 loss's target magnitudes and per-CTA slots.
struct WsMap {
    int64_t X, logmag, Y, frames, tmag, slots, end;
    std::vector<int64_t> level;
};

WsMap ws_map(const WunSpecHandle* h, int64_t B) {
    WsMap m;
    int64_t o = 0;
    auto take = [&](int64_t bytes) { const int64_t at = o; o += align256(bytes); return at; };
    const int64_t bins = B * h->n * (int64_t)kBins;
    m.X = take(bins * 8);
    m.logmag = take(B * h->n * (int64_t)kFreq * 4);
    const int L = h->cfg.num_layers;
    for (int d = 0; d < L; ++d) {
        const Layer& l = h->nets[0].down[d];
        m.level.push_back(take(B * l.Ho * (int64_t)l.Wo * l.Co * (d + 1 < L ? 2 : 1) * 4));
    }
    m.Y = take(bins * 8);
    m.frames = take(B * h->n * (int64_t)kFrame * 4);
    m.tmag = take(h->cfg.num_sources * bins * 4);
    m.slots = take(h->cfg.num_sources * (int64_t)WUN_EVAL_LOSS_CTAS * 8);
    m.end = o;
    return m;
}

int check_device() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(WUN_E_NOGPU, "no CUDA device: the spectrogram engine has no CPU fallback");
    }
    return WUN_OK;
}

int check_call(const WunSpecHandle* h, int64_t batch, const void* ws, int64_t ws_bytes) {
    if (batch < 1 || batch > 65535) return fail(WUN_E_INVALID, "batch out of range (1..65535)");
    if (!ws) return fail(WUN_E_INVALID, "null workspace");
    if (reinterpret_cast<uintptr_t>(ws) % 256 != 0) return fail(WUN_E_INVALID, "workspace must be 256-byte aligned");
    if (ws_bytes < ws_map(h, batch).end) return fail(WUN_E_INVALID, "workspace too small");
    return check_device();
}

}  // namespace

extern "C" {

int wun_spec_create(const WunSpecConfig* cfg, int64_t num_frames, WunSpecHandle** out) {
    if (!cfg || !out) return fail(WUN_E_INVALID, "null argument");
    *out = nullptr;
    if (cfg->num_channels != 1) return fail(WUN_E_SHAPE, "the spectrogram U-Net works on mono input only (mono_downmix)");
    if (cfg->num_sources != 2) return fail(WUN_E_SHAPE, "the spectrogram U-Net separates exactly 2 sources");
    const int L = cfg->num_layers, F = cfg->num_initial_filters;
    if (L < 1 || F < 1) return fail(WUN_E_INVALID, "num_layers and num_initial_filters must be >= 1");
    if (L > 9) return fail(WUN_E_SHAPE, "the 512 bins must be divisible by 2^num_layers");
    if ((int64_t)F << (L - 1) > 65536) return fail(WUN_E_INVALID, "num_initial_filters * 2^(num_layers-1) must be <= 65536");
    if (num_frames < kFrame || (num_frames - kFrame) % kHop != 0)
        return fail(WUN_E_SHAPE, "num_frames must be 1024 + 768 * m (the inverse STFT would be shorter than the input), got "
                                 + std::to_string(num_frames));
    const int64_t n = 1 + (num_frames - kFrame) / kHop;
    if (n % (1LL << L) != 0 || kFreq % (1 << L) != 0)
        return fail(WUN_E_SHAPE, "the " + std::to_string(n) + " STFT frames and the 512 bins must be divisible by 2^num_layers = "
                                 + std::to_string(1 << L));
    if (n > 65535) return fail(WUN_E_INVALID, "too many STFT frames");
    WunSpecHandle* h = new WunSpecHandle();
    h->cfg = *cfg;
    h->T = num_frames;
    h->n = (int)n;
    build_params(h);
    *out = h;
    return WUN_OK;
}

int wun_spec_destroy(WunSpecHandle* h) {
    delete h;
    return WUN_OK;
}

int64_t wun_spec_input_frames(const WunSpecHandle* h) { return h ? h->T : WUN_E_INVALID; }
int64_t wun_spec_output_frames(const WunSpecHandle* h) { return h ? h->T : WUN_E_INVALID; }
int64_t wun_spec_stft_frames(const WunSpecHandle* h) { return h ? h->n : WUN_E_INVALID; }
int64_t wun_spec_param_count(const WunSpecHandle* h) { return h ? (int64_t)h->params.size() : WUN_E_INVALID; }
int64_t wun_spec_param_numel(const WunSpecHandle* h) { return h ? h->numel : WUN_E_INVALID; }

int wun_spec_param_table(const WunSpecHandle* h, WunSpecParamInfo* out, int64_t capacity) {
    if (!h || !out) return fail(WUN_E_INVALID, "null argument");
    if (capacity < (int64_t)h->params.size()) return fail(WUN_E_INVALID, "param table capacity too small");
    memcpy(out, h->params.data(), h->params.size() * sizeof(WunSpecParamInfo));
    return WUN_OK;
}

int64_t wun_spec_workspace_bytes(const WunSpecHandle* h, int64_t batch) {
    if (!h || batch < 1) return WUN_E_INVALID;
    return ws_map(h, batch).end;
}

double wun_spec_forward_flops(const WunSpecHandle* h, int64_t batch) {
    if (!h) return 0.0;
    double macs = 0.0;
    for (const Net& net : h->nets) {
        for (const Layer& l : net.down) macs += (double)l.Ho * l.Wo * 25.0 * l.Ci * l.Co;
        for (const Layer& l : net.up) macs += (double)l.Hi * l.Wi * 25.0 * l.Ci * l.Co;
        macs += (double)net.mask.Hi * net.mask.Wi * 25.0 * net.mask.Ci * net.mask.Co;
    }
    return 2.0 * macs * (double)batch;
}

int64_t wun_spec_launches_forward(const WunSpecHandle* h, int return_spectrogram) {
    if (!h) return WUN_E_INVALID;
    const int64_t per_net = 2LL * h->cfg.num_layers + (return_spectrogram ? 0 : 2);    // L down, L-1 up, mask, iSTFT + OLA
    return 1 + h->cfg.num_sources * per_net;
}

int wun_spec_forward(WunSpecHandle* h, const float* params, const float* mix, int64_t batch, int return_spectrogram,
                     float* outputs, void* workspace, int64_t workspace_bytes, void* stream) {
    if (!h || !params || !mix || !outputs) return fail(WUN_E_INVALID, "null argument");
    int rc = check_call(h, batch, workspace, workspace_bytes);
    if (rc != WUN_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    const WsMap m = ws_map(h, batch);
    const int B = (int)batch, L = h->cfg.num_layers;
    float* X = reinterpret_cast<float*>(ws + m.X);
    float* logmag = reinterpret_cast<float*>(ws + m.logmag);
    auto level = [&](int d) { return reinterpret_cast<float*>(ws + m.level[d]); };

    SpecStft S{mix, h->T, h->n, X, logmag, nullptr};
    launch_spec_stft(S, B, st);
    const int64_t per_source = return_spectrogram ? (int64_t)B * h->n * kBins : (int64_t)B * h->T;
    for (int k = 0; k < h->cfg.num_sources; ++k) {
        const Net& net = h->nets[k];
        const float* x = logmag;
        int x_pitch = 1;
        for (int d = 0; d < L; ++d) {
            const Layer& l = net.down[d];
            const int y_pitch = d + 1 < L ? 2 * l.Co : l.Co;          // the skip half of level d's concatenation buffer
            SpecConv A{x, l.Hi, l.Wi, l.Ci, x_pitch, level(d), l.Ho, l.Wo, l.Co, y_pitch, 0,
                       params + l.w, params + l.b, params + l.beta, params + l.mean, params + l.var, B};
            launch_spec_down(A, st);
            x = level(d);
            x_pitch = y_pitch;
        }
        for (int i = 0; i + 1 < L; ++i) {
            const Layer& l = net.up[i];
            const int d = L - 2 - i;                                   // concat([enc_outputs[-i-1], current])
            SpecConv A{x, l.Hi, l.Wi, l.Ci, l.Ci, level(d), l.Ho, l.Wo, l.Co, 2 * l.Co, l.Co,
                       params + l.w, params + l.b, params + l.beta, params + l.mean, params + l.var, B};
            launch_spec_up(A, st);
            x = level(d);
        }
        const Layer& l = net.mask;
        SpecConv A{x, l.Hi, l.Wi, l.Ci, l.Ci, nullptr, l.Ho, l.Wo, 1, 1, 0,
                   params + l.w, params + l.b, nullptr, nullptr, nullptr, B};
        float* out = outputs + k * per_source;
        if (return_spectrogram) {
            launch_spec_mask(A, X, out, 1, st);
        } else {
            float* Y = reinterpret_cast<float*>(ws + m.Y);
            launch_spec_mask(A, X, Y, 0, st);
            launch_spec_istft(Y, h->n, B, reinterpret_cast<float*>(ws + m.frames), out, h->T, st);
        }
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(WUN_E_CUDA, std::string("spectrogram forward: ") + cudaGetErrorString(e));
    return WUN_OK;
}

int wun_spec_l1_batch_loss(WunSpecHandle* h, const float* est_mags, const float* targets, int64_t batch, double* state,
                           double* batch_loss, void* workspace, int64_t workspace_bytes, void* stream) {
    if (!h || !est_mags || !targets || !state) return fail(WUN_E_INVALID, "null argument");
    int rc = check_call(h, batch, workspace, workspace_bytes);
    if (rc != WUN_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    const WsMap m = ws_map(h, batch);
    const int K = h->cfg.num_sources;
    float* tmag = reinterpret_cast<float*>(ws + m.tmag);
    SpecStft S{targets, h->T, h->n, nullptr, nullptr, tmag};
    launch_spec_stft(S, K * (int)batch, st);
    launch_eval_loss(est_mags, tmag, K, batch * h->n * (int64_t)kBins, state, batch_loss,
                     reinterpret_cast<double*>(ws + m.slots), true, st);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(WUN_E_CUDA, std::string("spectrogram L1 loss: ") + cudaGetErrorString(e));
    return WUN_OK;
}

int wun_spec_gather_windows(WunSpecHandle* h, const float* padded, int64_t n_padded, const int64_t* starts,
                            int64_t n_windows, float* mix_batch, void* stream) {
    if (!h || !padded || !starts || !mix_batch) return fail(WUN_E_INVALID, "null argument");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    launch_gather_windows(padded, n_padded, (const long long*)starts, (int)n_windows, (int)h->T, 1, mix_batch,
                          (cudaStream_t)stream);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? WUN_OK : fail(WUN_E_CUDA, std::string("gather windows: ") + cudaGetErrorString(e));
}

int wun_spec_scatter_windows(WunSpecHandle* h, const float* outputs, const int64_t* starts, int64_t n_windows, float* preds,
                             int64_t n_frames, void* stream) {
    if (!h || !outputs || !starts || !preds) return fail(WUN_E_INVALID, "null argument");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    launch_scatter_windows(outputs, (const long long*)starts, (int)n_windows, h->cfg.num_sources, (int)h->T, 1, preds,
                           n_frames, (cudaStream_t)stream);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? WUN_OK : fail(WUN_E_CUDA, std::string("scatter windows: ") + cudaGetErrorString(e));
}

}  // extern "C"
