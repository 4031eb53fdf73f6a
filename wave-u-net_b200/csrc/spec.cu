// spec.cu - C ABI (include/wun.h, "spectrogram U-Net, inference" and "training") of the spectrogram U-Net baselines: shapes,
// the parameter table in TF creation order, the workspace maps and the launch sequences of get_output(training=False) (the
// reference's Models/UnetSpectrogramSeparator.py) over the kernels of kernels_spec.cu, and of one training step
// (Training.py:47-77) over those of kernels_spec_train.cu.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
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

// The concatenations tf.layers.dropout(rate=0.5) acts on: up step i < 3 drops concat level d = L - 2 - i.
bool dropped_level(int L, int d) { return d <= L - 2 && d >= L - 4; }

int level_pitch(const Layer& l, int d, int L) { return d + 1 < L ? 2 * l.Co : l.Co; }

// Training workspace at `batch`: the inference map, then per level the gradient twin of its concatenation buffer and the
// keep mask of a dropped level, the pre-batch-norm output of every layer (overwritten by its gradient in the backward),
// the mask (logits, then sigmoid) and its gradient, the K outputs the loss reads, the per-channel statistics and backward
// coefficients, the partial sums of the channel reductions, this call's per-channel sums, the partial sums of the weight
// gradients, and the loss's running-mean state.
struct TrainMap {
    WsMap base;
    std::vector<int64_t> glevel, drop, zdown, zup, sdown, sup;     // s*: per-channel (batch mean, rstd) of every layer
    int64_t mask, dlogit, out, coef, red, local, wpart, loss_state, end;
};

std::vector<SpecWgrad> wgrad_shapes(const WunSpecHandle* h, int B) {
    const Net& net = h->nets[0];
    const int L = h->cfg.num_layers;
    std::vector<SpecWgrad> out;
    for (int d = 0; d < L; ++d) {
        const Layer& l = net.down[d];
        SpecWgrad G{};
        G.Clo = l.Co; G.Chi = l.Ci; G.Hl = l.Ho; G.Wl = l.Wo; G.batch = B;
        out.push_back(G);
    }
    for (const Layer& l : net.up) {
        SpecWgrad G{};
        G.Clo = l.Ci; G.Chi = l.Co; G.Hl = l.Hi; G.Wl = l.Wi; G.batch = B;
        out.push_back(G);
    }
    SpecWgrad G{};
    G.Clo = net.mask.Ci; G.Chi = 1; G.Hl = net.mask.Hi; G.Wl = net.mask.Wi; G.batch = B;
    out.push_back(G);
    return out;
}

TrainMap train_map(const WunSpecHandle* h, int64_t B) {
    TrainMap m;
    m.base = ws_map(h, B);
    int64_t o = m.base.end;
    auto take = [&](int64_t bytes) { const int64_t at = o; o += align256(bytes); return at; };
    const Net& net = h->nets[0];
    const int L = h->cfg.num_layers, K = h->cfg.num_sources;
    int cmax = 1;
    int64_t rows_max = B * h->n * (int64_t)kFreq;
    for (int d = 0; d < L; ++d) {
        const Layer& l = net.down[d];
        const int64_t elems = B * l.Ho * (int64_t)l.Wo * level_pitch(l, d, L);
        m.glevel.push_back(take(elems * 4));
        m.drop.push_back(dropped_level(L, d) ? take(elems) : -1);
        m.zdown.push_back(take(B * l.Ho * (int64_t)l.Wo * l.Co * 4));
        m.sdown.push_back(take(l.Co * 8));
        cmax = std::max(cmax, l.Co);
    }
    for (const Layer& l : net.up) {
        m.zup.push_back(take(B * l.Ho * (int64_t)l.Wo * l.Co * 4));
        m.sup.push_back(take(l.Co * 8));
    }
    const int64_t bins = B * h->n * (int64_t)kBins;
    m.mask = take(rows_max * 4);
    m.dlogit = take(rows_max * 4);
    m.out = take(K * std::max(bins, B * h->T) * 4);
    m.coef = take(cmax * 8);
    m.red = take((int64_t)spec_chan_partials(rows_max) * cmax * 16);
    m.local = take(cmax * 16);
    int64_t wpart = 0;
    for (const SpecWgrad& G : wgrad_shapes(h, (int)B)) {
        const int P = spec_wgrad_partials(G);
        if (P > 1) wpart = std::max(wpart, (int64_t)P * 25 * G.Clo * G.Chi);
    }
    m.wpart = take(wpart * 4);
    m.loss_state = take(16);
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

// The widest batch-norm layer (the bottom one): a rank's gathered statistics take world * 16 bytes per channel of it.
int64_t widest_bn(const WunSpecHandle* h) { return h->nets[0].down.back().Co; }

// One U-Net's training forward and backward (source k), on the activation buffers every source shares.  The batch-norm
// statistics are those of the whole batch of `shard`: each layer's per-channel sums go through the shard's gather.
struct TrainCall {
    const WunSpecHandle* h;
    float* params;
    float* grads;
    char* ws;
    const TrainMap* m;
    int B;
    int raw_audio;
    unsigned long long seed;
    long long* step_state;
    const float* targets;          // [K][B][T]
    cudaStream_t st;
    WunSpecShard shard;

    // every rank's (sum 1, sum 2) of S.local (written by launch_spec_chan_sum) into S.gathered; one rank without a gather
    // reads its own
    int gather(SpecChanSum& S) const {
        if (!shard.gather) {
            S.gathered = S.local;
            return WUN_OK;
        }
        S.gathered = reinterpret_cast<const double2*>(shard.gathered);
        const int rc = shard.gather(shard.ctx, reinterpret_cast<const double*>(S.local), shard.gathered, 2LL * S.C, st);
        return rc == 0 ? WUN_OK : fail(WUN_E_CUDA, "spectrogram training: the batch-statistics gather failed (" +
                                                       std::to_string(rc) + ")");
    }

    template <class T> T* at(int64_t off) const { return reinterpret_cast<T*>(ws + off); }
    float* level(int d) const { return at<float>(m->base.level[d]); }
    float* glevel(int d) const { return at<float>(m->glevel[d]); }
    const uint8_t* drop(int d) const { return m->drop[d] >= 0 ? at<uint8_t>(m->drop[d]) : nullptr; }

    // batch statistics, moving averages, normalise + beta + activation into y
    int bn_forward(const Layer& l, const float* z, float2* stat, float* y, int y_pitch, float neg_slope) const {
        const long long N = (long long)B * l.Ho * l.Wo;
        SpecChanSum S{};
        S.mode = 0; S.z = z; S.N = N; S.C = l.Co;
        S.stat = stat;
        S.moving_mean = params + l.mean; S.moving_var = params + l.var;
        S.part = at<double2>(m->red);
        S.local = at<double2>(m->local);
        S.n = (double)(shard.global_batch * l.Ho * l.Wo);
        launch_spec_chan_sum(S, st);
        if (int rc = gather(S)) return rc;
        launch_spec_chan_finish(S, shard.world, st);
        launch_spec_bn_apply(z, N, l.Co, S.stat, params + l.beta, neg_slope, y, y_pitch, st);
        return WUN_OK;
    }

    // g, a: the layer's output gradient and activation at `pitch`; z (pre-BN output) becomes dz.  Also the gradients of
    // beta and of the conv bias (the fixed-order sum of dz).
    int bn_backward(const Layer& l, float* z, float2* stat, const float* g, const float* a, int pitch,
                    float neg_slope) const {
        const long long N = (long long)B * l.Ho * l.Wo;
        SpecChanSum S{};
        S.mode = 1; S.z = z; S.N = N; S.C = l.Co; S.stat = stat;
        S.part = at<double2>(m->red);
        S.g = g; S.a = a; S.pitch = pitch; S.neg_slope = neg_slope;
        S.coef = at<float2>(m->coef); S.out = grads + l.beta;
        S.local = at<double2>(m->local);
        S.n = (double)(shard.global_batch * l.Ho * l.Wo);
        launch_spec_chan_sum(S, st);
        if (int rc = gather(S)) return rc;
        launch_spec_chan_finish(S, shard.world, st);
        launch_spec_bn_backward(z, N, l.Co, g, a, pitch, neg_slope, S.stat, S.coef, st);
        bias_grad(l, z, N);
        return WUN_OK;
    }

    void bias_grad(const Layer& l, const float* dz, long long N) const {
        SpecChanSum S{};
        S.mode = 2; S.z = dz; S.N = N; S.C = l.Co; S.out = grads + l.b;
        S.part = at<double2>(m->red);
        launch_spec_chan_sum(S, st);
    }

    void wgrad(SpecWgrad G) const {
        G.part = at<float>(m->wpart);
        launch_spec_wgrad(G, st);
    }

    int run(int k) const;
};

int TrainCall::run(int k) const {
    const WunSpecHandle* H = h;
    const Net& net = H->nets[k];
    const int L = H->cfg.num_layers, K = H->cfg.num_sources;
    const float* logmag = at<float>(m->base.logmag);
    const float* X = at<float>(m->base.X);
    auto zd = [&](int d) { return at<float>(m->zdown[d]); };
    auto zu = [&](int i) { return at<float>(m->zup[i]); };
    auto sd = [&](int d) { return at<float2>(m->sdown[d]); };
    auto su = [&](int i) { return at<float2>(m->sup[i]); };
    // input of up step i: the bottom layer's output, or the (dropped) concatenation one level down
    auto up_in = [&](int i, const float** x, int* pitch, const uint8_t** dr, float** gx) {
        const int d = L - 1 - i;
        *x = level(d);
        *gx = glevel(d);
        *pitch = level_pitch(net.down[d], d, L);
        *dr = i == 0 ? nullptr : drop(d);
    };

    // ---- forward ----
    const float* x = logmag;
    int x_pitch = 1;
    for (int d = 0; d < L; ++d) {
        const Layer& l = net.down[d];
        SpecTrainConv A{x, l.Hi, l.Wi, l.Ci, x_pitch, nullptr, zd(d), l.Ho, l.Wo, l.Co, l.Co, 0, nullptr, 0,
                        params + l.w, (long long)l.Ci * l.Co, 1, l.Co, params + l.b, B};
        launch_spec_train_conv(A, 0, st);
        const int y_pitch = level_pitch(l, d, L);
        if (int rc = bn_forward(l, zd(d), sd(d), level(d), y_pitch, 0.2f)) return rc;
        x = level(d);
        x_pitch = y_pitch;
    }
    for (int d = 0; d < L; ++d)
        if (drop(d)) {
            const Layer& l = net.down[d];
            const long long per_sample = (long long)l.Ho * l.Wo * level_pitch(l, d, L);
            launch_spec_dropout(const_cast<uint8_t*>(drop(d)), B * per_sample, shard.sample_offset * per_sample, seed,
                                step_state, k, d, st);
        }
    for (int i = 0; i + 1 < L; ++i) {
        const Layer& l = net.up[i];
        const int d = L - 2 - i;
        const float* ux; int up; const uint8_t* udr; float* ug;
        up_in(i, &ux, &up, &udr, &ug);
        SpecTrainConv A{ux, l.Hi, l.Wi, l.Ci, up, udr, zu(i), l.Ho, l.Wo, l.Co, l.Co, 0, nullptr, 0,
                        params + l.w, (long long)l.Co * l.Ci, l.Ci, 1, params + l.b, B};
        launch_spec_train_conv(A, 1, st);
        if (int rc = bn_forward(l, zu(i), su(i), level(d) + l.Co, 2 * l.Co, 0.f)) return rc;
    }
    const Layer& ml = net.mask;
    const uint8_t* mdrop = L > 1 ? drop(0) : nullptr;
    float* mask = at<float>(m->mask);
    {
        SpecTrainConv A{level(0), ml.Hi, ml.Wi, ml.Ci, ml.Ci, mdrop, mask, ml.Ho, ml.Wo, 1, 1, 0, nullptr, 0,
                        params + ml.w, ml.Ci, ml.Ci, 1, params + ml.b, B};
        launch_spec_train_conv(A, 1, st);
    }
    const int64_t bins = (int64_t)B * H->n * kBins;
    float* out = at<float>(m->out) + k * (raw_audio ? (int64_t)B * H->T : bins);
    if (raw_audio) {
        float* Y = at<float>(m->base.Y);
        launch_spec_mask_apply(mask, (long long)B * H->n, X, Y, 0, st);
        launch_spec_istft(Y, H->n, B, at<float>(m->base.frames), out, H->T, st);
    } else {
        launch_spec_mask_apply(mask, (long long)B * H->n, X, out, 1, st);
    }

    // ---- backward ----
    // d loss / d output of the whole batch's mean: 1 / (global batch x elements per example x K)
    float* dlogit = at<float>(m->dlogit);
    const int64_t GB = shard.global_batch;
    SpecMaskBwd M{X, mask, dlogit, H->n, H->T, raw_audio, out, targets + (int64_t)k * B * H->T,
                  at<float>(m->base.tmag) + k * bins,
                  raw_audio ? (float)(1.0 / ((double)GB * H->T * K)) : (float)(1.0 / ((double)(GB * H->n * kBins) * K))};
    launch_spec_mask_backward(M, B, st);
    {
        SpecChanSum S{};
        S.mode = 2; S.z = dlogit; S.N = (long long)B * ml.Ho * ml.Wo; S.C = 1; S.out = grads + ml.b;
        S.part = at<double2>(m->red);
        launch_spec_chan_sum(S, st);
        SpecWgrad G{level(0), ml.Ci, mdrop, ml.Ci, dlogit, 1, 1, ml.Hi, ml.Wi, B, grads + ml.w, ml.Ci, 1, ml.Ci, nullptr};
        wgrad(G);
        SpecTrainConv D{dlogit, ml.Ho, ml.Wo, 1, 1, nullptr, glevel(0), ml.Hi, ml.Wi, ml.Ci, ml.Ci, 0, mdrop, 0,
                        params + ml.w, ml.Ci, 1, ml.Ci, nullptr, B};
        launch_spec_train_conv(D, 0, st);
    }
    for (int i = L - 2; i >= 0; --i) {
        const Layer& l = net.up[i];
        const int d = L - 2 - i;
        if (int rc = bn_backward(l, zu(i), su(i), glevel(d) + l.Co, level(d) + l.Co, 2 * l.Co, 0.f)) return rc;
        const float* ux; int up; const uint8_t* udr; float* ug;
        up_in(i, &ux, &up, &udr, &ug);
        SpecWgrad G{ux, up, udr, l.Ci, zu(i), l.Co, l.Co, l.Hi, l.Wi, B, grads + l.w, (long long)l.Co * l.Ci, 1, l.Ci,
                    nullptr};
        wgrad(G);
        // into the whole input: both halves of a concatenation, through its dropout mask
        SpecTrainConv D{zu(i), l.Ho, l.Wo, l.Co, l.Co, nullptr, ug, l.Hi, l.Wi, l.Ci, up, 0, udr, 0,
                        params + l.w, (long long)l.Co * l.Ci, 1, l.Ci, nullptr, B};
        launch_spec_train_conv(D, 0, st);
    }
    for (int d = L - 1; d >= 0; --d) {
        const Layer& l = net.down[d];
        const int pitch = level_pitch(l, d, L);
        if (int rc = bn_backward(l, zd(d), sd(d), glevel(d), level(d), pitch, 0.2f)) return rc;
        const float* xin = d == 0 ? logmag : level(d - 1);
        const int xin_pitch = d == 0 ? 1 : level_pitch(net.down[d - 1], d - 1, L);
        SpecWgrad G{zd(d), l.Co, nullptr, l.Co, xin, xin_pitch, l.Ci, l.Ho, l.Wo, B, grads + l.w, (long long)l.Ci * l.Co,
                    1, l.Co, nullptr};
        wgrad(G);
        if (d > 0) {
            // the skip gradient's second part, added to the part the concatenation passed back
            SpecTrainConv D{zd(d), l.Ho, l.Wo, l.Co, l.Co, nullptr, glevel(d - 1), l.Hi, l.Wi, l.Ci, xin_pitch, 0, nullptr,
                            1, params + l.w, (long long)l.Ci * l.Co, l.Co, 1, nullptr, B};
            launch_spec_train_conv(D, 1, st);
        }
    }
    return WUN_OK;
}

int check_train_call(const WunSpecHandle* h, int64_t batch, const void* ws, int64_t ws_bytes) {
    if (batch < 1 || batch > 65535) return fail(WUN_E_INVALID, "batch out of range (1..65535)");
    if (!ws) return fail(WUN_E_INVALID, "null workspace");
    if (reinterpret_cast<uintptr_t>(ws) % 256 != 0) return fail(WUN_E_INVALID, "workspace must be 256-byte aligned");
    if (ws_bytes < train_map(h, batch).end) return fail(WUN_E_INVALID, "workspace too small (wun_spec_train_workspace_bytes)");
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

int64_t wun_spec_train_workspace_bytes(const WunSpecHandle* h, int64_t batch) {
    if (!h || batch < 1) return WUN_E_INVALID;
    return train_map(h, batch).end;
}

double wun_spec_train_flops(const WunSpecHandle* h, int64_t batch) {
    if (!h) return 0.0;
    double first = 0.0;                                      // the first down layer has no input gradient (X is data)
    for (const Net& net : h->nets) {
        const Layer& l = net.down[0];
        first += 2.0 * (double)l.Ho * l.Wo * 25.0 * l.Ci * l.Co * (double)batch;
    }
    return 3.0 * wun_spec_forward_flops(h, batch) - first;
}

}  // extern "C"

namespace {

int forward_backward(WunSpecHandle* h, float* params, const float* mix, const float* targets, int64_t batch,
                     int raw_audio_loss, uint64_t seed, int64_t* step_state, float* grads, double* loss, void* workspace,
                     int64_t workspace_bytes, void* stream, const WunSpecShard& shard) {
    if (!h || !params || !mix || !targets || !step_state || !grads || !loss) return fail(WUN_E_INVALID, "null argument");
    int rc = check_train_call(h, batch, workspace, workspace_bytes);
    if (rc != WUN_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    const TrainMap m = train_map(h, batch);
    const int B = (int)batch, K = h->cfg.num_sources;
    cudaError_t e = cudaMemsetAsync(grads, 0, sizeof(float) * h->numel, st);   // the moving statistics get no gradient
    if (e == cudaSuccess) e = cudaMemsetAsync(ws + m.loss_state, 0, 16, st);
    if (e != cudaSuccess) return fail(WUN_E_CUDA, std::string("spectrogram training: ") + cudaGetErrorString(e));
    SpecStft S{mix, h->T, h->n, reinterpret_cast<float*>(ws + m.base.X), reinterpret_cast<float*>(ws + m.base.logmag),
               nullptr};
    launch_spec_stft(S, B, st);
    if (!raw_audio_loss) {
        SpecStft Tg{targets, h->T, h->n, nullptr, nullptr, reinterpret_cast<float*>(ws + m.base.tmag)};
        launch_spec_stft(Tg, K * B, st);
    }
    TrainCall call{h, params, grads, ws, &m, B, raw_audio_loss ? 1 : 0, (unsigned long long)seed, (long long*)step_state,
                   targets, st, shard};
    for (int k = 0; k < K; ++k) {
        rc = call.run(k);
        if (rc != WUN_OK) return rc;
    }
    const int64_t per = raw_audio_loss ? (int64_t)B * h->T : (int64_t)B * h->n * kBins;
    launch_eval_loss(reinterpret_cast<float*>(ws + m.out), raw_audio_loss ? targets : reinterpret_cast<float*>(ws + m.base.tmag),
                     K, per, reinterpret_cast<double*>(ws + m.loss_state), loss, reinterpret_cast<double*>(ws + m.base.slots),
                     !raw_audio_loss, st);
    launch_spec_step_advance((long long*)step_state, st);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail(WUN_E_CUDA, std::string("spectrogram training: ") + cudaGetErrorString(e));
    return WUN_OK;
}

}  // namespace

extern "C" {

int wun_spec_forward_backward(WunSpecHandle* h, float* params, const float* mix, const float* targets, int64_t batch,
                              int raw_audio_loss, uint64_t seed, int64_t* step_state, float* grads, double* loss,
                              void* workspace, int64_t workspace_bytes, void* stream) {
    WunSpecShard one{};
    one.rank = 0; one.world = 1; one.global_batch = batch; one.sample_offset = 0;
    return forward_backward(h, params, mix, targets, batch, raw_audio_loss, seed, step_state, grads, loss, workspace,
                            workspace_bytes, stream, one);
}

int wun_spec_forward_backward_dp(WunSpecHandle* h, float* params, const float* mix, const float* targets, int64_t batch,
                                 int raw_audio_loss, uint64_t seed, int64_t* step_state, float* grads, double* loss,
                                 void* workspace, int64_t workspace_bytes, void* stream, const WunSpecShard* shard) {
    if (!h || !shard) return fail(WUN_E_INVALID, "null argument");
    const WunSpecShard& s = *shard;
    if (s.world < 1 || s.rank < 0 || s.rank >= s.world) return fail(WUN_E_INVALID, "shard: need 0 <= rank < world");
    if (s.global_batch < batch || s.global_batch > 65535 || s.sample_offset < 0 || s.sample_offset + batch > s.global_batch)
        return fail(WUN_E_INVALID, "shard: need 0 <= sample_offset and sample_offset + batch <= global_batch <= 65535");
    if (s.world > 1 && !s.gather) return fail(WUN_E_INVALID, "shard: more than one rank needs a gather callback");
    if (s.gather && (!s.gathered || s.gathered_bytes < (int64_t)s.world * 16 * widest_bn(h)))
        return fail(WUN_E_INVALID, "shard: the gathered buffer needs world * 16 * num_initial_filters * 2^(num_layers-1) "
                                   "bytes");
    return forward_backward(h, params, mix, targets, batch, raw_audio_loss, seed, step_state, grads, loss, workspace,
                            workspace_bytes, stream, s);
}

int wun_spec_debug_train_level(const WunSpecHandle* h, int64_t batch, int level, int64_t* offset_bytes, int64_t* elems) {
    if (!h || batch < 1 || level < 0 || level >= h->cfg.num_layers || !offset_bytes || !elems)
        return fail(WUN_E_INVALID, "bad argument");
    const Layer& l = h->nets[0].down[level];
    *offset_bytes = train_map(h, batch).base.level[level];
    *elems = batch * l.Ho * (int64_t)l.Wo * level_pitch(l, level, h->cfg.num_layers);
    return WUN_OK;
}

int wun_spec_debug_train_buffer(const WunSpecHandle* h, int64_t batch, int what, int index, int64_t* offset_bytes,
                                int64_t* elems) {
    if (!h || batch < 1 || !offset_bytes || !elems || what < 0 || what > 2) return fail(WUN_E_INVALID, "bad argument");
    const int L = h->cfg.num_layers;
    const TrainMap m = train_map(h, batch);
    const Net& net = h->nets[0];
    if (what == 0) {
        if (index < 0 || index >= L || m.drop[index] < 0) return fail(WUN_E_INVALID, "level has no dropout mask");
        const Layer& l = net.down[index];
        *offset_bytes = m.drop[index];
        *elems = batch * l.Ho * (int64_t)l.Wo * level_pitch(l, index, L);
        return WUN_OK;
    }
    const std::vector<int64_t>& at = what == 1 ? m.sdown : m.sup;
    if (index < 0 || index >= (int)at.size()) return fail(WUN_E_INVALID, "no such layer");
    *offset_bytes = at[index];
    *elems = 2 * (what == 1 ? net.down[index] : net.up[index]).Co;
    return WUN_OK;
}

int wun_spec_adam_step_device(WunSpecHandle* h, float* params, const float* grads, float* m, float* v, float* state,
                              float lr, float beta1, float beta2, float eps, void* stream) {
    if (!h || !params || !grads || !m || !v || !state) return fail(WUN_E_INVALID, "null argument");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    // One pass over the flat buffer: a moving statistic has a zero gradient and zero slots, so Adam leaves it unchanged
    // bit for bit (m = v = 0, p - lr_t * 0 / eps = p) and only the trainable variables move.
    launch_adam(params, grads, m, v, h->numel, lr, beta1, beta2, eps, state, (cudaStream_t)stream);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? WUN_OK : fail(WUN_E_CUDA, std::string("spectrogram Adam: ") + cudaGetErrorString(e));
}

int wun_spec_feed_batch(WunSpecHandle* h, const float* pool, int64_t total_frames, const int64_t* track_offset,
                        const int64_t* track_length, int64_t n_tracks, int64_t batch, int augmentation, uint64_t seed,
                        int64_t* step_state, float* mix_out, float* targets_out, int64_t* chosen, void* stream) {
    if (!h || !pool || !track_offset || !track_length || !step_state || !mix_out || !targets_out)
        return fail(WUN_E_INVALID, "null argument");
    if (n_tracks < 1 || n_tracks > (1 << 30) || batch < 1 || batch > 65535 || total_frames < h->T)
        return fail(WUN_E_INVALID, "feeder: need >= 1 track, 1 <= batch <= 65535 and a pool of at least T frames");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    cudaError_t e = launch_feed_batch(pool, total_frames, (const long long*)track_offset, (const long long*)track_length,
                                      (int)n_tracks, (int)batch, h->cfg.num_sources, 1, (int)h->T, (int)h->T, augmentation,
                                      (unsigned long long)seed, (long long*)step_state, mix_out, targets_out,
                                      (long long*)chosen, (cudaStream_t)stream);
    return e == cudaSuccess ? WUN_OK : fail(WUN_E_CUDA, std::string("spectrogram feeder: ") + cudaGetErrorString(e));
}

}  // extern "C"
