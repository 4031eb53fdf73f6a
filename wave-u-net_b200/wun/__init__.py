"""ctypes binding of libwun.so (include/wun.h) - the only way Python reaches the CUDA engine.

No fallback of any kind lives here: if the shared library is missing the import fails loudly, and the
compute entry points fail with WUN_E_NOGPU when there is no CUDA device.
"""
import ctypes
import os

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.environ.get("WUN_LIB") or os.path.join(_PKG, "libwun.so")   # WUN_LIB: A/B-test another build

WUN_OK, WUN_E_INVALID, WUN_E_NOTIMPL, WUN_E_SHAPE, WUN_E_CUDA, WUN_E_NOGPU = 0, -1, -2, -3, -4, -5

# every symbol include/wun.h declares (tests check that the library exports all of them)
SYMBOLS = [
    "wun_get_padding", "wun_create", "wun_create_for_input", "wun_destroy", "wun_input_frames",
    "wun_output_frames", "wun_param_count", "wun_param_numel", "wun_param_table", "wun_workspace_bytes",
    "wun_forward_flops", "wun_forward_backward_flops", "wun_launches_forward",
    "wun_launches_forward_backward", "wun_forward", "wun_forward_backward", "wun_adam_step", "wun_adam_step_device", "wun_set_grad_buckets", "wun_stream_wait_grad_bucket",
    "wun_gather_windows", "wun_scatter_windows", "wun_feed_batch", "wun_last_error", "wun_version", "wun_describe",
    "wun_layer_kernel", "wun_debug_tensor", "wun_debug_run_conv", "wun_debug_run_layer", "wun_crc32c", "wun_debug_plan", "wun_debug_launches",
    "wun_bss_eval_workspace_bytes", "wun_bss_eval", "wun_resample_frames", "wun_resample",
    "wun_snippet_batch", "wun_eval_batch_loss",
]


class WunConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        "num_layers", "num_initial_filters", "filter_size", "merge_filter_size", "input_filter_size",
        "output_filter_size", "upsampling", "output_type", "context", "num_channels", "num_sources",
        "output_activation")]


class WunParamInfo(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 64), ("ndim", ctypes.c_int32), ("shape", ctypes.c_int32 * 3),
                ("offset", ctypes.c_int64), ("numel", ctypes.c_int64)]


class WunError(RuntimeError):
    def __init__(self, code, msg):
        RuntimeError.__init__(self, "libwun error %d: %s" % (code, msg))
        self.code = code


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "%s not found. Build it with wave-u-net_b200/build.sh (or __graft_entry__.build()). "
            "There is no CPU or PyTorch fallback for the Wave-U-Net engine." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    P, I64, F, VP = ctypes.POINTER, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p
    H = VP
    lib.wun_get_padding.argtypes = [P(WunConfig), I64, P(I64), P(I64)]
    lib.wun_create.argtypes = [P(WunConfig), I64, P(H)]
    lib.wun_create_for_input.argtypes = [P(WunConfig), I64, P(H)]
    lib.wun_destroy.argtypes = [H]
    for n in ("wun_input_frames", "wun_output_frames", "wun_param_count", "wun_param_numel",
              "wun_launches_forward", "wun_launches_forward_backward"):
        getattr(lib, n).argtypes = [H]
        getattr(lib, n).restype = I64
    lib.wun_param_table.argtypes = [H, P(WunParamInfo), I64]
    lib.wun_workspace_bytes.argtypes = [H, I64, ctypes.c_int]
    lib.wun_workspace_bytes.restype = I64
    for n in ("wun_forward_flops", "wun_forward_backward_flops"):
        getattr(lib, n).argtypes = [H, I64]
        getattr(lib, n).restype = ctypes.c_double
    lib.wun_forward.argtypes = [H, VP, VP, I64, ctypes.c_int, VP, VP, I64, VP]
    lib.wun_forward_backward.argtypes = [H, VP, VP, VP, I64, VP, VP, VP, F, VP, I64, VP]
    lib.wun_adam_step.argtypes = [H, VP, VP, VP, VP, I64, F, F, F, F, VP]
    lib.wun_adam_step_device.argtypes = [H, VP, VP, VP, VP, VP, F, F, F, F, VP]
    lib.wun_set_grad_buckets.argtypes = [H, ctypes.c_int, P(I64)]
    lib.wun_stream_wait_grad_bucket.argtypes = [H, ctypes.c_int, VP]
    lib.wun_gather_windows.argtypes = [H, VP, I64, VP, I64, VP, VP]
    lib.wun_scatter_windows.argtypes = [H, VP, VP, I64, VP, I64, VP]
    lib.wun_feed_batch.argtypes = [H, VP, I64, VP, VP, I64, I64, ctypes.c_int, ctypes.c_uint64, VP, VP, VP, VP, VP]
    lib.wun_last_error.restype = ctypes.c_char_p
    lib.wun_version.restype = ctypes.c_char_p
    lib.wun_describe.argtypes = [H, ctypes.c_char_p, I64]
    lib.wun_describe.restype = I64
    lib.wun_debug_tensor.argtypes = [H, ctypes.c_char_p, I64, ctypes.c_int, P(I64), P(I64), P(ctypes.c_int32)]
    lib.wun_debug_run_conv.argtypes = [H, ctypes.c_int, ctypes.c_int, VP, VP, I64, VP, I64, VP, P(ctypes.c_double)]
    lib.wun_debug_run_layer.argtypes = [H, ctypes.c_int, ctypes.c_int, ctypes.c_int, VP, VP, VP, I64, VP, I64, VP,
                                        P(ctypes.c_double)]
    lib.wun_layer_kernel.argtypes = [H, ctypes.c_int, ctypes.c_int]
    lib.wun_layer_kernel.restype = ctypes.c_char_p
    lib.wun_debug_plan.argtypes = [H, I64, ctypes.c_char_p, I64]
    lib.wun_debug_plan.restype = I64
    lib.wun_debug_launches.argtypes = [H, I64, ctypes.c_char_p, I64]
    lib.wun_debug_launches.restype = I64
    lib.wun_crc32c.argtypes = [ctypes.c_uint32, VP, ctypes.c_uint64]
    lib.wun_crc32c.restype = ctypes.c_uint32
    if hasattr(lib, "wun_bss_eval"):        # the host-simulation build (tests/hostsim, WUN_LIB) leaves the scoring kernels out
        lib.wun_bss_eval_workspace_bytes.argtypes = [I64, I64, I64, I64, I64]
        lib.wun_bss_eval_workspace_bytes.restype = I64
        lib.wun_bss_eval.argtypes = [VP, VP, I64, I64, I64, I64, I64, VP, VP, VP, I64, VP]
    if hasattr(lib, "wun_resample"):        # likewise the resampling kernel
        lib.wun_resample_frames.argtypes = [I64, I64, I64]
        lib.wun_resample_frames.restype = I64
        lib.wun_resample.argtypes = [VP, I64, I64, I64, I64, VP, VP, I64, I64, VP, I64, VP]
    if hasattr(lib, "wun_snippet_batch"):   # likewise the validation-loss kernels
        lib.wun_snippet_batch.argtypes = [VP, I64, I64, I64, I64, I64, VP, I64, I64, VP, VP, VP, VP]
        lib.wun_eval_batch_loss.argtypes = [VP, VP, I64, I64, VP, VP, VP, I64, VP]
    return lib


lib = _load()


def crc32c(data, crc=0):
    """CRC-32C of a bytes-like object / C-contiguous numpy array (host helper of the library, no GPU needed)."""
    import numpy as np
    a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data).view(np.uint8).reshape(-1)
    if a.size == 0:
        return int(crc) & 0xffffffff
    return int(lib.wun_crc32c(int(crc) & 0xffffffff, a.ctypes.data_as(ctypes.c_void_p), a.size))


def check(rc):
    if rc != WUN_OK:
        msg = lib.wun_last_error().decode("utf-8", "replace")
        if rc == WUN_E_NOTIMPL:
            raise NotImplementedError(msg)          # reference: UnetAudioSeparator.py:136,144
        if rc == WUN_E_SHAPE:
            raise AssertionError(msg)               # reference: asserts :55, :121, Utils.py:114-117
        raise WunError(rc, msg)


BSS_FILTER_LEN = 512


def bss_eval(references, estimates, win, hop, filters=False):
    """BSS Eval v4 of `estimates` against `references` (include/wun.h wun_bss_eval): both contiguous float32 CUDA tensors
    [nsrc, nsampl, nchan] on one device.  Returns float64 CUDA tensors (SDR, ISR, SIR, SAR), each [nsrc, nwin]; with
    filters=True also (C [nsrc, nchan, nsrc, nchan, 512], Cj [nsrc, nchan, nchan, 512]): the filters for all sources and
    for each source alone, indexed [target, estimate channel, (source,) reference channel, tap]."""
    import torch
    for t in (references, estimates):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 3, \
            "references / estimates must be contiguous float32 CUDA tensors [nsrc, nsampl, nchan]"
    assert estimates.shape == references.shape and estimates.device == references.device, "estimates must match references"
    nsrc, n, nchan = (int(s) for s in references.shape)
    nbytes = lib.wun_bss_eval_workspace_bytes(nsrc, nchan, n, int(win), int(hop))
    if nbytes < 0:
        raise WunError(WUN_E_INVALID, "bss_eval: need 1 <= nsrc <= 8, nchan 1 or 2, nsampl, win, hop >= 1 (got %d, %d, %d, %d, %d)"
                       % (nsrc, nchan, n, win, hop))
    nwin = (n - win) // hop + 1 if n >= win else 0
    dev = references.device
    metrics = torch.empty((4, nsrc, nwin), dtype=torch.float64, device=dev)
    filt = None
    if filters:
        filt = torch.empty(nsrc * nchan * (nsrc * nchan + nchan) * BSS_FILTER_LEN, dtype=torch.float64, device=dev)
    ws = torch.empty((nbytes + 255) // 256 * 32, dtype=torch.float64, device=dev)      # torch allocations are 256-B aligned
    with torch.cuda.device(dev):
        rc = lib.wun_bss_eval(references.data_ptr(), estimates.data_ptr(), nsrc, nchan, n, int(win), int(hop),
                              metrics.data_ptr() if nwin else None, filt.data_ptr() if filt is not None else None,
                              ws.data_ptr(), ws.numel() * 8, Engine._stream(dev))
    if rc != WUN_OK:
        raise WunError(rc, "wun_bss_eval failed")
    out = tuple(metrics)
    if filters:
        nc = nsrc * nchan * nsrc * nchan * BSS_FILTER_LEN
        out += (filt[:nc].view(nsrc, nchan, nsrc, nchan, BSS_FILTER_LEN),
                filt[nc:].view(nsrc, nchan, nchan, BSS_FILTER_LEN))
    return out


# resampy 0.2's 'kaiser_best' filter, which librosa 0.6.2 resample() uses by default: sinc_window(num_zeros=64, precision=9,
# window=kaiser(beta), rolloff).  These constants and the symmetric window below are recalled from resampy, not read from it.
KAISER_BEST_ZEROS = 64
KAISER_BEST_PRECISION = 2 ** 9
KAISER_BEST_ROLLOFF = 0.9475937167399596
KAISER_BEST_BETA = 14.769656459379492
_kaiser_best = None
_resample_tables = {}


def kaiser_best_filter():
    """(half window float64 [32769], precision): rolloff * sinc(rolloff * x) for x = 0 .. 64 zero crossings in steps of
    1/512, times the right half of a symmetric Kaiser window of length 65537 (resampy.filters.sinc_window).  Built once."""
    global _kaiser_best
    if _kaiser_best is None:
        import numpy as np
        import scipy.signal
        n = KAISER_BEST_PRECISION * KAISER_BEST_ZEROS
        sinc = KAISER_BEST_ROLLOFF * np.sinc(KAISER_BEST_ROLLOFF * np.linspace(0, KAISER_BEST_ZEROS, num=n + 1, endpoint=True))
        taper = scipy.signal.windows.kaiser(2 * n + 1, KAISER_BEST_BETA, sym=True)[n:]
        _kaiser_best = (taper * sinc, KAISER_BEST_PRECISION)
    return _kaiser_best


def resample_tables(sr_in, sr_out):
    """(win, delta) float64 numpy arrays as resampy.resample hands them to resample_f: the kaiser_best half window, times
    the ratio when downsampling, and its np.diff with a trailing zero."""
    import numpy as np
    win, _ = kaiser_best_filter()
    ratio = float(sr_out) / sr_in
    if ratio < 1:
        win = win * ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    return win, delta


def resample_frames(n_in, sr_in, sr_out):
    """librosa.resample's output length, ceil(n_in * sr_out / sr_in) (include/wun.h wun_resample_frames)."""
    n = lib.wun_resample_frames(int(n_in), int(sr_in), int(sr_out))
    if n < 0:
        raise ValueError("resample: need n_in >= 0 and positive rates (got %d, %d, %d)" % (n_in, sr_in, sr_out))
    return n


def resample(x, sr_in, sr_out):
    """librosa.resample(x.T, sr_in, sr_out).T with res_type='kaiser_best' (resampy 0.2) on the GPU, bit for bit
    (include/wun.h wun_resample): `x` a contiguous float32 CUDA tensor [n, C], C 1 or 2.  Returns `x` itself when the rates
    are equal, as librosa does; raises ValueError when the input is too short to give one output frame."""
    import torch
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2 and x.shape[1] in (1, 2), \
        "x must be a contiguous float32 CUDA tensor [n, 1 or 2]"
    sr_in, sr_out = int(sr_in), int(sr_out)
    if sr_in <= 0 or sr_out <= 0:
        raise ValueError("resample: sample rates must be positive (got %d, %d)" % (sr_in, sr_out))
    if sr_in == sr_out:
        return x
    n_in, nchan = (int(s) for s in x.shape)
    if int(n_in * (float(sr_out) / sr_in)) < 1:
        raise ValueError("resample: an input of %d frames is too short to resample from %d to %d Hz" % (n_in, sr_in, sr_out))
    dev = x.device
    key = (str(dev), sr_in, sr_out)
    tables = _resample_tables.get(key)
    if tables is None:
        tables = tuple(torch.from_numpy(t).to(dev) for t in resample_tables(sr_in, sr_out))
        _resample_tables[key] = tables
    win, delta = tables
    n_out = resample_frames(n_in, sr_in, sr_out)
    y = torch.empty((n_out, nchan), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        rc = lib.wun_resample(x.data_ptr(), n_in, nchan, sr_in, sr_out, win.data_ptr(), delta.data_ptr(), win.numel(),
                              KAISER_BEST_PRECISION, y.data_ptr(), n_out, Engine._stream(dev))
    if rc != WUN_OK:
        raise WunError(rc, "wun_resample failed")
    return y


EVAL_LOSS_CTAS = 264        # include/wun.h WUN_EVAL_LOSS_CTAS


def _check_f32(name, t, dim):
    import torch
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == dim, \
        "%s must be a contiguous float32 CUDA tensor with %d dimensions" % (name, dim)


def snippet_batch(pool, positions, batch, batch_state, mix_out, targets_out):
    """One evaluation batch cut out of a partition pool (include/wun.h wun_snippet_batch): `pool` float32 [K + 1, frames, C]
    (sources, then the mix), `positions` int64 [n_batches * batch] absolute snippet frames, `batch_state` int64 [1] the batch
    counter the call advances, `mix_out` [batch, T_in, C] and `targets_out` [K, batch, T_out, C] (centre crop).  All contiguous
    CUDA tensors on one device; the call is enqueued on its current stream."""
    import torch
    _check_f32("pool", pool, 3)
    _check_f32("mix_out", mix_out, 3)
    _check_f32("targets_out", targets_out, 4)
    for name, t in (("positions", positions), ("batch_state", batch_state)):
        assert t.is_cuda and t.dtype == torch.int64 and t.is_contiguous(), "%s must be a contiguous int64 CUDA tensor" % name
    dev = pool.device
    assert all(t.device == dev for t in (positions, batch_state, mix_out, targets_out)), "tensors on different devices"
    K, C = int(pool.shape[0]) - 1, int(pool.shape[2])
    t_in, t_out = int(mix_out.shape[1]), int(targets_out.shape[2])
    assert tuple(mix_out.shape) == (batch, t_in, C), ("mix_out shape", tuple(mix_out.shape))
    assert tuple(targets_out.shape) == (K, batch, t_out, C), ("targets_out shape", tuple(targets_out.shape))
    with torch.cuda.device(dev):
        rc = lib.wun_snippet_batch(pool.data_ptr(), int(pool.shape[1]), K, C, t_in, t_out, positions.data_ptr(),
                                   positions.numel(), int(batch), batch_state.data_ptr(), mix_out.data_ptr(),
                                   targets_out.data_ptr(), Engine._stream(dev))
    if rc != WUN_OK:
        raise WunError(rc, "wun_snippet_batch failed (K %d, C %d, T_in %d, T_out %d, %d positions, batch %d)"
                       % (K, C, t_in, t_out, positions.numel(), batch))


def eval_batch_loss(outputs, targets, state, workspace, batch_loss=None):
    """Test.test's per-batch loss and running mean on the device (include/wun.h wun_eval_batch_loss): `outputs` and
    `targets` float32 [K, ...] of one shape; `state` float64 [2] {total, n}, updated in place; `workspace` float64 with at
    least K * EVAL_LOSS_CTAS elements; `batch_loss` optional float64 [1] receiving this batch's loss."""
    import torch
    assert outputs.is_cuda and outputs.dtype == torch.float32 and outputs.is_contiguous(), "outputs: contiguous float32 CUDA"
    assert targets.shape == outputs.shape and targets.dtype == torch.float32 and targets.is_contiguous(), "targets must match outputs"
    for name, t in (("state", state), ("workspace", workspace), ("batch_loss", batch_loss)):
        if t is not None:
            assert t.is_cuda and t.dtype == torch.float64 and t.is_contiguous(), "%s must be a contiguous float64 CUDA tensor" % name
    dev = outputs.device
    assert all(t.device == dev for t in (targets, state, workspace) + ((batch_loss,) if batch_loss is not None else ())), \
        "tensors on different devices"
    assert state.numel() == 2, "state is {total, n}"
    K = int(outputs.shape[0])
    with torch.cuda.device(dev):
        rc = lib.wun_eval_batch_loss(outputs.data_ptr(), targets.data_ptr(), K, outputs.numel() // K, state.data_ptr(),
                                     batch_loss.data_ptr() if batch_loss is not None else None, workspace.data_ptr(),
                                     workspace.numel() * 8, Engine._stream(dev))
    if rc != WUN_OK:
        raise WunError(rc, "wun_eval_batch_loss failed (K %d, %d elements, workspace %d doubles)"
                       % (K, outputs.numel(), workspace.numel()))


_UPSAMPLING = {"linear": 0, "learned": 1}
_OUTPUT_TYPE = {"direct": 0, "difference": 1}
_ACTIVATION = {"tanh": 0, "linear": 1}


def config_from_model_config(mc):
    """model_config dict (Config.py) -> WunConfig; the keys are those UnetAudioSeparator.__init__
    reads (/root/reference/Models/UnetAudioSeparator.py:20-32)."""
    c = WunConfig()
    c.num_layers = int(mc["num_layers"])
    c.num_initial_filters = int(mc["num_initial_filters"])
    c.filter_size = int(mc["filter_size"])
    c.merge_filter_size = int(mc["merge_filter_size"])
    c.input_filter_size = int(mc["input_filter_size"])
    c.output_filter_size = int(mc["output_filter_size"])
    c.upsampling = _UPSAMPLING.get(mc["upsampling"], 0)     # reference: anything but 'learned' is bilinear (:110-117)
    c.output_type = _OUTPUT_TYPE.get(mc["output_type"], -1)
    c.context = 1 if mc["context"] else 0
    c.num_channels = 1 if mc["mono_downmix"] else 2
    c.num_sources = len(mc["source_names"])
    c.output_activation = _ACTIVATION.get(mc["output_activation"], -1)
    return c


def get_padding(cfg, num_frames):
    t_in, t_out = ctypes.c_int64(), ctypes.c_int64()
    check(lib.wun_get_padding(ctypes.byref(cfg), int(num_frames), ctypes.byref(t_in), ctypes.byref(t_out)))
    return t_in.value, t_out.value


class Engine(object):
    """One plan (fixed window length) of the CUDA engine."""

    def __init__(self, cfg, num_frames=None, input_frames=None):
        self._h = ctypes.c_void_p()
        self.cfg = cfg
        if input_frames is not None:
            check(lib.wun_create_for_input(ctypes.byref(cfg), int(input_frames), ctypes.byref(self._h)))
        else:
            check(lib.wun_create(ctypes.byref(cfg), int(num_frames), ctypes.byref(self._h)))
        self.T_in = lib.wun_input_frames(self._h)
        self.T_out = lib.wun_output_frames(self._h)
        n = lib.wun_param_count(self._h)
        arr = (WunParamInfo * n)()
        check(lib.wun_param_table(self._h, arr, n))
        self.param_table = [(a.name.decode(), tuple(a.shape[:a.ndim]), int(a.offset), int(a.numel)) for a in arr]
        self.param_numel = lib.wun_param_numel(self._h)
        self._ws = {}
        self._ws_last = None

    def __del__(self):
        try:
            if self._h:
                lib.wun_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- host-only queries -------------------------------------------------------------------
    def workspace_bytes(self, batch, training):
        return lib.wun_workspace_bytes(self._h, int(batch), 1 if training else 0)

    def forward_flops(self, batch):
        return lib.wun_forward_flops(self._h, int(batch))

    def forward_backward_flops(self, batch):
        return lib.wun_forward_backward_flops(self._h, int(batch))

    def launches(self, training):
        return (lib.wun_launches_forward_backward if training else lib.wun_launches_forward)(self._h)

    def describe(self):
        n = lib.wun_describe(self._h, None, 0)
        buf = ctypes.create_string_buffer(int(n))
        lib.wun_describe(self._h, buf, n)
        return buf.value.decode()

    def plan_audit(self, batch):
        """[dict] - one per tensor-core launch of a training step at `batch` (planner decisions; no GPU needed)."""
        n = lib.wun_debug_plan(self._h, int(batch), None, 0)
        if n < 0:
            raise RuntimeError("wun_debug_plan failed: %s" % lib.wun_last_error().decode())
        buf = ctypes.create_string_buffer(int(n))
        lib.wun_debug_plan(self._h, int(batch), buf, n)
        out = []
        for line in buf.value.decode().splitlines():
            parts = line.split()
            d = {"op": parts[0]}
            for kv in parts[1:]:
                k, v = kv.split("=", 1)
                d[k] = int(v) if v.lstrip("-").isdigit() else v
            out.append(d)
        return out

    def launch_descriptions(self, batch):
        """Every plane-convolution launch of a training step at `batch` as a list of dicts {"launch": {...}, "planes": [...],
        "cls": [...], "terms": [...]} (wun_debug_launches; host only).  The same dry run also leaves the weight-gradient groups in
        self.wgrad_groups and the step's other launches in self.step_launches: [(kind, {...})] with kind "first" (first layer,
        forward and weight gradient), "output" (output layer), "upsample" (one per up level) or "adam"."""
        n = lib.wun_debug_launches(self._h, int(batch), None, 0)
        if n < 0:
            raise RuntimeError("wun_debug_launches failed: %s" % lib.wun_last_error().decode())
        buf = ctypes.create_string_buffer(int(n))
        lib.wun_debug_launches(self._h, int(batch), buf, n)
        out, wg, step = [], [], []
        for line in buf.value.decode().splitlines():
            parts = line.split()
            d = {k: int(v) for k, v in (kv.split("=", 1) for kv in parts[1:])}
            if parts[0] in ("first", "output", "upsample", "adam"):
                step.append((parts[0], d))
            elif parts[0] == "launch":
                out.append({"launch": d, "planes": [], "cls": [], "terms": []})
            elif parts[0] == "wgrad":
                wg.append({"wgrad": d, "plane": None, "dpre": None, "terms": []})
            elif parts[0] in ("wplane", "wdpre"):
                wg[-1]["plane" if parts[0] == "wplane" else "dpre"] = d
            elif parts[0] == "wterm":
                wg[-1]["terms"].append(d)
            else:
                out[-1][{"plane": "planes", "cls": "cls", "term": "terms"}[parts[0]]].append(d)
        self.wgrad_groups = wg          # the weight-gradient (class, plane) groups of the same dry run
        self.step_launches = step
        return out

    def layer_kernel(self, layer, pass_):
        return lib.wun_layer_kernel(self._h, int(layer), int(pass_)).decode()

    def debug_tensor(self, name, batch, training):
        """View [batch, rows, C] of a saved activation inside the current workspace (tests only)."""
        off, rows, ch = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int32()
        check(lib.wun_debug_tensor(self._h, name.encode(), int(batch), 1 if training else 0, ctypes.byref(off),
                                   ctypes.byref(rows), ctypes.byref(ch)))
        ws = next((w for k, w in self._ws.items() if k[:2] == (int(batch), bool(training))), self._ws_last)
        n = int(batch) * rows.value * ch.value
        return ws[off.value:off.value + n].view(int(batch), rows.value, ch.value)

    def run_conv_layer(self, layer, iters, params, mix):
        """Benchmark hook: enqueue the forward kernel of one conv layer `iters` times (after a training step filled
        the workspace).  Returns the layer's algorithmic FLOPs per launch."""
        B = mix.shape[0]
        ws = self._workspace(B, True, mix.device)
        fl = ctypes.c_double()
        check(lib.wun_debug_run_conv(self._h, int(layer), int(iters), params.data_ptr(), mix.data_ptr(), B,
                                     ws.data_ptr(), ws.numel() * 4, self._stream(mix.device), ctypes.byref(fl)))
        return fl.value

    def run_layer_pass(self, layer, pass_, iters, params, mix, grads_scratch=None):
        """Benchmark hook: enqueue every launch of one pass (0 fwd, 1 dgrad, 2 wgrad) of conv layer `layer` `iters` times
        on the current stream, on the tensors a previous training step left in the workspace.  Returns the pass's
        algorithmic FLOPs per iteration."""
        B = mix.shape[0]
        ws = self._workspace(B, True, mix.device)
        fl = ctypes.c_double()
        check(lib.wun_debug_run_layer(self._h, int(layer), int(pass_), int(iters), params.data_ptr(), mix.data_ptr(),
                                      grads_scratch.data_ptr() if grads_scratch is not None else None, B,
                                      ws.data_ptr(), ws.numel() * 4, self._stream(mix.device), ctypes.byref(fl)))
        return fl.value

    # ---- device calls (torch tensors supply memory and the stream) --------------------------------
    def _workspace(self, batch, training, device):
        import torch
        # One workspace per (batch, mode, device), never freed while the engine lives: a captured CUDA graph bakes the
        # raw pointer in, and Training.optimise alternates training steps with forward-only validation.
        key = (int(batch), bool(training), str(device))
        ws = self._ws.get(key)
        if ws is None:
            nbytes = self.workspace_bytes(batch, training)
            ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=device)
            self._ws[key] = ws
        self._ws_last = ws
        return ws

    def release_workspaces(self):
        """Drop every cached workspace (only safe when no captured graph refers to them)."""
        self._ws = {}
        self._ws_last = None

    @staticmethod
    def _stream(device=None):
        """The current torch stream of the tensors' device (not of whatever device happens to be current)."""
        import torch
        return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)

    def _check_io(self, mix, targets=None, out=None, flat=()):
        import torch
        B = mix.shape[0]
        K, C = self.cfg.num_sources, self.cfg.num_channels
        assert mix.is_cuda and mix.dtype == torch.float32 and mix.is_contiguous(), "mix must be a contiguous float32 CUDA tensor"
        assert tuple(mix.shape[1:]) == (self.T_in, C), ("mix shape", tuple(mix.shape), "expected [B, %d, %d]" % (self.T_in, C))
        for name, t in (("targets", targets), ("outputs", out)):
            if t is None:
                continue
            assert t.is_cuda and t.device == mix.device and t.dtype == torch.float32 and t.is_contiguous(), name
            assert tuple(t.shape) == (K, B, self.T_out, C), (name, tuple(t.shape), "expected", (K, B, self.T_out, C))
        for t in flat:
            assert t.is_cuda and t.device == mix.device and t.dtype == torch.float32 and t.is_contiguous()
            assert t.numel() >= self.param_numel, ("flat buffer too small", t.numel(), self.param_numel)

    def forward(self, params, mix, training, out=None):
        import torch
        B = mix.shape[0]
        K, C = self.cfg.num_sources, self.cfg.num_channels
        if out is None:
            out = torch.empty((K, B, self.T_out, C), dtype=torch.float32, device=mix.device)
        self._check_io(mix, out=out, flat=(params,))
        ws = self._workspace(B, False, mix.device)
        with torch.cuda.device(mix.device):
            check(lib.wun_forward(self._h, params.data_ptr(), mix.data_ptr(), B, 1 if training else 0, out.data_ptr(),
                                  ws.data_ptr(), ws.numel() * 4, self._stream(mix.device)))
        return out

    def forward_backward(self, params, mix, targets, grads, loss, grad_scale=1.0, out=None):
        import torch
        B = mix.shape[0]
        self._check_io(mix, targets=targets, out=out, flat=(params, grads))
        ws = self._workspace(B, True, mix.device)
        with torch.cuda.device(mix.device):
            check(lib.wun_forward_backward(self._h, params.data_ptr(), mix.data_ptr(), targets.data_ptr(), B,
                                           out.data_ptr() if out is not None else None, loss.data_ptr(),
                                           grads.data_ptr(), float(grad_scale), ws.data_ptr(), ws.numel() * 4,
                                           self._stream(mix.device)))
        return loss

    def adam_step(self, params, grads, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8):
        import torch
        with torch.cuda.device(params.device):
            check(lib.wun_adam_step(self._h, params.data_ptr(), grads.data_ptr(), m.data_ptr(), v.data_ptr(), int(step),
                                    float(lr), float(beta1), float(beta2), float(eps), self._stream(params.device)))

    def adam_step_device(self, params, grads, m, v, state, lr, beta1=0.9, beta2=0.999, eps=1e-8):
        """Graph-safe Adam: `state` = device float32[3] {beta1_power, beta2_power, step} (include/wun.h)."""
        import torch
        with torch.cuda.device(params.device):
            check(lib.wun_adam_step_device(self._h, params.data_ptr(), grads.data_ptr(), m.data_ptr(), v.data_ptr(),
                                           state.data_ptr(), float(lr), float(beta1), float(beta2), float(eps),
                                           self._stream(params.device)))

    def set_grad_buckets(self, first_offsets):
        """Gradient buckets in production order (include/wun.h): strictly descending first flat offsets, the last one 0."""
        arr = (ctypes.c_int64 * len(first_offsets))(*[int(o) for o in first_offsets])
        check(lib.wun_set_grad_buckets(self._h, len(first_offsets), arr))
        self.grad_buckets = [int(o) for o in first_offsets]

    def stream_wait_grad_bucket(self, k, stream):
        """Make torch stream `stream` wait until bucket k of the last enqueued forward_backward is final."""
        check(lib.wun_stream_wait_grad_bucket(self._h, int(k), ctypes.c_void_p(stream.cuda_stream)))

    def feed_batch(self, pool, track_offset, track_length, batch, augmentation, seed, step_state, mix_out, targets_out,
                   chosen=None):
        """One training batch cut out of the device-resident track pool (wun_feed_batch): random snippet per example,
        random_amplify, centre crop.  All arguments are CUDA tensors owned by the caller (wun.feeder.DeviceFeeder)."""
        import torch
        K = targets_out.shape[0]
        assert K == self.cfg.num_sources and pool.shape[2] == self.cfg.num_channels
        assert pool.is_cuda and pool.dtype == torch.float32 and pool.is_contiguous() and pool.dim() == 3 and pool.shape[0] == K + 1
        assert track_offset.dtype == torch.int64 and track_length.dtype == torch.int64 and step_state.dtype == torch.int64
        assert tuple(mix_out.shape) == (batch, self.T_in, pool.shape[2]) and mix_out.is_contiguous()
        assert tuple(targets_out.shape) == (K, batch, self.T_out, pool.shape[2]) and targets_out.is_contiguous()
        with torch.cuda.device(mix_out.device):
          check(lib.wun_feed_batch(self._h, pool.data_ptr(), pool.shape[1], track_offset.data_ptr(), track_length.data_ptr(),
                                 track_offset.numel(), int(batch), int(bool(augmentation)), int(seed) & (2 ** 64 - 1),
                                 step_state.data_ptr(), mix_out.data_ptr(), targets_out.data_ptr(),
                                 chosen.data_ptr() if chosen is not None else None, self._stream(mix_out.device)))

    def gather_windows(self, padded, starts, mix_batch):
        check(lib.wun_gather_windows(self._h, padded.data_ptr(), padded.shape[0], starts.data_ptr(),
                                     starts.numel(), mix_batch.data_ptr(), self._stream(padded.device)))

    def scatter_windows(self, outputs, starts, preds):
        check(lib.wun_scatter_windows(self._h, outputs.data_ptr(), starts.data_ptr(), starts.numel(),
                                      preds.data_ptr(), preds.shape[1], self._stream(preds.device)))
