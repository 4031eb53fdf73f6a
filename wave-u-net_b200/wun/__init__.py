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
    "wun_bss_eval_workspace_bytes", "wun_bss_eval", "wun_bss_eval_v3_workspace_bytes", "wun_bss_eval_v3",
    "wun_bss_eval_ex_workspace_bytes", "wun_bss_eval_ex",
    "wun_resample_frames", "wun_resample",
    "wun_snippet_batch", "wun_eval_batch_loss",
    "wun_spec_create", "wun_spec_destroy", "wun_spec_input_frames", "wun_spec_output_frames", "wun_spec_stft_frames",
    "wun_spec_param_count", "wun_spec_param_numel", "wun_spec_param_table", "wun_spec_workspace_bytes",
    "wun_spec_forward_flops", "wun_spec_launches_forward", "wun_spec_forward", "wun_spec_l1_batch_loss",
    "wun_spec_gather_windows", "wun_spec_scatter_windows",
    "wun_spec_train_workspace_bytes", "wun_spec_train_flops", "wun_spec_forward_backward", "wun_spec_forward_backward_dp",
    "wun_spec_adam_step_device",
    "wun_spec_feed_batch", "wun_spec_debug_train_level", "wun_spec_debug_train_buffer",
    "wun_flac_find_frames", "wun_flac_decode_frames",
    "wun_flac_encode_workspace_bytes", "wun_flac_encode_capacity", "wun_flac_encode_frames",
]


class WunConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        "num_layers", "num_initial_filters", "filter_size", "merge_filter_size", "input_filter_size",
        "output_filter_size", "upsampling", "output_type", "context", "num_channels", "num_sources",
        "output_activation")]


class WunParamInfo(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 64), ("ndim", ctypes.c_int32), ("shape", ctypes.c_int32 * 3),
                ("offset", ctypes.c_int64), ("numel", ctypes.c_int64)]


class WunSpecConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("num_layers", "num_initial_filters", "num_channels", "num_sources")]


class WunSpecParamInfo(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 64), ("ndim", ctypes.c_int32), ("shape", ctypes.c_int32 * 4),
                ("offset", ctypes.c_int64), ("numel", ctypes.c_int64)]


# int gather(void* ctx, const double* local, double* gathered, int64_t count, void* stream) (include/wun.h WunSpecGatherFn)
SPEC_GATHER_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                  ctypes.c_void_p)


class WunSpecShard(ctypes.Structure):
    _fields_ = [("rank", ctypes.c_int32), ("world", ctypes.c_int32), ("global_batch", ctypes.c_int64),
                ("sample_offset", ctypes.c_int64), ("gathered", ctypes.c_void_p), ("gathered_bytes", ctypes.c_int64),
                ("gather", SPEC_GATHER_FN), ("ctx", ctypes.c_void_p)]


class WunFlacFrame(ctypes.Structure):
    _fields_ = [("offset", ctypes.c_int64), ("number", ctypes.c_int64), ("end", ctypes.c_int64),
                ("block_size", ctypes.c_int32), ("variable", ctypes.c_int32)]


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
    if hasattr(lib, "wun_bss_eval_v3"):     # likewise, and builds from before v3 (WUN_LIB)
        lib.wun_bss_eval_v3_workspace_bytes.argtypes = [I64, I64, I64, I64, I64, I64]
        lib.wun_bss_eval_v3_workspace_bytes.restype = I64
        lib.wun_bss_eval_v3.argtypes = lib.wun_bss_eval.argtypes
    if hasattr(lib, "wun_bss_eval_ex"):     # likewise, and builds from before the permutation search (WUN_LIB)
        lib.wun_bss_eval_ex_workspace_bytes.argtypes = [I64, I64, I64, I64, I64, ctypes.c_int, I64]
        lib.wun_bss_eval_ex_workspace_bytes.restype = I64
        lib.wun_bss_eval_ex.argtypes = [VP, VP, I64, I64, I64, I64, I64, ctypes.c_int, VP, VP, VP, VP, VP, I64, VP]
    if hasattr(lib, "wun_resample"):        # likewise the resampling kernel
        lib.wun_resample_frames.argtypes = [I64, I64, I64]
        lib.wun_resample_frames.restype = I64
        lib.wun_resample.argtypes = [VP, I64, I64, I64, I64, VP, VP, I64, I64, VP, I64, VP]
    if hasattr(lib, "wun_flac_find_frames"):    # likewise the FLAC decoder
        I32 = ctypes.c_int32
        lib.wun_flac_find_frames.argtypes = [VP, I64, I32, I32, I32, I32, VP, I64, VP, VP]
        lib.wun_flac_decode_frames.argtypes = [VP, I64, I32, I32, I32, I32, VP, VP, I64, VP, I64, VP, VP]
    if hasattr(lib, "wun_flac_encode_frames"):  # likewise the FLAC encoder
        I32 = ctypes.c_int32
        lib.wun_flac_encode_workspace_bytes.argtypes = [I64, I32, I32]
        lib.wun_flac_encode_workspace_bytes.restype = I64
        lib.wun_flac_encode_capacity.argtypes = [I64, I32, I32, I32]
        lib.wun_flac_encode_capacity.restype = I64
        lib.wun_flac_encode_frames.argtypes = [VP, I32, I64, I32, I32, I32, I32, VP, I64, VP, I64, VP, VP]
    if hasattr(lib, "wun_snippet_batch"):   # likewise the validation-loss kernels
        lib.wun_snippet_batch.argtypes = [VP, I64, I64, I64, I64, I64, VP, I64, I64, VP, VP, VP, VP]
        lib.wun_eval_batch_loss.argtypes = [VP, VP, I64, I64, VP, VP, VP, I64, VP]
    if hasattr(lib, "wun_spec_create"):     # likewise the spectrogram U-Net
        lib.wun_spec_create.argtypes = [P(WunSpecConfig), I64, P(H)]
        lib.wun_spec_destroy.argtypes = [H]
        for n in ("wun_spec_input_frames", "wun_spec_output_frames", "wun_spec_stft_frames", "wun_spec_param_count",
                  "wun_spec_param_numel"):
            getattr(lib, n).argtypes = [H]
            getattr(lib, n).restype = I64
        lib.wun_spec_param_table.argtypes = [H, P(WunSpecParamInfo), I64]
        lib.wun_spec_workspace_bytes.argtypes = [H, I64]
        lib.wun_spec_workspace_bytes.restype = I64
        lib.wun_spec_forward_flops.argtypes = [H, I64]
        lib.wun_spec_forward_flops.restype = ctypes.c_double
        lib.wun_spec_launches_forward.argtypes = [H, ctypes.c_int]
        lib.wun_spec_launches_forward.restype = I64
        lib.wun_spec_forward.argtypes = [H, VP, VP, I64, ctypes.c_int, VP, VP, I64, VP]
        lib.wun_spec_l1_batch_loss.argtypes = [H, VP, VP, I64, VP, VP, VP, I64, VP]
        lib.wun_spec_gather_windows.argtypes = [H, VP, I64, VP, I64, VP, VP]
        lib.wun_spec_scatter_windows.argtypes = [H, VP, VP, I64, VP, I64, VP]
        lib.wun_spec_train_workspace_bytes.argtypes = [H, I64]
        lib.wun_spec_train_workspace_bytes.restype = I64
        lib.wun_spec_train_flops.argtypes = [H, I64]
        lib.wun_spec_train_flops.restype = ctypes.c_double
        lib.wun_spec_forward_backward.argtypes = [H, VP, VP, VP, I64, ctypes.c_int, ctypes.c_uint64, VP, VP, VP, VP, I64,
                                                  VP]
        lib.wun_spec_forward_backward_dp.argtypes = lib.wun_spec_forward_backward.argtypes + [P(WunSpecShard)]
        lib.wun_spec_adam_step_device.argtypes = [H, VP, VP, VP, VP, VP, F, F, F, F, VP]
        lib.wun_spec_debug_train_level.argtypes = [H, I64, ctypes.c_int, P(I64), P(I64)]
        lib.wun_spec_debug_train_buffer.argtypes = [H, I64, ctypes.c_int, ctypes.c_int, P(I64), P(I64)]
        lib.wun_spec_feed_batch.argtypes = [H, VP, I64, VP, VP, I64, I64, ctypes.c_int, ctypes.c_uint64, VP, VP, VP, VP, VP]
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
BSS_MODES = ("v4", "v3")
BSS_V3_WORKSPACE_BYTES = 2 << 30        # 1-s frames at 44.1 kHz: 12 per pass at n = 4096 (4 stereo sources), 40 at n = 2048
BSS_FRAMEWISE_FILTERS, BSS_PERMUTATION, BSS_SOURCES = 1, 2, 4       # include/wun.h WUN_BSS_*


def bss_eval(references, estimates, win, hop, filters=False, mode="v4", max_workspace_bytes=BSS_V3_WORKSPACE_BYTES,
             permutation=False, sources_version=False, pair_metrics=False):
    """BSS Eval of `estimates` against `references` as museval.evaluate(..., mode=mode) computes it: both contiguous float32
    CUDA tensors [nsrc, nsampl, nchan] on one device.  Returns float64 CUDA tensors (SDR, ISR, SIR, SAR), each [nsrc, nwin];
    with filters=True also (C [nsrc, nchan, nsrc, nchan, 512], Cj [nsrc, nchan, nchan, 512]): the filters for all sources and
    for each source alone, indexed [target, estimate channel, (source,) reference channel, tap].

    mode="v4" (include/wun.h wun_bss_eval) solves the filters once over the whole track.  mode="v3" (wun_bss_eval_v3) solves
    them for every frame from its own samples; the filters then have a leading [nwin] axis and are NaN for silent frames.
    v3 processes frames in passes, as many per pass as fit in max_workspace_bytes (at least one); the results do not depend
    on it.

    museval's bss_eval switches (wun_bss_eval_ex): permutation=True scores every (reference, estimate) pair and keeps, per
    frame, the pairing with the largest mean SIR; row j of the metrics is then estimate j, and `perm` (int64 CUDA [nsrc,
    nwin], returned right after SAR) is the reference each estimate is scored against.  pair_metrics=True (with permutation)
    also returns the metrics of every pair, float64 [4, nsrc (reference), nsrc (estimate), nwin], after perm; Cj then holds
    every pair, [reference, estimate, estimate channel, reference channel, tap].  sources_version=True scores the "sources"
    decomposition: SDR = |P_j|^2 / |est - P_j|^2 and ISR NaN; SIR and SAR as in the images version."""
    import torch
    if mode not in BSS_MODES:
        raise ValueError("bss_eval: mode=%r, must be one of %s" % (mode, ", ".join(BSS_MODES)))
    if pair_metrics and not permutation:
        raise ValueError("bss_eval: pair_metrics=True needs permutation=True")
    for t in (references, estimates):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 3, \
            "references / estimates must be contiguous float32 CUDA tensors [nsrc, nsampl, nchan]"
    assert estimates.shape == references.shape and estimates.device == references.device, "estimates must match references"
    nsrc, n, nchan = (int(s) for s in references.shape)
    win, hop = int(win), int(hop)
    nwin = (n - win) // hop + 1 if n >= win > 0 and hop > 0 else 0
    flags = ((BSS_FRAMEWISE_FILTERS if mode == "v3" else 0) | (BSS_PERMUTATION if permutation else 0)
             | (BSS_SOURCES if sources_version else 0))
    nbytes = lib.wun_bss_eval_ex_workspace_bytes(nsrc, nchan, n, win, hop, flags, 1)
    if mode == "v3" and nbytes >= 0 and nwin > 1:
        per_frame = lib.wun_bss_eval_ex_workspace_bytes(nsrc, nchan, n, win, hop, flags, 2) - nbytes
        fit = 1 + max(0, int(max_workspace_bytes) - nbytes) // per_frame
        nbytes = lib.wun_bss_eval_ex_workspace_bytes(nsrc, nchan, n, win, hop, flags, min(fit, nwin))
    if nbytes < 0:
        raise WunError(WUN_E_INVALID, "bss_eval: need 1 <= nsrc <= 8, nchan 1 or 2, nsampl, win, hop >= 1 (got %d, %d, %d, %d, %d)"
                       % (nsrc, nchan, n, win, hop))
    dev = references.device
    npair = nsrc if permutation else 1
    metrics = torch.empty((4, nsrc, nwin), dtype=torch.float64, device=dev)
    perm = torch.empty((nsrc, nwin), dtype=torch.int64, device=dev) if permutation else None
    pairs = torch.empty((4, nsrc, nsrc, nwin), dtype=torch.float64, device=dev) if pair_metrics else None
    nc = nsrc * nchan * nsrc * nchan * BSS_FILTER_LEN
    fsz = nc + nsrc * nchan * npair * nchan * BSS_FILTER_LEN
    filt = torch.empty((nwin if mode == "v3" else 1) * fsz, dtype=torch.float64, device=dev) if filters else None
    ws = torch.empty((nbytes + 255) // 256 * 32, dtype=torch.float64, device=dev)      # torch allocations are 256-B aligned
    ptr = lambda t: t.data_ptr() if t is not None and nwin else None          # noqa: E731
    with torch.cuda.device(dev):
        rc = lib.wun_bss_eval_ex(references.data_ptr(), estimates.data_ptr(), nsrc, nchan, n, win, hop, flags, ptr(metrics),
                                 ptr(perm), ptr(pairs), filt.data_ptr() if filt is not None else None, ws.data_ptr(),
                                 ws.numel() * 8, Engine._stream(dev))
    if rc != WUN_OK:
        raise WunError(rc, "wun_bss_eval_ex (flags %d) failed" % flags)
    out = tuple(metrics)
    if permutation:
        out += (perm,)
    if pair_metrics:
        out += (pairs,)
    if filters:
        f = filt.view(-1, fsz)
        lead = (nwin,) if mode == "v3" else ()
        cj = (nsrc, nsrc) if permutation else (nsrc,)
        out += (f[:, :nc].reshape(lead + (nsrc, nchan, nsrc, nchan, BSS_FILTER_LEN)),
                f[:, nc:].reshape(lead + cj + (nchan, nchan, BSS_FILTER_LEN)))
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


def read_flac(source, verify_md5=True, device="cuda"):
    """(rate, bps, samples) of a FLAC stream decoded on the GPU (include/wun.h wun_flac_find_frames / wun_flac_decode_frames,
    DESIGN.md §4.10): `source` a path or bytes; `samples` an int32 CUDA tensor [n, channels] at full depth in FLAC's channel
    order.  With verify_md5 (the default) the samples are checked against STREAMINFO's MD5 unless that is all zero (not
    computed).  A stream that is not FLAC, is not 4-24 bits per sample, or whose frames do not chain raises ValueError."""
    import numpy as np
    import torch
    from . import flac
    if isinstance(source, (bytes, bytearray, memoryview)):
        data = bytes(source)
    else:
        with open(source, "rb") as f:
            data = f.read()
    info = flac.parse_stream(data)
    area = data[info.frames_start:]
    nbytes = len(area)
    dev = torch.device(device)
    if nbytes == 0:
        if info.total_samples:
            raise ValueError("FLAC: STREAMINFO says %d samples, the stream has no frames" % info.total_samples)
        return info.rate, info.bps, torch.zeros((0, info.channels), dtype=torch.int32, device=dev)
    si = (info.bps, info.channels, info.rate, info.max_block)
    buf = torch.frombuffer(bytearray(area), dtype=torch.uint8).to(dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    # a frame is at least ~10 bytes; most streams have far fewer candidates than this, and a second pass covers the rest
    capacity = nbytes // 256 + 1024
    with torch.cuda.device(dev):
        stream = Engine._stream(dev)
        while True:
            rec = torch.empty((capacity, ctypes.sizeof(WunFlacFrame)), dtype=torch.uint8, device=dev)
            check(lib.wun_flac_find_frames(buf.data_ptr(), nbytes, *si, rec.data_ptr(), capacity, count.data_ptr(), stream))
            found = int(count.item())
            if found <= capacity:
                break
            capacity = found
        dtype = np.dtype([(n, np.int64 if t is ctypes.c_int64 else np.int32) for n, t in WunFlacFrame._fields_])
        frames = rec[:found].cpu().numpy().view(dtype).reshape(-1)
        offsets, firsts, n = flac.chain_frames(frames, nbytes, info)
        out = torch.empty((n, info.channels), dtype=torch.int32, device=dev)
        status = torch.zeros(len(offsets), dtype=torch.int32, device=dev)
        off_d, first_d = torch.from_numpy(offsets).to(dev), torch.from_numpy(firsts).to(dev)
        check(lib.wun_flac_decode_frames(buf.data_ptr(), nbytes, *si, off_d.data_ptr(), first_d.data_ptr(), len(offsets),
                                         out.data_ptr(), n, status.data_ptr(), stream))
        bad = torch.nonzero(status).reshape(-1).cpu().numpy()
    if bad.size:
        j = int(bad[0])
        raise ValueError("FLAC frame %d at byte offset %d: %s" % (j, info.frames_start + int(offsets[j]),
                                                                  flac.STATUS.get(int(status[j]), "invalid")))
    if verify_md5 and info.md5 != bytes(16) and flac.md5_of(out, info.bps) != info.md5:
        raise ValueError("FLAC: the decoded samples do not match the stream's MD5")
    return info.rate, info.bps, out


FLAC_BLOCK_SIZE = 4096


def write_flac(samples, rate, bps, path=None, block_size=FLAC_BLOCK_SIZE):
    """The bytes of a FLAC stream of `samples` encoded on the GPU (include/wun.h wun_flac_encode_frames, DESIGN.md §4.11),
    written to `path` too when it is given.  `samples`: a CUDA tensor [n, channels] (or [n] for mono), int32 at full depth
    or float32 (quantised as wun.flac.quantise: x * 2^(bps-1) rounded half to even and clipped, the inverse of reading
    s / 2^(bps-1)).  4..24 bits per sample, 1..8 channels, any rate a frame header can express; fixed blocks of
    `block_size` (16..4608) in FLAC's streamable subset.  The host adds STREAMINFO (with the MD5 of the integer samples,
    as wun.read_flac checks it) and a VORBIS_COMMENT block; the frame area comes back in one device-to-host copy.  An int32
    sample outside the depth raises ValueError."""
    import numpy as np
    import torch
    from . import flac
    assert samples.is_cuda and samples.dtype in (torch.int32, torch.float32), \
        "samples must be an int32 or float32 CUDA tensor [n, channels]"
    x = samples.reshape(-1, 1) if samples.dim() == 1 else samples
    assert x.dim() == 2, "samples must be [n, channels]"
    x = x.contiguous()
    n, C = (int(v) for v in x.shape)
    rate, bps, block_size = int(rate), int(bps), int(block_size)
    ws_bytes = lib.wun_flac_encode_workspace_bytes(n, C, block_size)
    capacity = lib.wun_flac_encode_capacity(n, C, bps, block_size)
    if ws_bytes < 0 or capacity < 0 or not 4 <= bps <= 24:
        raise ValueError("write_flac: need 4 <= bps <= 24, 1 to 8 channels and 16 <= block_size <= 4608 (got bps %d, "
                         "%d channels, block_size %d)" % (bps, C, block_size))
    if not (0 < rate < (1 << 20) and flac.header_rate_ok(rate)):
        raise ValueError("write_flac: %d Hz cannot be written in a FLAC frame header" % rate)
    dev = x.device
    frames = (n + block_size - 1) // block_size
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    out = torch.empty(max(capacity, 4), dtype=torch.uint8, device=dev)
    offsets = torch.empty(frames + 1, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        rc = lib.wun_flac_encode_frames(x.data_ptr(), 1 if x.dtype == torch.float32 else 0, n, C, bps, rate, block_size,
                                        ws.data_ptr(), ws.numel(), out.data_ptr(), out.numel(), offsets.data_ptr(),
                                        Engine._stream(dev))
        if rc != WUN_OK:
            raise WunError(rc, "wun_flac_encode_frames failed")
        off = offsets.cpu().numpy()
        if off[-1] < 0:
            raise ValueError("write_flac: samples lie outside %d bits" % bps)
        ints = x if x.dtype == torch.int32 else ws[:n * C * 4].view(torch.int32).view(n, C)
        md5 = flac.md5_of(ints, bps)
        area = out[:int(off[-1])].cpu().numpy().tobytes()
    data = flac.assemble(area, off, block_size, rate, C, bps, n, md5)
    if path is not None:
        with open(path, "wb") as f:
            f.write(data)
    return data


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
        assert loss.is_cuda and loss.device == mix.device and loss.dtype == torch.float32, "loss must be a float32 CUDA tensor"
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


SPEC_BINS = 513             # include/wun.h WUN_SPEC_BINS


def spec_config_from_model_config(mc):
    """model_config dict (Config.py) -> WunSpecConfig: the keys UnetSpectrogramSeparator.__init__ reads."""
    c = WunSpecConfig()
    c.num_layers = int(mc["num_layers"])
    c.num_initial_filters = int(mc["num_initial_filters"])
    c.num_channels = 1 if mc["mono_downmix"] else 2
    c.num_sources = len(mc["source_names"])
    return c


class SpecEngine(object):
    """The spectrogram U-Net for one window length (include/wun.h wun_spec_*): the inference graph, and the training step
    (forward_backward, adam_step_device, feed_batch).  Mirrors the parts of Engine that Evaluate._separate_on_device,
    Test.test, Training.train and wun.feeder.DeviceFeeder use; T_in == T_out == the window length."""

    def __init__(self, cfg, num_frames=None, input_frames=None):
        self._h = ctypes.c_void_p()
        self.cfg = cfg
        check(lib.wun_spec_create(ctypes.byref(cfg), int(input_frames if input_frames is not None else num_frames),
                                  ctypes.byref(self._h)))
        self.T_in = lib.wun_spec_input_frames(self._h)
        self.T_out = lib.wun_spec_output_frames(self._h)
        self.stft_frames = lib.wun_spec_stft_frames(self._h)
        n = lib.wun_spec_param_count(self._h)
        arr = (WunSpecParamInfo * n)()
        check(lib.wun_spec_param_table(self._h, arr, n))
        self.param_table = [(a.name.decode(), tuple(a.shape[:a.ndim]), int(a.offset), int(a.numel)) for a in arr]
        self.param_numel = lib.wun_spec_param_numel(self._h)
        self._ws = {}
        self._train_ws = {}
        self._gathered = {}

    def __del__(self):
        try:
            if self._h:
                lib.wun_spec_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def workspace_bytes(self, batch):
        return lib.wun_spec_workspace_bytes(self._h, int(batch))

    def forward_flops(self, batch):
        return lib.wun_spec_forward_flops(self._h, int(batch))

    def train_workspace_bytes(self, batch):
        return lib.wun_spec_train_workspace_bytes(self._h, int(batch))

    def train_flops(self, batch):
        return lib.wun_spec_train_flops(self._h, int(batch))

    @property
    def trainable_ranges(self):
        """[(name, offset, numel)] of the variables Adam trains (kernels, biases, betas), in table order; the moving
        statistics are not among them."""
        return [(n, o, c) for n, _, o, c in self.param_table if not n.endswith(("/moving_mean", "/moving_variance"))]

    def launches(self, return_spectrogram=False):
        return lib.wun_spec_launches_forward(self._h, 1 if return_spectrogram else 0)

    def output_shape(self, batch, return_spectrogram=False):
        K = self.cfg.num_sources
        return (K, batch, self.stft_frames, SPEC_BINS) if return_spectrogram else (K, batch, self.T_out, 1)

    def _workspace(self, batch, device):
        import torch
        # kept while the engine lives: a captured CUDA graph (Test.test) bakes the pointer in
        key = (int(batch), str(device))
        ws = self._ws.get(key)
        if ws is None:
            ws = torch.empty((self.workspace_bytes(batch) + 3) // 4, dtype=torch.float32, device=device)
            self._ws[key] = ws
        return ws

    def forward(self, params, mix, training, out=None, return_spectrogram=False):
        """mix [B, T, 1] -> [K, B, T, 1] audio, or [K, B, n, 513] magnitudes with return_spectrogram.  Inference only."""
        import torch
        if training:
            raise NotImplementedError("the spectrogram U-Net runs in inference mode only (training=False)")
        B = int(mix.shape[0])
        assert mix.is_cuda and mix.dtype == torch.float32 and mix.is_contiguous(), "mix must be a contiguous float32 CUDA tensor"
        assert tuple(mix.shape[1:]) == (self.T_in, 1), ("mix shape", tuple(mix.shape), "expected [B, %d, 1]" % self.T_in)
        shape = self.output_shape(B, return_spectrogram)
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=mix.device)
        assert out.is_cuda and out.device == mix.device and out.dtype == torch.float32 and out.is_contiguous()
        assert tuple(out.shape) == shape, ("outputs", tuple(out.shape), "expected", shape)
        assert params.is_cuda and params.device == mix.device and params.dtype == torch.float32 and params.is_contiguous()
        assert params.numel() >= self.param_numel, ("flat buffer too small", params.numel(), self.param_numel)
        ws = self._workspace(B, mix.device)
        with torch.cuda.device(mix.device):
            check(lib.wun_spec_forward(self._h, params.data_ptr(), mix.data_ptr(), B, 1 if return_spectrogram else 0,
                                       out.data_ptr(), ws.data_ptr(), ws.numel() * 4, Engine._stream(mix.device)))
        return out

    def l1_batch_loss(self, est_mags, targets, state, batch_loss=None):
        """Test.test's U7a loss and running mean (wun_spec_l1_batch_loss): est_mags [K, B, n, 513] from forward(...,
        return_spectrogram=True), targets [K, B, T, 1] audio, state float64 [2] {total, n} updated in place."""
        import torch
        B = int(targets.shape[1])
        assert tuple(est_mags.shape) == self.output_shape(B, True) and est_mags.is_contiguous(), "est_mags shape"
        assert tuple(targets.shape) == self.output_shape(B, False) and targets.is_contiguous(), "targets shape"
        assert targets.dtype == torch.float32 and est_mags.dtype == torch.float32
        assert state.dtype == torch.float64 and state.numel() == 2 and state.is_cuda
        assert batch_loss is None or (batch_loss.dtype == torch.float64 and batch_loss.is_cuda)
        ws = self._workspace(B, targets.device)
        with torch.cuda.device(targets.device):
            check(lib.wun_spec_l1_batch_loss(self._h, est_mags.data_ptr(), targets.data_ptr(), B, state.data_ptr(),
                                             batch_loss.data_ptr() if batch_loss is not None else None, ws.data_ptr(),
                                             ws.numel() * 4, Engine._stream(targets.device)))

    def forward_backward(self, params, mix, targets, grads, loss, raw_audio_loss, seed, step_state, shard=None):
        """One training step's loss and gradients (wun_spec_forward_backward): mix [B, T, 1], targets [K, B, T, 1], grads
        float32 [param_numel], loss float64 [1], step_state int64 [1] (the dropout counter, advanced by one).  Updates the
        moving statistics inside `params`.
        shard (optional, e.g. wun.parallel.BatchStatsGather): this call is one rank's shard of a data-parallel step
        (wun_spec_forward_backward_dp).  It has rank, world, global_batch and sample_offset, and
        gather(local, gathered, stream) that puts every rank's float64 CUDA tensor `local` [count] into `gathered`
        [world * count] in rank order, only enqueueing work on the torch stream `stream`."""
        import torch
        B = int(mix.shape[0])
        assert mix.is_cuda and mix.dtype == torch.float32 and mix.is_contiguous(), "mix must be a contiguous float32 CUDA tensor"
        assert tuple(mix.shape[1:]) == (self.T_in, 1), ("mix shape", tuple(mix.shape), "expected [B, %d, 1]" % self.T_in)
        assert tuple(targets.shape) == self.output_shape(B) and targets.is_contiguous() and targets.dtype == torch.float32
        for t in (params, grads):
            assert t.is_cuda and t.device == mix.device and t.dtype == torch.float32 and t.is_contiguous()
            assert t.numel() >= self.param_numel, ("flat buffer too small", t.numel(), self.param_numel)
        assert loss.is_cuda and loss.dtype == torch.float64 and step_state.is_cuda and step_state.dtype == torch.int64
        key = (B, str(mix.device))
        ws = self._train_ws.get(key)        # kept while the engine lives: a captured CUDA graph bakes the pointer in
        if ws is None:
            ws = torch.empty((self.train_workspace_bytes(B) + 7) // 8 * 2, dtype=torch.float32, device=mix.device)
            self._train_ws[key] = ws
        args = (self._h, params.data_ptr(), mix.data_ptr(), targets.data_ptr(), B, 1 if raw_audio_loss else 0,
                int(seed) & (2 ** 64 - 1), step_state.data_ptr(), grads.data_ptr(), loss.data_ptr(), ws.data_ptr(),
                ws.numel() * 4, Engine._stream(mix.device))
        with torch.cuda.device(mix.device):
            if shard is None:
                check(lib.wun_spec_forward_backward(*args))
                return loss
            desc, errors, keep = self._shard_descriptor(shard, ws, mix.device)
            rc = lib.wun_spec_forward_backward_dp(*(args + (ctypes.byref(desc),)))     # `keep` holds the callback
            if errors:
                raise errors[0]
            check(rc)
        return loss

    def _shard_descriptor(self, shard, ws, device):
        """WunSpecShard for `shard`, with a gather callback that hands shard.gather torch views of the engine's buffers.
        Returns (descriptor, the list that receives the callback's exception, the objects to keep alive for the call)."""
        import torch
        world = int(shard.world)
        key = (world, str(device))
        gathered = self._gathered.get(key)  # kept like the workspace: a captured graph bakes the pointer in
        if gathered is None:
            widest = self.cfg.num_initial_filters << (self.cfg.num_layers - 1)
            gathered = torch.empty(world * 2 * widest, dtype=torch.float64, device=device)
            self._gathered[key] = gathered
        ws64 = ws.view(torch.float64)
        errors = []

        def gather(ctx, local, out, count, stream):
            try:
                lo, go = (local - ws64.data_ptr()) // 8, (out - gathered.data_ptr()) // 8
                shard.gather(ws64[lo:lo + count], gathered[go:go + world * count], torch.cuda.current_stream(device))
                return 0
            except BaseException as e:       # an exception cannot cross the C frames: re-raised after the call
                errors.append(e)
                return 1

        fn = SPEC_GATHER_FN(gather)
        desc = WunSpecShard(int(shard.rank), world, int(shard.global_batch), int(shard.sample_offset), gathered.data_ptr(),
                            gathered.numel() * 8, fn, None)
        return desc, errors, (fn, gather)

    def debug_train_level(self, batch, level, device):
        """Tests: view of concatenation level `level` [B, H, W, C] in the training workspace - after forward_backward the
        last source's down (LeakyReLU) and up (ReLU) activations."""
        off, n = ctypes.c_int64(), ctypes.c_int64()
        check(lib.wun_spec_debug_train_level(self._h, int(batch), int(level), ctypes.byref(off), ctypes.byref(n)))
        ws = self._train_ws[(int(batch), str(device))]
        H, W = self.stft_frames >> (level + 1), 512 >> (level + 1)
        return ws[off.value // 4:off.value // 4 + n.value].view(int(batch), H, W, -1)

    def debug_train_keep(self, batch, level, device):
        """Tests: the keep mask of dropped level `level` [B, H, W, C] uint8 in the training workspace (after forward_backward
        the last source's)."""
        import torch
        off, n = self._debug_train_buffer(batch, 0, level)
        ws = self._train_ws[(int(batch), str(device))]
        H, W = self.stft_frames >> (level + 1), 512 >> (level + 1)
        return ws.view(torch.uint8)[off:off + n].view(int(batch), H, W, -1)

    def debug_train_stats(self, batch, layer, up, device):
        """Tests: the batch statistics [C, 2] (mean, rstd) of down (or with `up`, up) layer `layer` in the training
        workspace (after forward_backward the last source's)."""
        off, n = self._debug_train_buffer(batch, 2 if up else 1, layer)
        ws = self._train_ws[(int(batch), str(device))]
        return ws[off // 4:off // 4 + n].view(-1, 2)

    def _debug_train_buffer(self, batch, what, index):
        off, n = ctypes.c_int64(), ctypes.c_int64()
        check(lib.wun_spec_debug_train_buffer(self._h, int(batch), int(what), int(index), ctypes.byref(off), ctypes.byref(n)))
        return off.value, n.value

    def adam_step_device(self, params, grads, m, v, state, lr, beta1=0.9, beta2=0.999, eps=1e-8):
        """Graph-safe Adam on the trainable variables: `state` = device float32[3] {beta1_power, beta2_power, step}."""
        import torch
        with torch.cuda.device(params.device):
            check(lib.wun_spec_adam_step_device(self._h, params.data_ptr(), grads.data_ptr(), m.data_ptr(), v.data_ptr(),
                                                state.data_ptr(), float(lr), float(beta1), float(beta2), float(eps),
                                                Engine._stream(params.device)))

    def feed_batch(self, pool, track_offset, track_length, batch, augmentation, seed, step_state, mix_out, targets_out,
                   chosen=None):
        """Engine.feed_batch for this window (wun_spec_feed_batch): T_in = T_out = T, one channel."""
        import torch
        K = targets_out.shape[0]
        assert K == self.cfg.num_sources and pool.shape[2] == 1
        assert pool.is_cuda and pool.dtype == torch.float32 and pool.is_contiguous() and pool.dim() == 3 and pool.shape[0] == K + 1
        assert track_offset.dtype == torch.int64 and track_length.dtype == torch.int64 and step_state.dtype == torch.int64
        assert tuple(mix_out.shape) == (batch, self.T_in, 1) and mix_out.is_contiguous()
        assert tuple(targets_out.shape) == (K, batch, self.T_out, 1) and targets_out.is_contiguous()
        with torch.cuda.device(mix_out.device):
            check(lib.wun_spec_feed_batch(self._h, pool.data_ptr(), pool.shape[1], track_offset.data_ptr(),
                                          track_length.data_ptr(), track_offset.numel(), int(batch), int(bool(augmentation)),
                                          int(seed) & (2 ** 64 - 1), step_state.data_ptr(), mix_out.data_ptr(),
                                          targets_out.data_ptr(), chosen.data_ptr() if chosen is not None else None,
                                          Engine._stream(mix_out.device)))

    def gather_windows(self, padded, starts, mix_batch):
        check(lib.wun_spec_gather_windows(self._h, padded.data_ptr(), padded.shape[0], starts.data_ptr(),
                                          starts.numel(), mix_batch.data_ptr(), Engine._stream(padded.device)))

    def scatter_windows(self, outputs, starts, preds):
        check(lib.wun_spec_scatter_windows(self._h, outputs.data_ptr(), starts.data_ptr(), starts.numel(),
                                           preds.data_ptr(), preds.shape[1], Engine._stream(preds.device)))
