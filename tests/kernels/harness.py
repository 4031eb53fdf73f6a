"""Per-launch kernel harness (TEST INFRASTRUCTURE): libwun_kernels.so = tests/kernels/harness.cu linked with the product's kernel
sources, built under tests/kernels/_build/ (git-ignored).  It replays ONE plane-convolution launch or ONE layer's weight gradient,
described in the text format wun_debug_launches writes, through the product's planner and launchers (tests/test_kernels_gpu.py).

build()        - compiles the library (None without nvcc); rebuilt when a source is newer than it.
load()         - the ctypes handle (builds first when stale and nvcc exists).
conv_text()    - a launch dict of wun.Engine.launch_descriptions (or a synthetic one) -> the description text.
wgrad_text()   - a layer's wgrad groups (wun.Engine.wgrad_groups entries) -> the description text.
"""
import ctypes
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(REPO, "wave-u-net_b200", "csrc")
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(BUILD, "libwun_kernels.so")
# WUN_KERNELS_LIB: run the tests against another build of the harness (e.g. one made from modified kernel sources)
OVERRIDE = os.environ.get("WUN_KERNELS_LIB")
SOURCES = [os.path.join(HERE, "harness.cu"), os.path.join(CSRC, "kernels_umma.cu"), os.path.join(CSRC, "kernels_simt.cu"),
           os.path.join(CSRC, "kernels_first.cu")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _deps():
    return SOURCES + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".h")]


def stale(path=LIB):
    if not os.path.exists(path):
        return True
    t = os.path.getmtime(path)
    return any(os.path.getmtime(d) > t for d in _deps())


def build():
    """Returns the library path, or None when there is no nvcc.  The kernels are compiled exactly as build.sh compiles them."""
    if not os.path.exists(NVCC):
        return None
    if stale():
        os.makedirs(BUILD, exist_ok=True)
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-diag-suppress",
                               "177", "-Xcompiler", "-fPIC", "-shared", "-I", CSRC, "-o", LIB] + SOURCES)
    return LIB


_lib = None


def load():
    global _lib
    if _lib is None:
        if OVERRIDE:
            _lib = _bind(ctypes.CDLL(OVERRIDE))
            return _lib
        if stale() and os.path.exists(NVCC):
            try:
                build()
            except OSError:                          # read-only checkout: use what __graft_entry__.build() left
                pass
        _lib = _bind(ctypes.CDLL(LIB))
    return _lib


def _bind(lib):
    P, I64, S = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_char_p
    lib.wkh_last_error.restype = S
    lib.wkh_plan_conv.argtypes = [S, ctypes.POINTER(I64)]
    lib.wkh_plan_wgrad.argtypes = [S, ctypes.POINTER(I64), ctypes.c_int]
    lib.wkh_run_conv.argtypes = [S, P, P, P, ctypes.c_int, P, I64, P]
    lib.wkh_run_wgrad.argtypes = [S, P, P, P, P, ctypes.c_float, ctypes.c_int, P, I64, P]
    lib.wkh_conv_steps.argtypes = [S, ctypes.POINTER(I64), I64]
    for f in (lib.wkh_plan_conv, lib.wkh_plan_wgrad, lib.wkh_run_conv, lib.wkh_run_wgrad, lib.wkh_conv_steps):
        f.restype = ctypes.c_int
    G, F, I = ctypes.POINTER(I64), ctypes.c_float, ctypes.c_int
    sig = {
        "wkh_first_partial_bytes": (I64, [I]), "wkh_first_supported": (I, [I, I, I]),
        "wkh_first_fwd": (I, [G, P, P, P, P, P, P]), "wkh_first_wgrad": (I, [G, P, P, P, P, P, F, P, I64, P]),
        "wkh_output_partial_bytes": (I, [G, G]), "wkh_output_fwd": (I, [G, F, P, P, P, P, P, P, P, P, I64, P, P]),
        "wkh_output_dgrad": (I, [G, P, P, P, P, P]), "wkh_output_wgrad": (I, [G, P, P, P, P, P, F, P, I64, P]),
        "wkh_upsample_partial_bytes": (I64, [I, I]), "wkh_upsample_bwd": (I, [G, P, P, P, P, P, P, F, P, I64, P, P]),
        "wkh_sigmoid": (I, [P, P, I, P]), "wkh_adam": (I, [P, P, P, P, I64, F, F, F, F, P, P]),
        "wkh_gather_windows": (I, [P, I64, P, I, I, I, P, P]), "wkh_scatter_windows": (I, [P, P, I, I, I, I, P, I64, P]),
    }
    for name, (res, args) in sig.items():
        if hasattr(lib, name):                   # (a harness built from older sources lacks them: the step-kernel tests fail by name)
            getattr(lib, name).restype = res
            getattr(lib, name).argtypes = args
    return lib


def geom(values):
    """A list of integers -> the int64 array the step-kernel entry points take as geometry."""
    return (ctypes.c_longlong * len(values))(*[int(v) for v in values])


FIRST_KEYS = ["C", "N", "k", "pad_left", "batch", "x_bstride", "T", "dec_bstride", "Td", "odd_bstride", "mo_lo", "mo_hi"]
OUTPUT_KEYS = ["batch", "T_in", "Tf", "T_out", "C", "F", "nconv", "K", "ofs", "pad_left", "crop_feat", "crop_out", "output_type",
               "activation", "training"]
UPSAMPLE_KEYS = ["batch", "N", "nmid", "C", "mid_mode"]


def first_geom(d):
    return geom([d[k] for k in FIRST_KEYS])


def output_geom(d):
    return geom([d[k] for k in OUTPUT_KEYS] + [d["w_off%d" % s] for s in range(8)] + [d["b_off%d" % s] for s in range(8)])


def upsample_geom(d):
    return geom([d[k] for k in UPSAMPLE_KEYS])


def output_partial_bytes(d):
    """-> (output_wgrad_partial_bytes, output_loss_partial_bytes) of an output-layer geometry."""
    out = (ctypes.c_longlong * 2)()
    _check(load().wkh_output_partial_bytes(output_geom(d), out), "wkh_output_partial_bytes")
    return int(out[0]), int(out[1])


def call(name, *args):
    """Runs one step-kernel entry point (wkh_<name>); raises on a malformed call or a CUDA error."""
    _check(getattr(load(), "wkh_" + name)(*args), "wkh_" + name)


CONV_KEYS = {
    "launch": ["layer", "pass", "N", "pairC", "w_sk", "w_sn", "W", "bias", "epilogue", "batch", "nplanes", "ncls"],
    "plane": ["i", "base", "bstride", "rstride", "r_lo", "r_hi", "C", "kind", "mid_mode", "xrows", "blend"],
    "cls": ["i", "base", "bstride", "rstride", "m_lo", "m_hi", "saved", "acc_lo", "acc_hi", "term_begin", "term_end", "pairC", "base2",
            "bstride2", "rstride2", "saved2", "acc_lo2", "acc_hi2", "lo0", "hi0", "lo1", "hi1"],
    "term": ["i", "plane", "d", "woff", "woff2"],
}
WGRAD_KEYS = {
    "wgrad": ["layer", "group", "N", "w_sk", "w_sn", "dW", "db", "m_lo", "m_hi", "nterms", "batch"],
    "wplane": CONV_KEYS["plane"][1:],
    "wterm": ["i", "d", "woff"],
}


def _line(kind, d, keys):
    return kind + " " + " ".join("%s=%d" % (k, d[k]) for k in keys)


def conv_text(D):
    out = [_line("launch", D["launch"], CONV_KEYS["launch"])]
    out += [_line("plane", dict(P, i=k), CONV_KEYS["plane"]) for k, P in enumerate(D["planes"])]
    out += [_line("cls", dict(q, i=k), CONV_KEYS["cls"]) for k, q in enumerate(D["cls"])]
    out += [_line("term", dict(t, i=k), CONV_KEYS["term"]) for k, t in enumerate(D["terms"])]
    return "\n".join(out) + "\n"


def wgrad_text(groups):
    out = []
    for G in groups:
        out.append(_line("wgrad", G["wgrad"], WGRAD_KEYS["wgrad"]))
        out.append(_line("wplane", G["plane"], WGRAD_KEYS["wplane"]))
        out.append(_line("wdpre", G["dpre"], WGRAD_KEYS["wplane"]))
        out += [_line("wterm", t, WGRAD_KEYS["wterm"]) for t in G["terms"]]
    return "\n".join(out) + "\n"


def _check(rc, what):
    if rc != 0:
        raise RuntimeError("%s: %s" % (what, load().wkh_last_error().decode() if rc == -1 else "CUDA error %d" % rc))


def plan_conv(text):
    """-> dict(eligible, NPAD, nsplit, MT, rows_alloc, TB, nbs, pack_bytes) (host only)."""
    out = (ctypes.c_longlong * 8)()
    _check(load().wkh_plan_conv(text.encode(), out), "wkh_plan_conv")
    return dict(zip(["eligible", "NPAD", "nsplit", "MT", "rows_alloc", "TB", "nbs", "pack_bytes"], list(out)))


def conv_steps(text):
    """-> dict(TB, nbs, cls=[dict(ngroups, tiles=[[(g, c, t0, nt, blk) per K step] per row tile])]): the steps the tensor-core
    conv walks, from the product's own next_step (host only)."""
    cap = 1 << 20
    out = (ctypes.c_longlong * cap)()
    n = load().wkh_conv_steps(text.encode(), out, cap)
    _check(0 if n >= 0 else -1, "wkh_conv_steps")
    v = list(out[:n])
    r = dict(TB=v[0], nbs=v[1], cls=[])
    i = 3
    for _ in range(v[2]):
        q = dict(ngroups=v[i], tiles=[])
        ntiles = v[i + 1]
        i += 2
        for _ in range(ntiles):
            k = v[i]
            q["tiles"].append([tuple(v[i + 1 + 5 * j:i + 6 + 5 * j]) for j in range(k)])
            i += 1 + 5 * k
        r["cls"].append(q)
    return r


GROUP_KEYS = ["swap", "NT", "n_mtiles", "n_ntiles", "taps_per_cta", "n_tapsets", "chunks_per_batch", "chunks_per_cta", "n_ctas_x", "slot0"]


def plan_wgrad(text):
    """-> dict(eligible, bulk, split_bytes, partial_bytes, ngroups, grid, nstages, arena_bytes, groups=[{GROUP_KEYS}]) (host only)."""
    n = 10 + 10 * 8
    out = (ctypes.c_longlong * n)()
    _check(load().wkh_plan_wgrad(text.encode(), out, n), "wkh_plan_wgrad")
    v = list(out)
    r = dict(eligible=v[0], bulk=v[1], split_bytes=v[2], partial_bytes=v[3], ngroups=v[4], grid=tuple(v[5:8]), nstages=v[8],
             arena_bytes=v[9])
    r["groups"] = [dict(zip(GROUP_KEYS, v[10 + 10 * g:20 + 10 * g])) for g in range(v[4])] if v[0] else []
    return r


def run_conv(text, ws, par, mix, kernel, arena, arena_bytes, stream):
    _check(load().wkh_run_conv(text.encode(), ws, par, mix, kernel, arena, arena_bytes, stream), "wkh_run_conv")


def run_wgrad(text, ws, par, mix, grads, scale, mode, arena, arena_bytes, stream):
    _check(load().wkh_run_wgrad(text.encode(), ws, par, mix, grads, scale, mode, arena, arena_bytes, stream), "wkh_run_wgrad")
