"""What the launch-by-launch GPU suites (tests/test_kernels_gpu.py, test_step_kernels_gpu.py, test_wgrad_tiles.py and
test_configurations_gpu.py) share: the sentinel and guard words, the float-regime bounds, the per-family report, the element
checks, guarded device buffers, the harness library (tests/kernels) and the engine of a configuration."""
import os
import sys
from collections import defaultdict

import numpy as np
import pytest
import torch

import Config
import wun
from oracle import wave_unet_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernels"))
import harness as H  # noqa: E402

SENTINEL = np.float32(7.0e30)
GUARD = 64
U32 = 2.0 ** -24                     # unit roundoff of fp32
# Bounds of the float regime, |got - ref| <= bound * ref_abs.  The tensor-core conv, dgrad and wgrad (3-MMA split): ~3 * 2^-17
# per product; fp32 accumulation over the launch's k16 steps on top.  Worst err / ref_abs measured on one H100 80GB HBM3 (700 W
# power limit): 2.5e-5 (replayed wgrad), 2.4e-5 (synthetic wgmma conv) - 5x below the bound.
TAU = 2.0 ** -13
# The other kernels (recursive summation: error <= depth * u * sum |terms|, depth = longest chain of fp32 additions):
TAU_FIRST = 2.0 ** -16               # forward: <= 16 taps x 2 channels + bias = 33-term sums
TAU_RED = 2.0 ** -13                 # weight / interp gradients: per-thread rows + 8 or 16 groups + <= 528 + batch CTA sums (~2^-14.8)
TAU_OUT = 2.0 ** -16                 # output conv: ofs * (C + F) + 1 terms (<= 3 * 34); dgrad <= ofs * 16 terms
TAU_UP = 2.0 ** -20                  # upsampling gradient: 4 terms and the slope
# kernel family -> its bound: the first key the family's name contains (sigmoid and Adam are ulp-bounded and have none)
BOUNDS = {"first fwd": TAU_FIRST, "first wgrad": TAU_RED, "output fwd": TAU_OUT, "output dgrad": TAU_OUT, "output wgrad": TAU_RED,
          "upsample bwd": TAU_UP, "fwd": TAU, "dgrad": TAU, "wgrad": TAU}
WORST = defaultdict(float)          # kernel family -> worst err / ref_abs of the float regime
COUNTS = defaultdict(int)           # kernel family -> cases run
EXACT = defaultdict(int)            # kernel family -> exact-regime cases that matched bit for bit


def print_report(title, prefix="", required=()):
    """Prints a row per kernel family whose name starts with `prefix`: the cases run, the exact-regime matches, the worst
    err / ref_abs of the float regime (err / bound for the ulp-bounded families) and the bound.  Each `required` family must
    have run."""
    print("\n%-44s %6s %6s %10s %10s" % (title, "cases", "exact", "worst", "bound"))
    for fam in sorted(f for f in COUNTS if f.startswith(prefix)):
        w = WORST.get(fam, WORST.get(fam + " (err/bound)"))
        bound = next((b for k, b in BOUNDS.items() if k in fam), None)
        print("%-44s %6d %6s %10s %10s" % (fam, COUNTS[fam], EXACT.get(fam, "-"), "-" if w is None else "%.2e" % w,
                                          "-" if w is None else "ulp" if bound is None else "%.2e" % bound))
    for fam in required:
        assert COUNTS.get(fam, 0) > 0, fam


def check(family, got, ref, tol, what, ref_abs=None):
    """|got - ref| <= tol everywhere (torch tensors on any device, ref in float64).  The report keeps the worst err / ref_abs,
    or without ref_abs (ulp-bounded families) the worst err / tol as "family (err/bound)"."""
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError("%s: %d of %d elements beyond the bound; first: got %r ref %r tol %r" % (
            what, int(bad.sum()), bad.numel(), float(got.reshape(-1)[i]), float(ref.reshape(-1)[i]), float(tol.reshape(-1)[i])))
    scale, key = (ref_abs, family) if ref_abs is not None else (tol, family + " (err/bound)")
    nz = scale > 0
    if bool(nz.any()):
        WORST[key] = max(WORST[key], float((err[nz] / scale[nz]).max()))


def exact_eq(family, got, ref32, what):
    same = got.view(torch.int32) == ref32.view(torch.int32)
    if not bool(same.all()):
        i = int(torch.nonzero(~same.reshape(-1))[0])
        raise AssertionError("%s (%s): %d of %d differ; first got %r want %r" % (what, family, int((~same).sum()), same.numel(),
                                                                                float(got.reshape(-1)[i]), float(ref32.reshape(-1)[i])))


def f32_exact(x64, what):
    """Exact regime: a float64 value the kernel computes in fp32 must be representable (no rounding anywhere)."""
    assert bool((x64.float().double() == x64).all()), "%s: the exact regime left fp32 - shrink the case" % what
    return x64.float()


class Mem(object):
    """Named float32 device buffers, each framed by GUARD sentinel words.  ptr(name) = the first data word (0 for None)."""

    def __init__(self):
        self.t = {}

    def add(self, name, data):
        data = data.reshape(-1).float()
        full = torch.full((data.numel() + 2 * GUARD,), float(SENTINEL), device="cuda")
        full[GUARD:GUARD + data.numel()] = data
        self.t[name] = full
        return full[GUARD:GUARD + data.numel()]

    def arena(self, name, nbytes):
        """A partial-sum arena of exactly nbytes, NaN-filled, guard after it."""
        assert nbytes % 4 == 0
        return self.add(name, torch.full((nbytes // 4,), float("nan"), device="cuda"))

    def ptr(self, name):
        return 0 if name is None else self.t[name].data_ptr() + 4 * GUARD

    def d(self, name):
        return self.t[name][GUARD:self.t[name].numel() - GUARD]

    def snapshot(self):
        return {k: v.clone() for k, v in self.t.items()}

    def restore(self, snap):
        for k, v in snap.items():
            self.t[k].copy_(v)

    def check_rest(self, before, outs, what):
        """Every word outside the outputs (outs: name -> bool mask over the data words) keeps its bits, guards included."""
        for k, full in self.t.items():
            keep = torch.ones(full.numel(), dtype=torch.bool, device="cuda")
            if k in outs:
                keep[GUARD:GUARD + outs[k].numel()] = ~outs[k].reshape(-1)
            same = full.view(torch.int32)[keep] == before[k].view(torch.int32)[keep]
            assert bool(same.all()), "%s: %d words of %s outside the outputs changed" % (what, int((~same).sum()), k)


def stream():
    return torch.cuda.current_stream().cuda_stream


def gpu_lib():
    assert torch.cuda.is_available()
    assert os.path.exists(H.LIB) or os.path.exists(H.NVCC), "tests/kernels/_build/libwun_kernels.so is missing and there is no nvcc"
    lib = H.load()
    assert hasattr(lib, "wkh_upsample_bwd"), "libwun_kernels.so predates the step-kernel entry points"
    return lib


def lib_or_skip():
    if H.stale() and not os.path.exists(H.NVCC):
        pytest.skip("no nvcc to build tests/kernels")
    return H.load()


def set_env(monkeypatch, env):
    """Only the WUN_ switches of `env` are set for the test."""
    for k in [k for k in os.environ if k.startswith("WUN_")]:
        monkeypatch.delenv(k)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def engine(named, ov, batch, nf):
    """-> (model config, input frames, engine, conv launch descriptions) of a training step at `batch` (host only); the engine's
    wgrad_groups and step_launches are then those of that batch.  nf None: the preset's num_frames."""
    cfg = Config.build_config(named, ov, experiment_id=0)["model_config"]
    t_in, _ = O.get_padding(cfg, nf or cfg["num_frames"])
    eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
    return cfg, t_in, eng, eng.launch_descriptions(batch)
