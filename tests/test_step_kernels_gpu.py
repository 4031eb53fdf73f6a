"""The rest of a training step, launch by launch, against float64: the first-layer forward and weight gradient (kernels_first.cu),
the output layer's forward (estimates, difference output, clip, loss, dL/dpre), dgrad and weight gradient, the upsampling backward
with the interp gradient, sigmoid, Adam and the window gather / scatter of prediction (kernels_simt.cu).

Each launch runs alone through tests/kernels/harness.cu (the product's own launchers) on buffers framed by GUARD sentinel words;
words the launch contract says are never read (gaps of wide batch strides, partial-sum arenas before they are written) hold NaN.
Every word outside a launch's outputs must keep its bits, gradients are pre-filled (the contract is +=), the partial-sum arenas
are exactly as long as the product's size functions say and followed by a guard, and every reduction runs twice with the same
bits.  The regimes and the report are those of tests/test_kernels_gpu.py:
  exact - activations k/4 in [-4, 4], weights integers in [-3, 3], blend weights in {1/4, 1/2, 3/4}, power-of-two scales and
          inv_count: every sum is exact in fp32 (checked per case), so the result must equal float64 bit for bit, with the fp32
          epilogues applied in the kernels' order.
  float - random data over a wide dynamic range: |got - ref| <= TAU * ref_abs (+ a stated ulp allowance for tanhf / expf /
          sqrtf and division), ref_abs the same computation on |x| and |w|.  A power check per family shows TAU flags one
          dropped item of the kind that family can lose.
Replays run every first / output / upsample / adam launch the engine emits for the configurations of test_kernels_gpu.REPLAYS
and M5 at batch 16, on random buffers of the exported geometry.
"""
import os
import sys

import numpy as np
import pytest

import Config
import wun
from oracle import wave_unet_oracle as O
import test_kernels_gpu as K

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernels"))
import harness as H  # noqa: E402

SENTINEL, GUARD, WORST, COUNTS, EXACT = K.SENTINEL, K.GUARD, K.WORST, K.COUNTS, K.EXACT
U32 = 2.0 ** -24                     # unit roundoff of fp32
# Bounds of the float regime (recursive summation: error <= depth * u * sum |terms|, depth = longest chain of fp32 additions):
TAU_FIRST = 2.0 ** -16               # forward: <= 16 taps x 2 channels + bias = 33-term sums
TAU_RED = 2.0 ** -13                 # weight / interp gradients: per-thread rows + 8 or 16 groups + <= 528 + batch CTA sums (~2^-14.8)
TAU_OUT = 2.0 ** -16                 # output conv: ofs * (C + F) + 1 terms (<= 3 * 34); dgrad <= ofs * 16 terms
TAU_UP = 2.0 ** -20                  # upsampling gradient: 4 terms and the slope


def _torch():
    import torch
    return torch


def _gpu_lib():
    torch = _torch()
    assert torch.cuda.is_available()
    lib = H.load()
    assert hasattr(lib, "wkh_upsample_bwd"), "libwun_kernels.so predates the step-kernel entry points"
    return lib


# ------------------------------------------------------------------------------------------------
# guarded device buffers
# ------------------------------------------------------------------------------------------------
class Mem(object):
    """Named float32 device buffers, each framed by GUARD sentinel words.  ptr(name) = the first data word (0 for None)."""

    def __init__(self):
        self.t = {}

    def add(self, name, data):
        torch = _torch()
        data = data.reshape(-1).float()
        full = torch.full((data.numel() + 2 * GUARD,), float(SENTINEL), device="cuda")
        full[GUARD:GUARD + data.numel()] = data
        self.t[name] = full
        return full[GUARD:GUARD + data.numel()]

    def arena(self, name, nbytes):
        """A partial-sum arena of exactly nbytes, NaN-filled, guard after it."""
        torch = _torch()
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
        torch = _torch()
        for k, full in self.t.items():
            keep = torch.ones(full.numel(), dtype=torch.bool, device="cuda")
            if k in outs:
                keep[GUARD:GUARD + outs[k].numel()] = ~outs[k].reshape(-1)
            same = full.view(torch.int32)[keep] == before[k].view(torch.int32)[keep]
            assert bool(same.all()), "%s: %d words of %s outside the outputs changed" % (what, int((~same).sum()), k)


def data(gen, n, regime, kind="act"):
    torch = _torch()
    if regime == "exact":
        if kind == "w":
            return torch.randint(-3, 4, (n,), generator=gen, device="cuda").float()
        if kind == "blend":
            return torch.tensor([0.25, 0.5, 0.75], device="cuda")[torch.randint(0, 3, (n,), generator=gen, device="cuda")]
        return torch.randint(-16, 17, (n,), generator=gen, device="cuda").float() / 4
    if kind == "blend":
        return torch.rand(n, generator=gen, device="cuda")
    return torch.randn(n, generator=gen, device="cuda") * torch.exp2(torch.rand(n, generator=gen, device="cuda") * 12 - 6)


def f32_exact(x64, what):
    """Exact regime: a float64 value the kernel computes in fp32 must be representable (no rounding anywhere)."""
    assert bool((x64.float().double() == x64).all()), "%s: the exact regime left fp32 - shrink the case" % what
    return x64.float()


def check(family, got, ref, tol, what, ref_abs=None):
    """|got - ref| <= tol everywhere.  The report keeps the worst err / ref_abs, or without ref_abs (ulp-bounded families) the
    worst err / tol as "family (err/bound)"."""
    torch = _torch()
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
    torch = _torch()
    same = got.view(torch.int32) == ref32.view(torch.int32)
    if not bool(same.all()):
        i = int(torch.nonzero(~same.reshape(-1))[0])
        raise AssertionError("%s (%s): %d of %d differ; first got %r want %r" % (what, family, int((~same).sum()), same.numel(),
                                                                                float(got.reshape(-1)[i]), float(ref32.reshape(-1)[i])))


def lrelu32(y32):
    return _torch().maximum(y32 * np.float32(0.2), y32)


def slope(x):
    return _torch().where(x > 0, 1.0, 0.2).to(x.dtype)


def stream():
    return _torch().cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------
# first layer
# ------------------------------------------------------------------------------------------------
def first_gather(G, X, q):
    """X [B, T, C] float64 -> the window of every row of class q: [B, M, k, C] (zero outside [0, T))."""
    torch = _torch()
    lo, hi = (0, G["Td"]) if q == 0 else (G["mo_lo"], G["mo_hi"])
    m = torch.arange(lo, hi, device="cuda")
    t = 2 * m[:, None] + q + torch.arange(G["k"], device="cuda")[None, :] - G["pad_left"]
    ok = (t >= 0) & (t < G["T"])
    return X[:, t.clamp(0, G["T"] - 1), :] * ok[None, :, :, None]


def first_views(G, mem, names):
    B, C, N = G["batch"], G["C"], G["N"]
    x = mem.d(names[0]).view(B, G["x_bstride"])[:, :G["T"] * C].view(B, G["T"], C)
    dec = mem.d(names[1]).view(B, G["dec_bstride"])[:, :G["Td"] * N].view(B, G["Td"], N)
    no = G["mo_hi"] - G["mo_lo"]
    odd = mem.d(names[2]).view(B, G["odd_bstride"])[:, :no * N].view(B, no, N)
    return x, dec, odd


def first_masks(G, mem, names):
    torch = _torch()
    out = {}
    for nm, bst, rows in ((names[1], G["dec_bstride"], G["Td"]), (names[2], G["odd_bstride"], G["mo_hi"] - G["mo_lo"])):
        msk = torch.zeros(G["batch"], bst, dtype=torch.bool, device="cuda")
        msk[:, :rows * G["N"]] = True
        out[nm] = msk
    return out


def first_memory(G, gen, regime, with_grads):
    """x (batch stride = x_bstride, NaN past T*C), W, bias, the forward outputs (sentinel: written) and for the weight gradient
    the gradient tensors g_dec / g_odd (NaN in their stride gaps), dW / db pre-filled."""
    torch = _torch()
    B, C, N, k = G["batch"], G["C"], G["N"], G["k"]
    mem = Mem()
    x = torch.full((B, G["x_bstride"]), float("nan"), device="cuda")
    x[:, :G["T"] * C] = data(gen, B * G["T"] * C, regime).view(B, -1)
    mem.add("x", x)
    mem.add("W", data(gen, k * C * N, regime, "w"))
    mem.add("bias", data(gen, N, regime))
    no = G["mo_hi"] - G["mo_lo"]
    for nm, bst, rows in (("dec", G["dec_bstride"], G["Td"]), ("odd", G["odd_bstride"], no)):
        if with_grads:
            g = torch.full((B, bst), float("nan"), device="cuda")
            g[:, :rows * N] = data(gen, B * rows * N, regime).view(B, -1)
            mem.add(nm, g)
        else:
            mem.add(nm, torch.full((B * bst,), float(SENTINEL), device="cuda"))
    if with_grads:
        mem.add("dW", data(gen, k * C * N, regime))
        mem.add("db", data(gen, N, regime))
    return mem


def run_first_fwd(G, regime, seed, family="first fwd"):
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    mem = first_memory(G, gen, regime, False)
    before = mem.snapshot()
    H.call("first_fwd", H.first_geom(G), mem.ptr("x"), mem.ptr("dec"), mem.ptr("odd"), mem.ptr("W"), mem.ptr("bias"), stream())
    torch.cuda.synchronize()
    mem.check_rest(before, first_masks(G, mem, ("x", "dec", "odd")), "first fwd %s" % G.get("name"))
    x, dec, odd = first_views(G, mem, ("x", "dec", "odd"))
    W = mem.d("W").double().view(G["k"], G["C"], G["N"])
    b = mem.d("bias").double()
    for q, got in ((0, dec), (1, odd)):
        Xg = first_gather(G, x.double(), q)
        pre = torch.einsum("bmjc,jcn->bmn", Xg, W) + b
        if regime == "exact":
            exact_eq(family, got, lrelu32(f32_exact(pre, "first fwd")), "first fwd %s class %d" % (G.get("name"), q))
        else:
            pre_abs = torch.einsum("bmjc,jcn->bmn", Xg.abs(), W.abs()) + b.abs()
            ref = torch.maximum(0.2 * pre, pre)
            check(family, got, ref, TAU_FIRST * pre_abs + U32 * ref.abs(), "first fwd %s class %d" % (G.get("name"), q), pre_abs)
            if q == 0:      # power: one dropped boundary tap (the last tap of the first row of a tile) is above the bound
                j = G["k"] - 1
                c = 0.2 * (Xg[:, 0, j, :, None] * W[j][None]).sum(1).abs()
                assert bool((c > TAU_FIRST * pre_abs[:, 0] + U32 * ref[:, 0].abs()).any()), "first fwd: a dropped tap is below the bound"
    if regime == "exact":
        EXACT[family] += 1
    COUNTS[family] += 1


def run_first_wgrad(G, regime, seed, scale=0.5, null_db=False, family="first wgrad"):
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    mem = first_memory(G, gen, regime, True)
    pb = int(H.load().wkh_first_partial_bytes(G["batch"]))
    mem.arena("part", pb)
    before = mem.snapshot()
    results = []
    for _ in range(2):
        mem.restore(before)
        H.call("first_wgrad", H.first_geom(G), mem.ptr("x"), mem.ptr("dec"), mem.ptr("odd"), mem.ptr("dW"),
               0 if null_db else mem.ptr("db"), scale, mem.ptr("part"), pb, stream())
        torch.cuda.synchronize()
        outs = {"dW": torch.ones_like(mem.d("dW"), dtype=torch.bool), "part": torch.ones_like(mem.d("part"), dtype=torch.bool)}
        if not null_db:
            outs["db"] = torch.ones_like(mem.d("db"), dtype=torch.bool)
        mem.check_rest(before, outs, "first wgrad %s" % G.get("name"))
        results.append((mem.d("dW").clone(), mem.d("db").clone()))
    for a, b in zip(results[0], results[1]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "first wgrad: two runs differ"
    dW, db = results[0]
    assert not bool(torch.isnan(dW).any() or torch.isnan(db).any()), "first wgrad: NaN from an unwritten partial slot"
    x, gdec, godd = first_views(G, mem, ("x", "dec", "odd"))
    s = torch.zeros(G["k"], G["C"], G["N"], dtype=torch.float64, device="cuda")
    sa, sb, sba = torch.zeros_like(s), torch.zeros(G["N"], dtype=torch.float64, device="cuda"), None
    sba = torch.zeros_like(sb)
    for q, g in ((0, gdec), (1, godd)):
        Xg = first_gather(G, x.double(), q)
        s += torch.einsum("bmjc,bmn->jcn", Xg, g.double())
        sa += torch.einsum("bmjc,bmn->jcn", Xg.abs(), g.double().abs())
        sb += g.double().sum((0, 1))
        sba += g.double().abs().sum((0, 1))
    w0, b0 = before["dW"][GUARD:-GUARD].double(), before["db"][GUARD:-GUARD].double()
    refs = [(dW, w0.view_as(s) + scale * s, scale * sa + w0.abs().view_as(s), "dW")]
    if not null_db:
        refs.append((db, b0 + scale * sb, scale * sba + b0.abs(), "db"))
    else:
        assert torch.equal(db.view(torch.int32), b0.float().view(torch.int32))
    for got, ref, rabs, nm in refs:
        got = got.view_as(ref)
        if regime == "exact":
            assert bool((rabs * 16 / min(scale, 1.0) < 2 ** 24).all()), "first wgrad: case too large for the exact regime"
            exact_eq(family, got, f32_exact(ref, "first wgrad"), "first wgrad %s %s" % (G.get("name"), nm))
        else:
            check(family, got, ref, TAU_RED * rabs, "first wgrad %s %s" % (G.get("name"), nm), rabs)
    if regime == "float":   # power: one dropped 128-row block (item 0, class 0, rows 0..127) is above the bound
        Xg = first_gather(G, x.double(), 0)
        blk = (scale * torch.einsum("bmjc,bmn->jcn", Xg[:1, :128], gdec.double()[:1, :128])).abs()
        assert bool((blk > TAU_RED * refs[0][2]).any()), "first wgrad: a dropped 128-row block is below the bound"
    if regime == "exact":
        EXACT[family] += 1
    COUNTS[family] += 1


def first_case(C, N, k, pad, T, batch, stride_pad=0, name=None):
    Td = (T + 1) // 2 + 2                                   # the last rows read x past T (zero)
    mo_lo, mo_hi = 3, Td - 5 - (k % 3)                      # a shorter odd class: its CTAs exit early on the last row tile
    return dict(C=C, N=N, k=k, pad_left=pad, batch=batch, T=T, x_bstride=T * C + stride_pad * C, Td=Td, dec_bstride=Td * N + stride_pad * N,
                mo_lo=mo_lo, mo_hi=mo_hi, odd_bstride=(mo_hi - mo_lo) * N + stride_pad * N, name=name or "C%dN%dk%dp%dT%db%d" % (C, N, k, pad, T, batch))


def first_cases():
    cs = []
    lib = H.load()
    for C, N in ((1, 16), (1, 24), (2, 16), (2, 24)):
        kmax = max(k for k in range(1, 17) if lib.wkh_first_supported(C, N, k))
        for k in range(1, kmax + 1):
            for pad in sorted({0, (k - 1) // 2}):
                cs.append(first_case(C, N, k, pad, 601 + 37 * k, 1 + (k % 3), stride_pad=(k % 2) * 5))
    return cs


# ------------------------------------------------------------------------------------------------
# output layer
# ------------------------------------------------------------------------------------------------
def out_case(*, batch, Tf, C, F, K_, ofs, output_type, activation, training, pad=None, name=""):
    nconv = K_ - 1 if output_type == 1 else K_
    pad = (ofs - 1) // 2 if pad is None else pad
    T_out = Tf - (ofs - 1) + 2 * pad                       # 'valid' conv of the feature rows, with pad rows of zeros on the left
    crop_feat, crop_out = 7, 7 + 3
    T_in = max(crop_feat + Tf, crop_out + T_out) + 5
    G = dict(batch=batch, T_in=T_in, Tf=Tf, T_out=T_out, C=C, F=F, nconv=nconv, K=K_, ofs=ofs, pad_left=pad, crop_feat=crop_feat,
             crop_out=crop_out, output_type=output_type, activation=activation, training=training, name=name)
    off = 16                                                # the output convs' weights and biases, NaN between them
    for s in range(8):
        if s < nconv:
            G["w_off%d" % s] = off
            off += ofs * (C + F) * C + 9
            G["b_off%d" % s] = off
            off += C + 5
        else:
            G["w_off%d" % s] = G["b_off%d" % s] = -1
    G["n_params"] = off + 16
    return G


def out_params(G, gen, regime):
    torch = _torch()
    p = torch.full((G["n_params"],), float("nan"), device="cuda")
    Cin = G["C"] + G["F"]
    for s in range(G["nconv"]):
        w0, b0 = G["w_off%d" % s], G["b_off%d" % s]
        p[w0:w0 + G["ofs"] * Cin * G["C"]] = data(gen, G["ofs"] * Cin * G["C"], regime, "w")
        p[b0:b0 + G["C"]] = data(gen, G["C"], regime)
    return p


def out_weights(G, par):
    """-> W [nconv, ofs, Cin, C], bias [nconv, C] (float64)"""
    torch = _torch()
    Cin = G["C"] + G["F"]
    W = torch.stack([par[G["w_off%d" % s]:G["w_off%d" % s] + G["ofs"] * Cin * G["C"]].view(G["ofs"], Cin, G["C"]) for s in range(G["nconv"])])
    b = torch.stack([par[G["b_off%d" % s]:G["b_off%d" % s] + G["C"]] for s in range(G["nconv"])])
    return W.double(), b.double()


def out_input(G, mix, feat):
    """[B, T_out, ofs, Cin]: the output conv's window of every frame, zero outside [0, Tf) (float64)"""
    torch = _torch()
    B = G["batch"]
    X = torch.cat([mix.view(B, G["T_in"], G["C"])[:, G["crop_feat"]:G["crop_feat"] + G["Tf"]], feat.view(B, G["Tf"], G["F"])], 2).double()
    t = torch.arange(G["T_out"], device="cuda")[:, None] + torch.arange(G["ofs"], device="cuda")[None, :] - G["pad_left"]
    ok = (t >= 0) & (t < G["Tf"])
    return X[:, t.clamp(0, G["Tf"] - 1), :] * ok[None, :, :, None]


def out_memory(G, gen, regime, dpre=False, feat_sign=False):
    torch = _torch()
    B, C = G["batch"], G["C"]
    mem = Mem()
    mem.add("par", out_params(G, gen, regime))
    mem.add("mix", data(gen, B * G["T_in"] * C, regime))
    f = data(gen, B * G["Tf"] * G["F"], regime)
    if feat_sign:
        f[torch.rand(f.numel(), generator=gen, device="cuda") < 0.1] = 0.0       # slope 0.2 at exactly 0
    mem.add("feat", f)
    if dpre:
        mem.add("dpre", data(gen, B * G["T_out"] * G["nconv"] * C, regime))
    return mem


def run_output_fwd(G, regime, seed, targets=True, outputs=True, family="output fwd"):
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    B, C, K_, nconv, T_out = G["batch"], G["C"], G["K"], G["nconv"], G["T_out"]
    inv = 1.0 / (B * T_out * C * K_)
    assert regime != "exact" or inv == 2.0 ** round(np.log2(inv)), "exact regime needs a power-of-two inv_count"
    mem = out_memory(G, gen, regime)
    n_src = K_ * B * T_out * C
    if targets:
        mem.add("tg", data(gen, n_src, regime))
        mem.add("dpre", torch.full((B * T_out * nconv * C,), float(SENTINEL), device="cuda"))
        mem.add("loss", torch.zeros(1, device="cuda") + (0.5 if regime == "exact" else 0.0))      # pre-filled accumulator
        lb = H.output_partial_bytes(G)[1]
        mem.arena("lpart", lb)
        mem.add("lcount", torch.zeros(1, device="cuda"))                  # the CTA counter: 0 before, 0 again after
    if outputs:
        mem.add("out", torch.full((n_src,), float(SENTINEL), device="cuda"))
    before = mem.snapshot()
    res = []
    for _ in range(2):
        mem.restore(before)
        H.call("output_fwd", H.output_geom(G), inv, mem.ptr("par"), mem.ptr("mix"), mem.ptr("feat"), mem.ptr("tg") if targets else 0,
               mem.ptr("out") if outputs else 0, mem.ptr("dpre") if targets else 0, mem.ptr("loss") if targets else 0,
               mem.ptr("lpart") if targets else 0, H.output_partial_bytes(G)[1], mem.ptr("lcount") if targets else 0, stream())
        torch.cuda.synchronize()
        outs = {}
        for nm in ("out", "dpre", "loss", "lpart"):
            if nm in mem.t:
                outs[nm] = torch.ones_like(mem.d(nm), dtype=torch.bool)
        mem.check_rest(before, outs, "output fwd %s" % G["name"])
        res.append({nm: mem.d(nm).clone() for nm in ("out", "dpre", "loss") if nm in mem.t})
    for nm in res[0]:
        assert torch.equal(res[0][nm].view(torch.int32), res[1][nm].view(torch.int32)), "output fwd %s: two runs differ" % nm
    W, b = out_weights(G, mem.d("par"))
    Xw = out_input(G, mem.d("mix"), mem.d("feat"))
    pre = torch.einsum("btjc,sjco->btso", Xw, W) + b                     # [B, T_out, nconv, C]
    pre_abs = torch.einsum("btjc,sjco->btso", Xw.abs(), W.abs()) + b.abs()
    tanh = G["activation"] == 0
    clip = lambda v: v.clamp(-1.0, 1.0)                                  # noqa: E731
    est = pre.tanh() if tanh else (pre if G["training"] else clip(pre))
    est_tol = TAU_OUT * pre_abs + (4 * U32 * est.abs() if tanh else 0)   # tanhf: <= 2 ulp, plus the conv's rounding
    srcs, tols = [est[:, :, s] for s in range(nconv)], [est_tol[:, :, s] for s in range(nconv)]
    mixo = mem.d("mix").view(B, G["T_in"], C)[:, G["crop_out"]:G["crop_out"] + T_out].double()
    if G["output_type"] == 1:
        last = mixo - est.sum(2)
        if not G["training"]:
            last = clip(last)
        srcs.append(last)
        tols.append(est_tol.sum(2) + 2 * nconv * U32 * (mixo.abs() + est.abs().sum(2)))
    exact = regime == "exact"
    if outputs:
        got = res[0]["out"].view(K_, B, T_out, C)
        for s in range(K_):
            if exact:
                exact_eq(family, got[s], f32_exact(srcs[s], "estimates"), "output fwd %s source %d" % (G["name"], s))
            else:
                check(family, got[s], srcs[s], tols[s], "output fwd %s source %d" % (G["name"], s), pre_abs[:, :, s] if s < nconv else None)
    if targets:
        tg = mem.d("tg").view(K_, B, T_out, C).double()
        e = [srcs[s] - tg[s] for s in range(K_)]
        glast = 2 * e[nconv] * inv if G["output_type"] == 1 else torch.zeros_like(e[0])
        dp = torch.stack([2 * e[s] * inv - glast for s in range(nconv)], 2)
        if tanh:
            dp = dp * (1 - est * est)
        loss = 0.5 * exact + sum(float((x * x).sum()) for x in e) * inv
        got_dp = res[0]["dpre"].view(B, T_out, nconv, C)
        got_loss = float(res[0]["loss"][0])
        etol = [tols[s] + U32 * (srcs[s].abs() + tg[s].abs()) for s in range(K_)]
        ltol = inv * sum(float((2 * e[s].abs() * etol[s]).sum()) for s in range(K_)) + 2.0 ** -18 * abs(loss)
        if exact:
            exact_eq(family, got_dp, f32_exact(dp, "dpre"), "output fwd %s dpre" % G["name"])
            if sum(float((x * x).sum()) for x in e) * 16 < 2 ** 24:     # every partial loss sum exact
                assert got_loss == loss, ("loss", got_loss, loss)
            else:
                assert abs(got_loss - loss) <= 2.0 ** -18 * abs(loss), ("loss", got_loss, loss)
        else:
            gl_tol = 2 * inv * etol[nconv] if G["output_type"] == 1 else 0
            dp_tol = torch.stack([2 * inv * etol[s] + gl_tol for s in range(nconv)], 2) + 4 * U32 * dp.abs()
            if tanh:
                glin = torch.stack([(2 * e[s] * inv - glast).abs() for s in range(nconv)], 2)
                dp_tol = dp_tol + glin * (2 * est_tol + 4 * U32)
            check(family, got_dp, dp, dp_tol, "output fwd %s dpre" % G["name"])
            assert abs(got_loss - loss) <= ltol, ("loss", got_loss, loss, ltol)
    if not exact and not tanh and G["training"]:
        # power: one dropped boundary tap (frame 0 reading feature row 0 with pad > 0, else row Tf-1 of the last frame).  Only where
        # the estimate is the conv itself: tanh (saturated on random data) and the test-time clip can hide any tap
        t, j = (0, G["pad_left"]) if G["pad_left"] else (T_out - 1, G["ofs"] - 1)
        c = (Xw[:, t, j][:, None, :, None] * W[:, j][None]).sum(2).abs()     # [B, nconv, C]
        assert bool((c > est_tol[:, t]).any()), "output fwd: a dropped boundary tap is below the bound"
    if exact:
        EXACT[family] += 1
    COUNTS[family] += 1


def run_output_dgrad(G, regime, seed, family="output dgrad"):
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    B, C, F, Tf, T_out, nconv, ofs = G["batch"], G["C"], G["F"], G["Tf"], G["T_out"], G["nconv"], G["ofs"]
    mem = out_memory(G, gen, regime, dpre=True, feat_sign=True)
    mem.add("gfeat", torch.full((B * Tf * F,), float(SENTINEL), device="cuda"))
    before = mem.snapshot()
    H.call("output_dgrad", H.output_geom(G), mem.ptr("par"), mem.ptr("feat"), mem.ptr("dpre"), mem.ptr("gfeat"), stream())
    torch.cuda.synchronize()
    mem.check_rest(before, {"gfeat": torch.ones_like(mem.d("gfeat"), dtype=torch.bool)}, "output dgrad %s" % G["name"])
    W, _ = out_weights(G, mem.d("par"))
    Wf = W[:, :, C:, :]                                                   # [nconv, ofs, F, C]
    dp = mem.d("dpre").view(B, T_out, nconv, C).double()
    # frame t reads feature row t + j - pad: gfeat[r] = sum_j dp[r - j + pad] . W[j]
    r = torch.arange(Tf, device="cuda")[:, None] - torch.arange(ofs, device="cuda")[None, :] + G["pad_left"]
    ok = (r >= 0) & (r < T_out)
    D = dp[:, r.clamp(0, T_out - 1)] * ok[None, :, :, None, None]       # [B, Tf, ofs, nconv, C]
    s = torch.einsum("brjso,sjfo->brf", D, Wf)
    sa = torch.einsum("brjso,sjfo->brf", D.abs(), Wf.abs())
    a = mem.d("feat").view(B, Tf, F)
    got = mem.d("gfeat").view(B, Tf, F)
    if regime == "exact":
        exact_eq(family, got, f32_exact(s, "dgrad").float() * torch.where(a > 0, 1.0, np.float32(0.2)), "output dgrad %s" % G["name"])
        EXACT[family] += 1
    else:
        ref = s * slope(a.double())
        check(family, got, ref, TAU_OUT * sa + U32 * ref.abs(), "output dgrad %s" % G["name"], sa)
        # power: the edge taps of feature rows 0 and Tf-1 (what a dgrad skipping tap j = 0 or ofs-1 loses)
        for rr, j in ((0, min(G["pad_left"], ofs - 1)), (Tf - 1, max(0, Tf - 1 + G["pad_left"] - (T_out - 1)))):
            c = (0.2 * torch.einsum("bso,sfo->bf", D[:, rr, j], Wf[:, j])).abs()
            assert bool((c > TAU_OUT * sa[:, rr] + U32 * ref[:, rr].abs()).any()), "output dgrad: a dropped edge tap is below the bound"
    COUNTS[family] += 1


def run_output_wgrad(G, regime, seed, scale=2.0, family="output wgrad"):
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    B, C, F, T_out, nconv, ofs = G["batch"], G["C"], G["F"], G["T_out"], G["nconv"], G["ofs"]
    mem = out_memory(G, gen, regime, dpre=True)
    grads = torch.full((G["n_params"],), float(SENTINEL), device="cuda")
    Cin = C + F
    gmask = torch.zeros(G["n_params"], dtype=torch.bool, device="cuda")
    for s in range(nconv):
        gmask[G["w_off%d" % s]:G["w_off%d" % s] + ofs * Cin * C] = True
        gmask[G["b_off%d" % s]:G["b_off%d" % s] + C] = True
    grads[gmask] = data(gen, int(gmask.sum()), regime)
    mem.add("grads", grads)
    pb = H.output_partial_bytes(G)[0]
    mem.arena("part", pb)
    before = mem.snapshot()
    res = []
    for _ in range(2):
        mem.restore(before)
        H.call("output_wgrad", H.output_geom(G), mem.ptr("par"), mem.ptr("mix"), mem.ptr("feat"), mem.ptr("dpre"), mem.ptr("grads"),
               scale, mem.ptr("part"), pb, stream())
        torch.cuda.synchronize()
        mem.check_rest(before, {"grads": gmask, "part": torch.ones_like(mem.d("part"), dtype=torch.bool)}, "output wgrad %s" % G["name"])
        res.append(mem.d("grads").clone())
    assert torch.equal(res[0].view(torch.int32), res[1].view(torch.int32)), "output wgrad: two runs differ"
    got = res[0]
    assert not bool(torch.isnan(got[gmask]).any()), "output wgrad: NaN from an unwritten partial slot"
    Xw = out_input(G, mem.d("mix"), mem.d("feat"))                    # [B, T_out, ofs, Cin]
    dp = mem.d("dpre").view(B, T_out, nconv, C).double()
    sW = scale * torch.einsum("btjc,btso->sjco", Xw, dp)
    aW = scale * torch.einsum("btjc,btso->sjco", Xw.abs(), dp.abs())
    sb, ab = scale * dp.sum((0, 1)), scale * dp.abs().sum((0, 1))
    g0 = before["grads"][GUARD:-GUARD].double()
    power_b, power_w = False, False
    for s in range(nconv):
        w0, b0 = G["w_off%d" % s], G["b_off%d" % s]
        for lo, n, sm, am, nm in ((w0, ofs * Cin * C, sW[s], aW[s], "dW"), (b0, C, sb[s], ab[s], "db")):
            ref = g0[lo:lo + n] + sm.reshape(-1)
            rabs = g0[lo:lo + n].abs() + am.reshape(-1)
            if regime == "exact":
                assert bool((rabs * 64 < 2 ** 24).all()), "output wgrad: case too large for the exact regime"
                exact_eq(family, got[lo:lo + n], f32_exact(ref, "output wgrad"), "output wgrad %s conv %d %s" % (G["name"], s, nm))
            else:
                check(family, got[lo:lo + n], ref, TAU_RED * rabs, "output wgrad %s conv %d %s" % (G["name"], s, nm), rabs)
                # power: the bias "channel" (one term per frame) and one 64-row chunk of tap 0 are above the bound
                if nm == "db":
                    power_b = power_b or bool((sm.abs() > TAU_RED * rabs).any())
                else:
                    blk = (scale * torch.einsum("tc,to->co", Xw[0, :64, 0], dp[0, :64, s])).abs().reshape(-1)
                    power_w = power_w or bool((blk > TAU_RED * rabs[:blk.numel()]).any())
    if regime == "float":
        assert power_b and power_w, ("output wgrad: a dropped bias channel / row chunk is below the bound", power_b, power_w)
    else:
        EXACT[family] += 1
    COUNTS[family] += 1


def output_cases():
    cs = []
    for ot in (0, 1):
        for act in (0, 1):
            for tr in (0, 1):
                # B * T_out * C * K a power of two (inv_count exact); ofs 1 and 3 with both paddings
                cs.append(out_case(batch=2, Tf=256 + 0, C=2, F=24, K_=2, ofs=1, output_type=ot, activation=act, training=tr,
                                   name="ot%d_act%d_tr%d_ofs1" % (ot, act, tr)))
                cs.append(out_case(batch=4, Tf=128, C=1, F=31, K_=4, ofs=3, pad=1, output_type=ot, activation=act, training=tr,
                                   name="ot%d_act%d_tr%d_ofs3_same" % (ot, act, tr)))
                cs.append(out_case(batch=1, Tf=258, C=2, F=8, K_=2, ofs=3, pad=0, output_type=ot, activation=act, training=tr,
                                   name="ot%d_act%d_tr%d_ofs3_valid" % (ot, act, tr)))
    # nconv * C = WUN_MAX_OUT_COLS (8 sources, stereo, direct); F = 33 (Cin + 1 = 36 > 32: the second cbase pass)
    cs.append(out_case(batch=2, Tf=64, C=2, F=33, K_=8, ofs=1, output_type=0, activation=1, training=1, name="cols16_F33"))
    cs.append(out_case(batch=2, Tf=66, C=2, F=12, K_=8, ofs=3, pad=0, output_type=1, activation=0, training=1, name="diff8_ofs3"))
    return cs


# ------------------------------------------------------------------------------------------------
# upsampling backward
# ------------------------------------------------------------------------------------------------
def up_ref(G, due, dmid, x, w, scale):
    """-> gx (float64, before the slope), dvar sum (float64, before w(1-w) scale), their |.| versions"""
    torch = _torch()
    B, N, nmid, C = G["batch"], G["N"], G["nmid"], G["C"]
    due, dmid, x = due.view(B, N, C).double(), dmid.view(B, nmid, C).double(), x.view(B, N, C).double()
    dm = torch.zeros(B, N + 1, C, dtype=torch.float64, device="cuda")
    dm[:, 1:nmid + 1] = dmid                                 # dm[s + 1] = dmid[s] (0 past nmid)
    w = w.double()
    g = due + w * dm[:, 1:] + (1 - w) * dm[:, :-1]
    ga = due.abs() + w.abs() * dm[:, 1:].abs() + (1 - w).abs() * dm[:, :-1].abs()
    if G["mid_mode"] == 1:                                  # MID_CLAMP: the last row's "next" row is itself
        g[:, N - 1] += (1 - w) * dm[:, N]
        ga[:, N - 1] += (1 - w).abs() * dm[:, N].abs()
    xn = torch.zeros_like(x)
    xn[:, :-1] = x[:, 1:]
    diff = (x - xn)[:, :nmid]
    dv = (dmid * diff).sum((0, 1))
    dva = (dmid.abs() * (x.abs() + xn.abs())[:, :nmid]).sum((0, 1))
    return g, ga, dv, dva


def run_upsample(G, regime, seed, learned, scale=0.5, family="upsample bwd"):
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    B, N, nmid, C = G["batch"], G["N"], G["nmid"], G["C"]
    mem = Mem()
    mem.add("due", data(gen, B * N * C, regime))
    mem.add("dmid", data(gen, B * nmid * C, regime))
    x = data(gen, B * N * C, regime)
    x[torch.rand(x.numel(), generator=gen, device="cuda") < 0.1] = 0.0
    mem.add("x", x)
    mem.add("gx", torch.full((B * N * C,), float(SENTINEL), device="cuda"))
    if learned:
        mem.add("blend", data(gen, C, regime, "blend"))
        mem.add("dvar", data(gen, C, "exact"))
        pb = int(H.load().wkh_upsample_partial_bytes(B, C))
        mem.arena("part", pb)
        mem.add("count", torch.zeros(1, device="cuda"))                   # the CTA counter: 0 before, 0 again after
    else:
        pb = 0
    before = mem.snapshot()
    res = []
    for _ in range(2 if learned else 1):
        mem.restore(before)
        H.call("upsample_bwd", H.upsample_geom(G), mem.ptr("due"), mem.ptr("dmid"), mem.ptr("x"), mem.ptr("gx"),
               mem.ptr("blend") if learned else 0, mem.ptr("dvar") if learned else 0, scale, mem.ptr("part") if learned else 0, pb,
               mem.ptr("count") if learned else 0, stream())
        torch.cuda.synchronize()
        outs = {"gx": torch.ones_like(mem.d("gx"), dtype=torch.bool)}
        if learned:
            outs["dvar"] = torch.ones_like(mem.d("dvar"), dtype=torch.bool)
            outs["part"] = torch.ones_like(mem.d("part"), dtype=torch.bool)
        mem.check_rest(before, outs, "upsample %s" % G["name"])
        res.append((mem.d("gx").clone(), mem.d("dvar").clone() if learned else None))
    if learned:
        assert torch.equal(res[0][1].view(torch.int32), res[1][1].view(torch.int32)), "upsample %s: two runs give different dvar bits" % G["name"]
        assert torch.equal(res[0][0].view(torch.int32), res[1][0].view(torch.int32))
    w = mem.d("blend") if learned else torch.full((C,), 0.5, device="cuda")
    g, ga, dv, dva = up_ref(G, mem.d("due"), mem.d("dmid"), mem.d("x"), w, scale)
    xs = mem.d("x").view(B, N, C)
    got = res[0][0].view(B, N, C)
    w64 = w.double()
    fac = w64 * (1 - w64) * scale
    if regime == "exact":
        exact_eq(family, got, f32_exact(g, "upsample gx") * torch.where(xs > 0, 1.0, np.float32(0.2)), "upsample %s gx" % G["name"])
        if learned:
            v = f32_exact(f32_exact(dv * w64, "dvar").double() * (1 - w64), "dvar").double() * scale
            ref = before["dvar"][GUARD:-GUARD].double() + f32_exact(v, "dvar").double()
            exact_eq(family, res[0][1], f32_exact(ref, "dvar"), "upsample %s dvar" % G["name"])
        EXACT[family] += 1
    else:
        ref = g * slope(xs.double())
        check(family, got, ref, TAU_UP * ga + U32 * ref.abs(), "upsample %s gx" % G["name"], ga)
        if learned:
            d0 = before["dvar"][GUARD:-GUARD].double()
            rabs = d0.abs() + dva * fac.abs()
            check(family, res[0][1], d0 + dv * fac, TAU_RED * rabs + 4 * U32 * (dv * fac).abs(), "upsample %s dvar" % G["name"], rabs)
            # power: one MID neighbour of one row (item 0, row 0 .. the first rows' dm * x[s+1] term) is above the bound
            r = min(8, nmid, N - 1)
            c = (mem.d("dmid").view(B, nmid, C)[0, :r].double() * xs[0, 1:r + 1].double()).abs().max(0).values * fac.abs()
            assert bool((c > TAU_RED * rabs).any()), "upsample dvar: a dropped MID neighbour is below the bound"
        # power for gx: the MID_CLAMP boundary term of row N-1 / the dmid[s-1] neighbour of row 1
        if G["mid_mode"] == 1:
            c = ((1 - w64) * mem.d("dmid").view(B, nmid, C)[:, N - 1].double()).abs() * 0.2
            assert bool((c > TAU_UP * ga[:, N - 1] + U32 * ref[:, N - 1].abs()).any()), "upsample: the clamp term is below the bound"
    COUNTS[family] += 1


def up_cases():
    cs = []
    for mode in (0, 1, 2):
        for B, N, C in ((1, 40, 24), (3, 300, 50), (16, 2000, 72), (2, 9000, 17)):
            nmid = N - 1 if mode == 0 else N
            cs.append(dict(batch=B, N=N, nmid=nmid, C=C, mid_mode=mode, name="mode%d_B%d_N%d_C%d" % (mode, B, N, C)))
    return cs


# ------------------------------------------------------------------------------------------------
# Adam, sigmoid, gather / scatter
# ------------------------------------------------------------------------------------------------
def run_adam(n, seed, device_state, steps=1, family="adam"):
    torch = _torch()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    mem = Mem()
    pad = 7                                                  # words past n: must keep their bits
    for nm in ("p", "g", "m", "v"):
        v = data(gen, n + pad, "float")
        if nm == "v":
            v = v.abs()
        mem.add(nm, v)
    b1, b2, eps, lr = np.float32(0.9), np.float32(0.999), np.float32(1e-8), np.float32(1e-3)
    state = torch.tensor([b1 ** 3, b2 ** 3, 3.0], device="cuda") if device_state else None
    if device_state:
        mem.add("state", state)
    for step in range(steps):
        before = mem.snapshot()
        if device_state:
            st = mem.d("state").double()
            lr_t = float(lr) * np.sqrt(1 - float(st[1])) / (1 - float(st[0]))
        else:
            lr_t = float(np.float32(float(lr) * np.sqrt(1 - 0.999 ** (step + 4)) / (1 - 0.9 ** (step + 4))))
        H.call("adam", mem.ptr("p"), mem.ptr("g"), mem.ptr("m"), mem.ptr("v"), n, float(lr) if device_state else lr_t, float(b1), float(b2),
               float(eps), mem.ptr("state") if device_state else 0, stream())
        torch.cuda.synchronize()
        outs = {nm: torch.arange(n + pad, device="cuda") < n for nm in ("p", "m", "v")}
        if device_state:
            outs["state"] = torch.ones(3, dtype=torch.bool, device="cuda")
        mem.check_rest(before, outs, "adam n=%d" % n)
        p0, g, m0, v0 = [before[nm][GUARD:GUARD + n].double() for nm in ("p", "g", "m", "v")]
        m = float(b1) * m0 + (1 - float(b1)) * g
        v = float(b2) * v0 + (1 - float(b2)) * g * g
        upd = lr_t * m / (v.sqrt() + float(eps))
        upd_abs = lr_t * (float(b1) * m0.abs() + (1 - float(b1)) * g.abs()) / (v.sqrt() + float(eps))
        # fp32: 2 roundings in m and v, sqrtf / division / lr_t each <= 1 ulp (0.5 ulp IEEE), the update's subtraction
        check(family, mem.d("m")[:n], m, 4 * U32 * (float(b1) * m0.abs() + (1 - float(b1)) * g.abs()), "adam m n=%d" % n)
        check(family, mem.d("v")[:n], v, 4 * U32 * v, "adam v n=%d" % n)
        # the final subtraction alone may round by half an ulp of p: one full ulp of margin on it
        ptol = 2 * U32 * (p0.abs() + upd.abs()) + 2.0 ** -19 * upd_abs
        check(family, mem.d("p")[:n], p0 - upd, ptol, "adam p n=%d" % n)
        if n % 4:       # power: the n % 4 tail left unchanged would be seen
            t = slice(n - n % 4, n)
            assert bool((upd[t].abs() > ptol[t]).any()), "adam: the tail is below the bound"
        if device_state:
            st = mem.d("state")
            want = torch.tensor([float(before["state"][GUARD]) * b1, float(before["state"][GUARD + 1]) * b2,
                                 float(before["state"][GUARD + 2]) + 1], device="cuda")
            assert torch.equal(st, want.float()), ("adam_advance", st, want)
    COUNTS[family] += 1


# ------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
def test_first_layer_matches_float64(regime):
    _gpu_lib()
    for i, G in enumerate(first_cases()):
        run_first_fwd(G, regime, 100 + i)
        run_first_wgrad(G, regime, 300 + i, scale=0.5 if i % 2 else 2.0, null_db=(i % 7 == 3))
    if regime == "float":
        # a batch large enough that rows_per_cta grows past 128 (several 128-row blocks per CTA), wide batch strides, batch 1
        for C, N in ((1, 16), (1, 24), (2, 16), (2, 24)):
            G = first_case(C, N, 5, 2, 8001, 20, stride_pad=3, name="big_C%dN%d" % (C, N))
            run_first_fwd(G, regime, 11)
            run_first_wgrad(G, regime, 12)
        G = first_case(2, 24, 15, 7, 300001, 1, name="long_b1")
        run_first_fwd(G, regime, 13)
        run_first_wgrad(G, regime, 14)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
def test_output_layer_matches_float64(regime):
    _gpu_lib()
    for i, G in enumerate(output_cases()):
        if regime == "exact" and G["activation"] == 0:
            continue                                          # tanhf: float regime only
        run_output_fwd(G, regime, 500 + i)
        run_output_fwd(G, regime, 600 + i, targets=(i % 2 == 0), outputs=(i % 2 == 1))
        run_output_dgrad(G, regime, 700 + i)
        run_output_wgrad(G, regime, 800 + i)
    # B * Tf * F above 132 * 16 * 256: output_dgrad_kernel's grid-stride loop runs; many row chunks in the wgrad
    G = out_case(batch=16, Tf=8192, C=2, F=24, K_=2, ofs=1, output_type=1, activation=1, training=1, name="b16_long")
    run_output_dgrad(G, regime, 900)
    run_output_fwd(G, regime, 901)
    if regime == "float":
        run_output_wgrad(G, regime, 902)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
def test_upsample_backward_matches_float64(regime):
    _gpu_lib()
    for i, G in enumerate(up_cases()):
        for learned in (False, True):
            if learned and G["mid_mode"] == 1:
                continue                                      # the plan never pairs learned upsampling with MID_CLAMP (host test)
            if regime == "exact" and G["batch"] * G["N"] > 20000 and learned:
                continue                                      # dvar sums leave the exact range
            run_upsample(G, regime, 1000 + i, learned)


@pytest.mark.gpu
def test_adam_matches_float64():
    _gpu_lib()
    for n in (0, 1, 2, 3, 4, 5, 4097, 132 * 8 * 256 * 4 + 13):
        for dev in (False, True):
            if n == 0:
                torch = _torch()
                z = torch.zeros(8, device="cuda")
                H.call("adam", z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), 0, 1e-3, 0.9, 0.999, 1e-8, 0, stream())
                torch.cuda.synchronize()
                assert not bool(z.any())
                continue
            run_adam(n, 40 + n % 97, dev, steps=3 if dev else 1)


@pytest.mark.gpu
def test_sigmoid_extreme_inputs():
    torch = _torch()
    _gpu_lib()
    xs = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 1.0, -1.0, 15.0, -15.0, 87.0, -87.0, 88.5, -88.5, 89.0, -89.0, 100.0, -100.0,
                       1e30, -1e30, float("inf"), float("-inf"), float("nan")], device="cuda")
    xs = torch.cat([xs, torch.randn(1000, device="cuda") * 30])
    mem = Mem()
    mem.add("x", xs)
    mem.add("y", torch.full_like(xs, float(SENTINEL)))
    before = mem.snapshot()
    H.call("sigmoid", mem.ptr("x"), mem.ptr("y"), xs.numel(), stream())
    torch.cuda.synchronize()
    mem.check_rest(before, {"y": torch.ones(xs.numel(), dtype=torch.bool, device="cuda")}, "sigmoid")
    y, x = mem.d("y"), xs.double()
    ref = 1.0 / (1.0 + torch.exp(-x))
    fin = ~torch.isnan(x)
    assert bool(torch.isnan(y[~fin]).all())
    # expf <= 2 ulp, the add and the division <= 0.5 ulp each; below 2^-126 the result is subnormal (absolute floor)
    check("sigmoid", y[fin], ref[fin], 4 * U32 * ref[fin].abs() + 2.0 ** -126, "sigmoid")
    assert bool((y[fin] >= 0).all() & (y[fin] <= 1).all())
    COUNTS["sigmoid"] += 1


@pytest.mark.gpu
def test_gather_scatter_windows_bit_exact():
    torch = _torch()
    _gpu_lib()
    for C, T_in, T_out, n_frames, K_ in ((2, 300, 100, 1234, 3), (1, 64, 16, 50, 2), (2, 1000, 400, 100000, 4)):
        step = T_out
        starts = list(range(0, n_frames - T_out + 1, step))
        if not starts or starts[-1] + T_out < n_frames:
            starts.append(n_frames - T_out)                   # the shifted last window overlaps its predecessor
        nw = len(starts)
        n_padded = n_frames + (T_in - T_out) // 2 + 3          # windows near the end read past n_padded (zeros)
        st = torch.tensor(starts, dtype=torch.int64, device="cuda")
        padded = torch.randn(n_padded * C + 8, device="cuda")
        padded[n_padded * C:] = float("nan")                   # never read
        out = torch.full((nw * T_in * C + GUARD,), float(SENTINEL), device="cuda")
        H.call("gather_windows", padded.data_ptr(), n_padded, st.data_ptr(), nw, T_in, C, out.data_ptr(), stream())
        torch.cuda.synchronize()
        src = (st[:, None] * C + torch.arange(T_in * C, device="cuda")[None, :]).reshape(-1)
        want = torch.where(src < n_padded * C, padded[src.clamp(max=n_padded * C - 1)], torch.zeros((), device="cuda"))
        assert torch.equal(out[:nw * T_in * C].view(torch.int32), want.view(torch.int32))
        assert bool((out[nw * T_in * C:] == SENTINEL).all())
        assert starts[-1] + T_in > n_padded                    # the case reaches the zero fill
        outs = torch.randn(K_ * nw * T_out * C, device="cuda")
        preds = torch.full((K_ * n_frames * C + GUARD,), float(SENTINEL), device="cuda")
        H.call("scatter_windows", outs.data_ptr(), st.data_ptr(), nw, K_, T_out, C, preds.data_ptr(), n_frames, stream())
        torch.cuda.synchronize()
        ref = torch.full((K_, n_frames, C), float(SENTINEL), device="cuda")
        o = outs.view(K_, nw, T_out, C)
        for w in range(nw):                                    # in order: the last window wins where it overlaps
            a, b = starts[w], min(starts[w] + T_out, n_frames)
            ref[:, a:b] = o[:, w, :b - a]
        assert torch.equal(preds[:K_ * n_frames * C].view(torch.int32), ref.reshape(-1).view(torch.int32))
        assert bool((preds[K_ * n_frames * C:] == SENTINEL).all())
    COUNTS["gather/scatter"] += 1


# ------------------------------------------------------------------------------------------------
# replays: the step launches the engine emits
# ------------------------------------------------------------------------------------------------
REPLAYS = K.REPLAYS + [("M5_full_b16", ["full"], {}, 16, None, {})]


def _engine(named, ov, batch, nf):
    cfg = Config.build_config(named, ov, experiment_id=0)["model_config"]
    t_in, _ = O.get_padding(cfg, nf or cfg["num_frames"])
    eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
    eng.launch_descriptions(batch)
    return eng


@pytest.mark.gpu
@pytest.mark.parametrize("name,named,ov,batch,nf,env", REPLAYS, ids=[r[0] for r in REPLAYS])
def test_replayed_step_launches_match_float64(name, named, ov, batch, nf, env, monkeypatch):
    torch = _torch()
    _gpu_lib()
    for k in [k for k in os.environ if k.startswith("WUN_")]:
        monkeypatch.delenv(k)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = _engine(named, ov, batch, nf)
    kinds = [k for k, _ in eng.step_launches]
    assert kinds.count("output") == 1 and kinds.count("adam") == 1
    for i, (kind, d) in enumerate(eng.step_launches):
        if kind == "first":
            G = dict(d, name="%s_first" % name)
            run_first_fwd(G, "float", 20 + i, family="replay first fwd")
            run_first_wgrad(G, "float", 40 + i, scale=1.0, family="replay first wgrad")
        elif kind == "output":
            G = dict(d, name="%s_output" % name, training=1)
            n = 16
            for s in range(8):
                n = max(n, d["w_off%d" % s] + d["ofs"] * (d["C"] + d["F"]) * d["C"] + 8, d["b_off%d" % s] + d["C"] + 8)
            G["n_params"] = n
            run_output_fwd(G, "float", 60, family="replay output fwd")
            run_output_dgrad(G, "float", 61, family="replay output dgrad")
            run_output_wgrad(G, "float", 62, scale=1.0, family="replay output wgrad")
        elif kind == "upsample":
            G = dict(d, name="%s_up%d" % (name, d["level"]))
            run_upsample(G, "float", 80 + i, d["dvar"] >= 0, scale=1.0, family="replay upsample bwd")
        elif kind == "adam" and batch == 1 and name.startswith("M"):
            run_adam(d["n"], 99, True, family="replay adam")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# host tests (no GPU)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,named,ov,batch,nf,env", REPLAYS, ids=[r[0] for r in REPLAYS])
def test_exported_step_launches_parse_and_learned_upsampling_never_clamps(name, named, ov, batch, nf, env, monkeypatch):
    """Host only: every configuration exports one output and one adam line, one upsample line per level (with an interp gradient
    exactly for learned upsampling) and a first line exactly when the dedicated first layer runs.  The kernel's interp gradient
    at row N-1 is only right for MID_ZERO and MID_VALID: the plan never builds learned upsampling with MID_CLAMP."""
    lib = K._lib_or_skip()
    for k in [k for k in os.environ if k.startswith("WUN_")]:
        monkeypatch.delenv(k)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = Config.build_config(named, ov, experiment_id=0)["model_config"]
    eng = _engine(named, ov, batch, nf)
    kinds = [k for k, _ in eng.step_launches]
    assert kinds.count("output") == 1 and kinds.count("adam") == 1
    ups = [d for k, d in eng.step_launches if k == "upsample"]
    assert sorted(d["level"] for d in ups) == list(range(cfg["num_layers"]))
    learned = cfg["upsampling"] == "learned"
    for d in ups:
        assert (d["dvar"] >= 0) == learned and (d["blend"] >= 0) == learned
        assert not (d["dvar"] >= 0 and d["mid_mode"] == 1)
        assert d["batch"] == batch and d["nmid"] in (d["N"], d["N"] - 1)
    dedicated = bool(lib.wkh_first_supported(cfg["num_channels"], cfg["num_initial_filters"], cfg["input_filter_size"]))
    assert kinds.count("first") == (1 if dedicated else 0), (kinds.count("first"), dedicated)
    for d in (d for k, d in eng.step_launches if k == "first"):
        assert d["batch"] == batch and d["k"] == cfg["input_filter_size"] and d["N"] == cfg["num_initial_filters"]
    assert dict(eng.step_launches)["adam"]["n"] == eng.param_numel
    monkeypatch.setenv("WUN_FIRST_LAYER", "0")
    eng0 = _engine(named, ov, batch, nf)
    assert "first" not in [k for k, _ in eng0.step_launches]


@pytest.mark.gpu
def test_zz_step_report():
    """Prints the case count per kernel family, the exact-regime matches and the worst err / ref_abs of the float regime."""
    print("\nkernel family                   cases  exact(bit for bit)  worst err/ref_abs (err/bound for the ulp-bounded)")
    for fam in sorted(COUNTS):
        w = WORST.get(fam, WORST.get(fam + " (err/bound)"))
        print("%-30s %6d %10s %22s" % (fam, COUNTS[fam], EXACT.get(fam, "-"), ("%.2e" % w) if w is not None else "-"))
    for fam in ("first fwd", "first wgrad", "output fwd", "output dgrad", "output wgrad", "upsample bwd", "adam", "sigmoid",
                "gather/scatter"):
        assert COUNTS.get(fam, 0) > 0, fam
