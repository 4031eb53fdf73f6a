"""The conv / dgrad / wgrad launch builders and runners of tests/test_kernels_gpu.py, which test_wgrad_tiles.py and
test_configurations_gpu.py run too: synthetic launch descriptions and their memory images, one synthetic launch through
tests/kernels/harness.cu against the float64 interpreter (tests/launch_interp.py), and the replay of every conv and wgrad launch
of a configuration.  The regimes and checks are described in tests/test_kernels_gpu.py."""
from collections import defaultdict

import numpy as np
import torch

from launch_checks import COUNTS, EXACT, GUARD, SENTINEL, TAU, H, check, engine, stream
from launch_interp import PAR_BASE, WS_BASE, plane_rows, run_launch, run_wgrad_layer


# ------------------------------------------------------------------------------------------------
# synthetic launch descriptions
# ------------------------------------------------------------------------------------------------
class Synth(object):
    """Allocates tensors in a synthetic workspace / parameter buffer and records which elements hold data."""

    def __init__(self):
        self.n = {"ws": GUARD, "par": GUARD}
        self.out_tensors = []        # (offset, elements) of every output tensor: sentinel outside the views

    def alloc(self, buf, n):
        off = (self.n[buf] + 63) // 64 * 64
        self.n[buf] = off + n + GUARD
        return off

    @staticmethod
    def addr(buf, off):
        return {"ws": WS_BASE, "par": PAR_BASE}[buf] + 4 * off


def make_plane(S, batch, C, r_lo, r_hi, step=1, Ct=None, coff=0, kind=0, mid_mode=0, blend=False):
    Ct = Ct or C + coff
    if kind == 1 and mid_mode != 0:              # the "next" row of plane row r is tensor row r + 1: plane row = tensor row
        T, row_offset, step = r_hi, 0, 1
    else:
        pad = 3
        row_offset = pad - r_lo * step
        T = pad + (r_hi - r_lo + 1) * step + pad
    off = S.alloc("ws", batch * T * Ct)
    bl = S.addr("ws", S.alloc("ws", C)) if blend else -1
    return dict(base=S.addr("ws", off + row_offset * Ct + coff), bstride=T * Ct, rstride=step * Ct, r_lo=r_lo, r_hi=r_hi, C=C,
                kind=kind, mid_mode=mid_mode, xrows=T, blend=bl)


def make_out(S, batch, Nh, lo, hi, Ct=None, coff=0, saved=False):
    Ct = Ct or Nh + coff
    pad = 2
    T = pad + (hi - lo) + pad
    off = S.alloc("ws", batch * T * Ct)
    S.out_tensors.append((off, batch * T * Ct))
    rel = (pad - lo) * Ct + coff
    sv = -1
    if saved:
        soff = S.alloc("ws", batch * T * Ct)
        sv = S.addr("ws", soff + rel)
    return S.addr("ws", off + rel), T * Ct, Ct, sv


def conv_desc(*, dg, N, batch, planes, classes, bias=True, epi=None, pair=None, name=""):
    """planes: make_plane kwargs; classes: dict(m=(lo, hi), terms=[(plane, d)], acc=(lo, hi), saved, Ct, coff).
    pair: dict(h=[(lo0, hi0), (lo1, hi1)], missing=[(term, half)], acc2, saved2): one pair-merged class of N = 2 * pairC."""
    S = Synth()
    P = [make_plane(S, batch, **p) for p in planes]
    pairC = N // 2 if pair else 0
    Nh = pairC or N
    if dg:
        w_sk, w_sn = 1, max(p["C"] for p in P)
    else:
        w_sk, w_sn = Nh, 1
    W0 = None
    cls, terms = [], []
    for qi, q in enumerate(classes):
        tb = len(terms)
        for j, (p, d) in enumerate(sorted(q["terms"])):
            wo = []
            for half in range(2 if pair else 1):
                if pair and (j, half) in pair.get("missing", []):
                    wo.append(-1)
                    continue
                ext = (P[p]["C"] - 1) * w_sk + (Nh - 1) * w_sn + 1
                off = S.alloc("par", ext)
                W0 = off if W0 is None else W0
                wo.append(off - W0)
            terms.append(dict(i=len(terms), plane=p, d=d, woff=wo[0], woff2=wo[1] if pair else -1))
        if pair:
            lo = min(pair["h"][0][0], pair["h"][1][0])
            hi = max(pair["h"][0][1], pair["h"][1][1])
        else:
            lo, hi = q["m"]
        base, bst, rst, sv = make_out(S, batch, Nh, lo, hi, q.get("Ct"), q.get("coff", 0), q.get("saved", False))
        acc = q.get("acc", (0, 0))
        c = dict(i=qi, base=base, bstride=bst, rstride=rst, m_lo=lo, m_hi=hi, saved=sv, acc_lo=acc[0], acc_hi=acc[1],
                 term_begin=tb, term_end=len(terms), pairC=pairC, base2=-1, bstride2=0, rstride2=0, saved2=-1, acc_lo2=0, acc_hi2=0,
                 lo0=0, hi0=0, lo1=0, hi1=0)
        if pair:
            base2, bst2, rst2, sv2 = make_out(S, batch, Nh, lo, hi, None, 0, pair.get("saved2", False))
            acc2 = pair.get("acc2", (0, 0))
            c.update(base2=base2, bstride2=bst2, rstride2=rst2, saved2=sv2, acc_lo2=acc2[0], acc_hi2=acc2[1], lo0=pair["h"][0][0],
                     hi0=pair["h"][0][1], lo1=pair["h"][1][0], hi1=pair["h"][1][1])
        cls.append(c)
    b_addr = S.addr("par", S.alloc("par", Nh)) if (bias and not dg) else -1
    if epi is None:
        epi = 1 if dg else 0
    L = dict(layer=0, N=N, pairC=pairC, w_sk=w_sk, w_sn=w_sn, W=S.addr("par", W0), bias=b_addr, epilogue=epi, batch=batch,
             nplanes=len(P), ncls=len(cls))
    L["pass"] = 1 if dg else 0
    return dict(launch=L, planes=P, cls=cls, terms=terms, synth=S, name=name)


def _halves(D, q):
    L = D["launch"]
    if L["pairC"]:
        return [(q["base"], q["bstride"], q["rstride"], q["saved"], q["acc_lo"], q["acc_hi"], q["lo0"], q["hi0"], L["pairC"]),
                (q["base2"], q["bstride2"], q["rstride2"], q["saved2"], q["acc_lo2"], q["acc_hi2"], q["lo1"], q["hi1"], L["pairC"])]
    return [(q["base"], q["bstride"], q["rstride"], q["saved"], q["acc_lo"], q["acc_hi"], q["m_lo"], q["m_hi"], L["N"])]


def _grid(off, b_n, bst, m, rst, n):
    return (off + np.arange(b_n)[:, None, None] * bst + np.asarray(m)[None, :, None] * rst + np.arange(n)[None, None, :]).reshape(-1)


def conv_outputs(D):
    """-> (ws offsets the launch writes, of which: rows that accumulate, and the saved-activation offsets it reads)."""
    B = D["launch"]["batch"]
    out, acc, saved = [], [], []
    for q in D["cls"]:
        for (base, bst, rst, sv, alo, ahi, lo, hi, n) in _halves(D, q):
            off = (base - WS_BASE) // 4
            m = np.arange(lo, hi)
            out.append(_grid(off, B, bst, m, rst, n))
            ma = m[(m >= alo) & (m < ahi)]
            acc.append(_grid(off, B, bst, ma, rst, n))
            if sv >= 0:
                saved.append(_grid((sv - WS_BASE) // 4, B, bst, m, rst, n))
    cat = lambda x: np.concatenate(x) if x else np.zeros(0, np.int64)       # noqa: E731
    return cat(out), cat(acc), cat(saved)


def plane_reads(P, B):
    """ws offsets of every element a plane view may read: its valid rows (and the MID "next" rows) and its blend vector."""
    off = (P["base"] - WS_BASE) // 4
    r = np.arange(P["r_lo"], P["r_hi"])
    idx = [_grid(off, B, P["bstride"], r, P["rstride"], P["C"])]
    if P["kind"] == 1:
        rn = r if P["mid_mode"] == 0 else r[r + 1 < P["xrows"]]
        idx.append(_grid(off, B, P["bstride"], rn + 1, P["rstride"], P["C"]))
    return np.concatenate(idx)


# The exact regimes with non-zero lo halves: one side of every product carries up to 12 significant bits (j / 2^10, |j| <= 2^12;
# its bf16 lo half is mostly non-zero), the other is exact in bf16, so hi*hi + hi*lo + lo*hi is the product itself.  exact_lo_x:
# activations / the wgrad's plane side carry the 12 bits, weights / the gradient side are integers in [-3, 3].  exact_lo_w: the
# reverse, against activations / plane rows k/4 in [-1, 1].  The exact side is zero with probability 1 - rho, rho chosen per
# case (lo_density) so that every sum stays within 2^23 units of the product grid.
LO_REGIMES = ("exact_lo_x", "exact_lo_w")
LO_BITS = 2.0 ** -10
LO_MEAN = 2048.0                       # mean |j| of the 12-bit side, in units of LO_BITS
SUM_UNITS = 2.0 ** 23                  # |partial sums| below 2^23 grid units: exact in fp32 in any order


def data(rng, n, regime, kind="act", rho=1.0):
    if regime in LO_REGIMES and kind != "blend":
        if (kind == "act") == (regime == "exact_lo_x"):
            return (rng.integers(-4096, 4097, n) * LO_BITS).astype(np.float32)
        v = rng.integers(-3, 4, n) if kind == "w" else rng.integers(-4, 5, n) / 4.0
        return (v * (rng.random(n) < rho)).astype(np.float32)
    if regime.startswith("exact"):
        if kind == "w":
            return rng.integers(-3, 4, n).astype(np.float32)
        if kind == "blend":
            return rng.choice(np.array([0.25, 0.5, 0.75], np.float32), n)
        return (rng.integers(-16, 17, n) / 4.0).astype(np.float32)
    if kind == "blend":
        return rng.uniform(0.0, 1.0, n).astype(np.float32)
    return (rng.standard_normal(n) * 2.0 ** rng.uniform(-6, 6, n)).astype(np.float32)


def lo_unit(regime, planes):
    """The grid of the products of a lo regime: the plane side's grid refined by MID blends (weights in quarters) or midpoints."""
    refine = max([4 if P["kind"] == 1 and P["blend"] >= 0 else 2 if P["kind"] == 1 else 1 for P in planes])
    return (LO_BITS if regime == "exact_lo_x" else 0.25 * LO_BITS) / refine, refine


def lo_density(regime, planes, nterms):
    """rho of the exact side: nterms products of mean LO_MEAN x (mean exact-side units) stay near SUM_UNITS / 2."""
    mean = 12.0 / 7.0 if regime == "exact_lo_x" else 20.0 / 9.0
    return min(1.0, SUM_UNITS / 2 / (nterms * LO_MEAN * mean * lo_unit(regime, planes)[1]))


def lo_fraction(x):
    """The fraction of x whose bf16 lo half is non-zero: split_hi_lo's hi = round to nearest even of the top 16 bits."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    hi = ((b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)
    return float(np.mean(x.astype(np.float32) - hi != 0))


def assert_lo_regime(name, regime, side, ref_abs, unit):
    """The lo regime is not vacuous (most of the 12-bit side has lo != 0) and its sums are exact in any order."""
    frac = lo_fraction(side)
    assert frac > 0.5, "%s (%s): only %.2f of the 12-bit side has a non-zero lo half" % (name, regime, frac)
    worst = float(np.max(ref_abs)) / unit
    assert worst < SUM_UNITS, "%s (%s): sum |terms| reaches %.3g grid units - shrink the case" % (name, regime, worst)


def fill_conv(D, rng, regime):
    S, L, B = D["synth"], D["launch"], D["launch"]["batch"]
    ws = np.full(S.n["ws"] + GUARD, np.nan, np.float32)
    par = np.full(S.n["par"] + GUARD, np.nan, np.float32)
    rho = 1.0
    if regime in LO_REGIMES:                             # products per output: the channels of every term of a class
        nterms = max(sum(D["planes"][t["plane"]]["C"] for t in D["terms"][q["term_begin"]:q["term_end"]]) for q in D["cls"])
        rho = lo_density(regime, D["planes"], nterms)
    side = []                                            # the 12-bit side of a lo regime
    for P in D["planes"]:
        idx = plane_reads(P, B)
        ws[idx] = data(rng, idx.size, regime, rho=rho)
        side.append(ws[idx])
        if P["blend"] >= 0:
            b0 = (P["blend"] - WS_BASE) // 4
            ws[b0:b0 + P["C"]] = data(rng, P["C"], regime, "blend")
    W0 = (L["W"] - PAR_BASE) // 4
    Nh = L["pairC"] or L["N"]
    wside = []
    for t in D["terms"]:
        C = D["planes"][t["plane"]]["C"]
        for wo in (t["woff"], t["woff2"] if L["pairC"] else -1):
            if wo >= 0:
                idx = (W0 + wo + np.arange(C)[:, None] * L["w_sk"] + np.arange(Nh)[None, :] * L["w_sn"]).reshape(-1)
                par[idx] = data(rng, idx.size, regime, "w", rho)
                wside.append(par[idx])
    if regime == "exact_lo_w":
        side = wside
    if L["bias"] >= 0:
        b0 = (L["bias"] - PAR_BASE) // 4
        par[b0:b0 + Nh] = data(rng, Nh, regime)
    for off, n in S.out_tensors:
        ws[off:off + n] = SENTINEL
    out, acc, saved = conv_outputs(D)
    ws[acc] = data(rng, acc.size, regime)
    if saved.size:
        s = data(rng, saved.size, regime)
        s[rng.random(saved.size) < 0.1] = 0.0            # slope 0.2 at exactly 0 (MaximumGrad)
        ws[saved] = s
    return {"ws": ws, "par": par, "mix": np.zeros(64, np.float32)}, np.concatenate(side)


# ------------------------------------------------------------------------------------------------
# synthetic weight-gradient layers
# ------------------------------------------------------------------------------------------------
def p(C, lo, hi, **kw):
    """The make_plane arguments of one plane of a case table."""
    return dict(C=C, r_lo=lo, r_hi=hi, **kw)


def wgrad_layer(*, batch, cout, planes, classes, groups, name=""):
    """planes: make_plane kwargs (activation side; C = that plane's input channels); classes: (m_lo, m_hi) of each forward class
    (its gradient view, C = cout); groups: (class, plane, [(tap, d)]).  dW is [taps][cin_tot][cout] (w_sk = cout, w_sn = 1)."""
    S = Synth()
    P = [make_plane(S, batch, **q) for q in planes]
    coff = np.cumsum([0] + [q["C"] for q in P])
    cin_tot = int(coff[-1])
    ntap = 1 + max(t for _, _, ts in groups for t, _ in ts)
    Gv = [make_plane(S, batch, cout, lo, hi) for lo, hi in classes]
    grads_n = {"n": GUARD}
    dW = 256
    db = dW + ntap * cin_tot * cout + 128
    out = []
    for gi, (q, pl, ts) in enumerate(groups):
        lo, hi = classes[q]
        out.append(dict(wgrad=dict(layer=0, group=gi, N=cout, w_sk=cout, w_sn=1, dW=dW, db=db, m_lo=lo, m_hi=hi, nterms=len(ts),
                                   batch=batch),
                        plane=P[pl], dpre=Gv[q],
                        terms=[dict(i=i, d=d, woff=int((t * cin_tot + coff[pl]) * cout)) for i, (t, d) in enumerate(ts)]))
    grads_n["n"] = db + cout + 256
    return dict(groups=out, synth=S, grads_n=grads_n["n"], name=name, batch=batch)


def wgrad_outputs(groups):
    idx = []
    for G in groups:
        g = G["wgrad"]
        C = G["plane"]["C"]
        for t in G["terms"]:
            idx.append((g["dW"] + t["woff"] + np.arange(C)[:, None] * g["w_sk"] + np.arange(g["N"])[None, :] * g["w_sn"]).reshape(-1))
        idx.append(g["db"] + np.arange(g["N"]))
    return np.unique(np.concatenate(idx))


def wgrad_rows(W):
    """The longest reduction of a wgrad case: batch x the rows of all its classes (a dW element receives <= 2 class sums)."""
    ranges = {(G["wgrad"]["m_lo"], G["wgrad"]["m_hi"]) for G in W["groups"]}
    return W["batch"] * sum(hi - lo for lo, hi in ranges)


def lo_fits(W):
    """Whether a wgrad case can take the lo regimes: the bias sums of 12-bit gradient rows stay within SUM_UNITS / 2."""
    return wgrad_rows(W) * LO_MEAN <= SUM_UNITS / 2


def fill_wgrad(W, rng, regime):
    """-> (memory, pre-filled gradient buffer, the 12-bit side of a lo regime).  The lo regimes put the plane side in place of
    the activations and the gradient side in place of the weights."""
    S, B = W["synth"], W["batch"]
    ws = np.full(S.n["ws"] + GUARD, np.nan, np.float32)
    rho = lo_density(regime, [G["plane"] for G in W["groups"]], wgrad_rows(W)) if regime in LO_REGIMES else 1.0
    seen = set()
    side = []
    for G in W["groups"]:
        for P, kind in ((G["plane"], "act"), (G["dpre"], "w" if regime in LO_REGIMES else "act")):
            if P["base"] in seen:
                continue
            seen.add(P["base"])
            idx = plane_reads(P, B)
            ws[idx] = data(rng, idx.size, regime, kind, rho)
            if (kind == "act") == (regime == "exact_lo_x"):
                side.append(ws[idx])
            if P["blend"] >= 0:
                b0 = (P["blend"] - WS_BASE) // 4
                ws[b0:b0 + P["C"]] = data(rng, P["C"], regime, "blend")
    grads = np.full(W["grads_n"], SENTINEL, np.float32)
    out = wgrad_outputs(W["groups"])
    grads[out] = data(rng, out.size, "exact") if regime.startswith("exact") else 0.0
    return {"ws": ws, "par": np.zeros(64, np.float32), "mix": np.zeros(64, np.float32)}, grads, np.concatenate(side or [np.zeros(0)])


# ------------------------------------------------------------------------------------------------
# running one launch
# ------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _arena(nbytes):
    return torch.empty(max(int(nbytes), 256) + 256, dtype=torch.uint8, device="cuda")


def run_conv_case(D, kernel, regime, seed):
    """Runs one conv description on the GPU and checks every output element and the bits of everything else."""
    family = ("simt " if kernel else "wgmma ") + ("dgrad" if D["launch"]["pass"] else "fwd")
    if regime in LO_REGIMES:
        family += " " + regime
    rng = np.random.default_rng(seed)
    mem, side = fill_conv(D, rng, regime)
    text = H.conv_text(D)
    plan = H.plan_conv(text)
    ws_d, par_d, mix_d = _dev(mem["ws"]), _dev(mem["par"]), _dev(mem["mix"])
    arena = _arena(plan["pack_bytes"])
    H.run_conv(text, ws_d.data_ptr(), par_d.data_ptr(), mix_d.data_ptr(), kernel, arena.data_ptr(), arena.numel() - 256, stream())
    torch.cuda.synchronize()
    got = ws_d.cpu().numpy()
    out, _, _ = conv_outputs(D)
    keep = np.ones(got.size, bool)
    keep[out] = False
    assert np.array_equal(got.view(np.uint32)[keep], mem["ws"].view(np.uint32)[keep]), \
        "%s: %d elements outside the output views changed" % (D["name"], int((got.view(np.uint32)[keep] != mem["ws"].view(np.uint32)[keep]).sum()))
    m64 = {k: v.astype(np.float64) for k, v in mem.items()}
    if regime in LO_REGIMES:
        mabs = {k: v.astype(np.float64) for k, v in mem.items()}
        run_launch(mabs, D, "abs")
        assert_lo_regime(D["name"], regime, side, mabs["ws"][out], lo_unit(regime, D["planes"])[0])
    if regime.startswith("exact"):
        fma = np.zeros(got.size, bool)
        run_launch(m64, D, "f32", fma)
        g, r = got[out], m64["ws"][out].astype(np.float32)
        ok = (g == r) | (fma[out] & (np.abs(g.astype(np.float64) - r) <= np.spacing(np.abs(r))))
        assert ok.all(), "%s (%s): %d of %d outputs differ; first at %d: got %r want %r" % (
            D["name"], family, int((~ok).sum()), ok.size, int(np.flatnonzero(~ok)[0]), g[~ok][0], r[~ok][0])
        EXACT[family] += 1
    else:
        run_launch(m64, D, "f64")
        mabs = {k: v.astype(np.float64) for k, v in mem.items()}
        run_launch(mabs, D, "abs")
        rabs = torch.from_numpy(mabs["ws"][out])
        check(family, torch.from_numpy(got[out]), torch.from_numpy(m64["ws"][out]), TAU * rabs, D["name"], rabs)
        if kernel == 0:
            conv_power_check(D, {k: v.astype(np.float64) for k, v in mem.items()}, mabs["ws"])
    COUNTS[family] += 1


def conv_power_check(D, mem, ref_abs):
    """The bound must flag a launch that drops ONE tap of ONE boundary row: that term's contribution (times the smallest
    epilogue factor, the 0.2 slope) exceeds TAU * ref_abs somewhere in the row."""
    L = D["launch"]
    for q in D["cls"]:
        for m in (q["m_hi"] - 1, q["m_lo"]):
            for t in D["terms"][q["term_begin"]:q["term_end"]]:
                P = D["planes"][t["plane"]]
                if not (P["r_lo"] <= m + t["d"] < P["r_hi"]) or t["woff"] < 0:
                    continue
                x = plane_rows(mem, P, 0, np.array([m + t["d"]]))[0]
                W0 = (L["W"] - PAR_BASE) // 4
                Nh = L["pairC"] or L["N"]
                w = mem["par"][W0 + t["woff"] + np.arange(P["C"])[:, None] * L["w_sk"] + np.arange(Nh)[None, :] * L["w_sn"]]
                contrib = 0.2 * np.abs(x @ w)
                base, bst, rst = q["base"], q["bstride"], q["rstride"]
                if L["pairC"] and not (q["lo0"] <= m < q["hi0"]):
                    continue
                idx = (base - WS_BASE) // 4 + m * rst + np.arange(Nh)
                assert (contrib > TAU * ref_abs[idx]).any(), (D["name"], "one dropped tap is below the bound")
                return
    raise AssertionError("%s: no boundary row with a valid tap for the power check" % D["name"])


def run_wgrad_case(W, mode, regime, seed, scale):
    family = ["wgrad bulk+fused colsum", "wgrad bulk+colsum", "wgrad converter-fed", "wgrad simt"][mode]
    if regime in LO_REGIMES:
        family += " " + regime
    rng = np.random.default_rng(seed)
    mem, grads, side = fill_wgrad(W, rng, regime)
    text = H.wgrad_text(W["groups"])
    plan = H.plan_wgrad(text)
    ws_d = _dev(mem["ws"])
    arena = _arena(plan["arena_bytes"])
    results = []
    for rep in range(2 if mode in (0, 1) else 1):
        g_d = _dev(grads)
        H.run_wgrad(text, ws_d.data_ptr(), ws_d.data_ptr(), ws_d.data_ptr(), g_d.data_ptr(), scale, mode, arena.data_ptr(),
                    arena.numel() - 256, stream())
        torch.cuda.synchronize()
        results.append(g_d.cpu().numpy())
    got = results[0]
    if len(results) > 1:
        # mode 1 takes the bias gradient from launch_colsum, whose CTAs add their column sums with float atomics (the engine's
        # WUN_SPLIT_COLSUM=0 form): there only dW is reproducible bit for bit
        same = results[0].view(np.uint32) == results[1].view(np.uint32)
        if mode == 1:
            same[W["groups"][0]["wgrad"]["db"] + np.arange(W["groups"][0]["wgrad"]["N"])] = True
        assert same.all(), "%s: two runs differ at %d elements" % (W["name"], int((~same).sum()))
    assert np.array_equal(ws_d.cpu().numpy().view(np.uint32), mem["ws"].view(np.uint32)), "%s: the workspace changed" % W["name"]
    out = wgrad_outputs(W["groups"])
    keep = np.ones(got.size, bool)
    keep[out] = False
    assert np.array_equal(got.view(np.uint32)[keep], grads.view(np.uint32)[keep]), "%s: gradient elements outside dW / db changed" % W["name"]
    m64 = {k: v.astype(np.float64) for k, v in mem.items()}
    ref = grads.astype(np.float64)
    run_wgrad_layer(m64, W["groups"], ref, "f64", scale)
    if regime in LO_REGIMES:
        rabs = np.zeros_like(ref)
        run_wgrad_layer(m64, W["groups"], rabs, "abs", scale)
        unit, _ = lo_unit(regime, [G["plane"] for G in W["groups"]])
        db = np.zeros(rabs.size, bool)
        for G in W["groups"]:
            db[G["wgrad"]["db"] + np.arange(G["wgrad"]["N"])] = True
        # dW: products of the plane and gradient grids; db: sums of the gradient side alone (LO_BITS or integers)
        units = np.where(db, rabs / (abs(scale) * (LO_BITS if regime == "exact_lo_w" else 1.0)), rabs / (abs(scale) * unit))
        assert_lo_regime(W["name"], regime, side, units[out], 1.0)
    if regime.startswith("exact"):
        g, r = got[out], ref[out]
        ok = g.astype(np.float64) == r
        assert ok.all(), "%s (%s): %d of %d gradient elements differ; first: got %r want %r" % (
            W["name"], family, int((~ok).sum()), ok.size, g[~ok][0], r[~ok][0])
        EXACT[family] += 1
    else:
        rabs = np.zeros_like(ref)
        run_wgrad_layer(m64, W["groups"], rabs, "abs", scale)
        r = torch.from_numpy(rabs[out])
        check(family, torch.from_numpy(got[out]), torch.from_numpy(ref[out]), TAU * r, W["name"], r)
        if mode == 0:
            wgrad_power_check(W, m64, rabs, scale)
    COUNTS[family] += 1


def wgrad_power_check(W, mem, rabs, scale):
    """The bound must flag a wgrad that drops ONE 64-row chunk (the first one of batch item 0 of group 0, tap 0)."""
    G = W["groups"][0]
    g, t = G["wgrad"], G["terms"][0]
    rows = np.arange(g["m_lo"], min(g["m_lo"] + 64, g["m_hi"]))
    X = plane_rows(mem, G["plane"], 0, rows + t["d"])
    Y = plane_rows(mem, G["dpre"], 0, rows)
    contrib = np.abs(scale * (X.T @ Y))
    idx = g["dW"] + t["woff"] + np.arange(G["plane"]["C"])[:, None] * g["w_sk"] + np.arange(g["N"])[None, :]
    assert (contrib > TAU * rabs[idx]).any(), (W["name"], "one dropped chunk is below the bound")


# Device bytes a replay holds per workspace word at its peak: the float32 workspace, its copy from before the launch, the
# expected-bits copy, two float64 copies (reference and ref_abs) and the output index list.
REPLAY_BYTES_PER_WORD = 4 + 4 + 4 + 8 + 8 + 8


def replay_conv_and_wgrad(name, named, ov, batch, nf, prefix="replay "):
    """Runs every conv / dgrad launch and every layer's weight gradient the engine emits for one configuration at `batch` alone,
    on random workspace contents, against the float64 interpreter (bound TAU, every word outside the views unchanged).  The
    kernel families are reported as `prefix` + family.  Returns the number of launches replayed."""
    cfg, t_in, eng, descs = engine(named, ov, batch, nf)
    layers = defaultdict(list)
    for G in eng.wgrad_groups:
        layers[G["wgrad"]["layer"]].append(G)
    margin = 1 << 16
    n_ws = eng.workspace_bytes(batch, True) // 4 + 2 * margin
    need = REPLAY_BYTES_PER_WORD * n_ws
    free = torch.cuda.mem_get_info()[0]
    assert need < 0.9 * free, "%s: the replay needs %.1f GB of device memory, %.1f GB are free" % (name, need / 1e9, free / 1e9)
    gen = torch.Generator(device="cuda").manual_seed(7)
    ws_full = torch.randn(n_ws, device="cuda", generator=gen)
    ws = ws_full[margin:]
    par = torch.randn(eng.param_numel + 64, device="cuda", generator=gen) * 0.1
    mix = torch.randn(batch * t_in * cfg["num_channels"] + 64, device="cuda", generator=gen)
    # (blend vectors of learned upsampling are random here too: the interpreter and the bound take any weights)
    ran = 0
    for D in descs:
        text = H.conv_text(D)
        pc = H.plan_conv(text)
        kernel = 0 if pc["eligible"] else 1
        before = ws_full.clone()
        arena = _arena(pc["pack_bytes"])
        H.run_conv(text, ws.data_ptr(), par.data_ptr(), mix.data_ptr(), kernel, arena.data_ptr(), arena.numel() - 256, stream())
        torch.cuda.synchronize()
        mem = {"ws": before[margin:].double(), "par": par.double(), "mix": mix.double()}
        run_launch(mem, D, "f64")
        ref = mem["ws"]
        mem = {"ws": before[margin:].double(), "par": par.double(), "mix": mix.double()}
        run_launch(mem, D, "abs")
        out, _, _ = conv_outputs(D)
        out_t = torch.as_tensor(out, device="cuda")
        expect = before.clone()
        expect[margin:][out_t] = ws[out_t]
        assert torch.equal(ws_full.view(torch.int32), expect.view(torch.int32)), (name, D["launch"]["layer"], D["launch"]["pass"],
                                                                                  "outside the views")
        del expect
        fam = prefix + ("wgmma " if kernel == 0 else "simt ") + ("dgrad" if D["launch"]["pass"] else "fwd")
        rabs = mem["ws"][out_t]
        check(fam, ws[out_t], ref[out_t], TAU * rabs, "%s layer %d pass %d" % (name, D["launch"]["layer"], D["launch"]["pass"]), rabs)
        COUNTS[fam] += 1
        ran += 1
        ws_full.copy_(before)
    grads = torch.zeros(eng.param_numel + 64, device="cuda")
    for layer, groups in sorted(layers.items()):
        text = H.wgrad_text(groups)
        pw = H.plan_wgrad(text)
        mode = (0 if pw["bulk"] else 2) if pw["eligible"] else 3
        arena = _arena(pw["arena_bytes"])
        grads.zero_()
        H.run_wgrad(text, ws.data_ptr(), par.data_ptr(), mix.data_ptr(), grads.data_ptr(), 1.0, mode, arena.data_ptr(),
                    arena.numel() - 256, stream())
        torch.cuda.synchronize()
        mem = {"ws": ws.double(), "par": par.double(), "mix": mix.double()}
        ref = torch.zeros(grads.numel(), dtype=torch.float64, device="cuda")
        run_wgrad_layer(mem, groups, ref, "f64")
        rabs = torch.zeros_like(ref)
        run_wgrad_layer(mem, groups, rabs, "abs")
        out = torch.as_tensor(wgrad_outputs(groups), device="cuda")
        keep = torch.ones(grads.numel(), dtype=torch.bool, device="cuda")
        keep[out] = False
        assert not grads[keep].any(), (name, layer, "gradient elements outside dW / db changed")
        fam = prefix + ("wgrad" if mode != 3 else "simt wgrad")
        check(fam, grads[out], ref[out], TAU * rabs[out], "%s layer %d wgrad" % (name, layer), rabs[out])
        COUNTS[fam] += 1
        ran += 1
    assert ran > 0
    return ran
