"""The tensor-core (wgmma) conv / dgrad, weight pack, split pass, wgrad and fixed-order reduction kernels - and their CUDA-core
fallbacks - launch by launch against a float64 interpreter of the same launch (tests/launch_interp.py), element by element.

One launch at a time runs through tests/kernels/harness.cu (libwun_kernels.so: the product's planner and launchers, fed the
text that wun_debug_launches writes).  Synthetic launches reach the edges no configuration does (every NPAD / NT, partly filled
last splits, the scalar epilogue, MID boundary rows, empty groups, ...); the planner must accept each one and choose the variant
the case is for.  Replays run every conv and wgrad launch the planner emits for real configurations.

Two input regimes:
  exact - activations k/4 in [-4, 4], weights integers in [-3, 3], MID blend weights in {1/4, 1/2, 3/4}, power-of-two scales:
          the bf16 hi/lo split and every product are exact and every sum stays below 2^24, so the fp32 result must equal the
          float64 sums bit for bit whatever the MMA order; the epilogue is applied in float32 in the kernels' order.  Any
          indexing error (tap, row, chunk, split column, class, batch item, MID neighbour, accumulate range) is a mismatch.
  float - random data over a wide dynamic range with mixed signs: |got - ref| <= TAU * ref_abs at every element, ref_abs the
          same launch on |x| and |w|.  A power check proves the bound sees one dropped tap of a boundary row (conv) and one
          dropped 64-row chunk (wgrad).
Memory the contract says is never read holds NaN (rows outside [r_lo, r_hi), gaps between weight slices, rows around views);
every workspace / gradient element outside the launch's outputs must keep its bits; weight and bias gradients are pre-filled
(the contract is +=); every bulk-fed wgrad runs twice and must give the same bits (the fixed-order reduction).

Run with -s to see the case count per kernel family, the worst err / ref_abs of the float regime and the exact matches.
"""
import os
import sys
from collections import defaultdict

import numpy as np
import pytest

import Config
import wun
from launch_interp import PAR_BASE, WS_BASE, class_key, plane_rows, run_launch, run_wgrad_layer
from oracle import wave_unet_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernels"))
import harness as H  # noqa: E402

# 3-MMA split: ~3 * 2^-17 per product; fp32 accumulation over the launch's k16 steps on top.  Worst err / ref_abs measured on
# one H100 80GB HBM3 (700 W power limit): 2.5e-5 (replayed wgrad), 2.4e-5 (synthetic wgmma conv) - 5x below the bound.
TAU = 2.0 ** -13
SENTINEL = np.float32(7.0e30)
GUARD = 64
WORST = defaultdict(float)          # kernel family -> worst err / ref_abs of the float regime
COUNTS = defaultdict(int)           # kernel family -> cases run
EXACT = defaultdict(int)            # kernel family -> exact-regime cases that matched bit for bit


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


def data(rng, n, regime, kind="act"):
    if regime == "exact":
        if kind == "w":
            return rng.integers(-3, 4, n).astype(np.float32)
        if kind == "blend":
            return rng.choice(np.array([0.25, 0.5, 0.75], np.float32), n)
        return (rng.integers(-16, 17, n) / 4.0).astype(np.float32)
    if kind == "blend":
        return rng.uniform(0.0, 1.0, n).astype(np.float32)
    return (rng.standard_normal(n) * 2.0 ** rng.uniform(-6, 6, n)).astype(np.float32)


def fill_conv(D, rng, regime):
    S, L, B = D["synth"], D["launch"], D["launch"]["batch"]
    ws = np.full(S.n["ws"] + GUARD, np.nan, np.float32)
    par = np.full(S.n["par"] + GUARD, np.nan, np.float32)
    for P in D["planes"]:
        idx = plane_reads(P, B)
        ws[idx] = data(rng, idx.size, regime)
        if P["blend"] >= 0:
            b0 = (P["blend"] - WS_BASE) // 4
            ws[b0:b0 + P["C"]] = data(rng, P["C"], regime, "blend")
    W0 = (L["W"] - PAR_BASE) // 4
    Nh = L["pairC"] or L["N"]
    for t in D["terms"]:
        C = D["planes"][t["plane"]]["C"]
        for wo in (t["woff"], t["woff2"] if L["pairC"] else -1):
            if wo >= 0:
                idx = (W0 + wo + np.arange(C)[:, None] * L["w_sk"] + np.arange(Nh)[None, :] * L["w_sn"]).reshape(-1)
                par[idx] = data(rng, idx.size, regime, "w")
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
    return {"ws": ws, "par": par, "mix": np.zeros(64, np.float32)}


# ------------------------------------------------------------------------------------------------
# the conv case table
# ------------------------------------------------------------------------------------------------
def p(C, lo, hi, **kw):
    return dict(C=C, r_lo=lo, r_hi=hi, **kw)


def taps(plane, d0, n):
    return [(plane, d0 + j) for j in range(n)]


def conv_cases():
    cs = []
    # every NPAD, forward and dgrad (N >= 96: enough row tiles that nsplit is not doubled)
    for N in (16, 32, 48, 64, 80, 96, 112, 128):
        for dg in (False, True):
            big = N >= 96
            B, rows = (16, 600) if big else (3, 300)
            cs.append(conv_desc(name="npad%d_%s" % (N, "dg" if dg else "fwd"), dg=dg, N=N, batch=B,
                                planes=[p(24, -2, rows + 3)],
                                classes=[dict(m=(5, 5 + rows), terms=taps(0, -2, 5), saved=dg, acc=(100, 250) if dg else (0, 0))]))
    # output-channel splits: doubled (sparse launch), partly filled last split, nsplit 3 / 4, scalar epilogue (N % 4 != 0)
    for N, B, rows, dg in ((200, 1, 256, False), (264, 2, 300, True), (136, 16, 600, False), (100, 1, 129, True),
                           (98, 1, 200, False), (500, 3, 140, False), (18, 3, 130, True), (20, 1, 64, False), (136, 1, 255, True)):
        cs.append(conv_desc(name="split_N%d_%s" % (N, "dg" if dg else "fwd"), dg=dg, N=N, batch=B, planes=[p(24, 0, rows)],
                            classes=[dict(m=(0, rows), terms=taps(0, -1, 3), saved=dg)]))
    # scalar epilogue by alignment: unaligned output base / row stride not a multiple of 4
    cs.append(conv_desc(name="unaligned_base_fwd", dg=False, N=32, batch=3, planes=[p(16, 0, 300)],
                        classes=[dict(m=(0, 300), terms=taps(0, -1, 3), Ct=40, coff=1)]))
    cs.append(conv_desc(name="odd_rstride_dg", dg=True, N=48, batch=3, planes=[p(8, 0, 257)],
                        classes=[dict(m=(1, 257), terms=taps(0, -3, 4), Ct=51, saved=True, acc=(0, 60))]))
    # C_in tails: 8 (half chunk), 24, 136 and 264 (chunk tails); tap span 24 (rows_alloc 152) with a long K loop
    for C, nt, dg in ((8, 3, False), (24, 25, True), (136, 25, False), (264, 7, True), (136, 25, True)):
        cs.append(conv_desc(name="cin%d_taps%d_%s" % (C, nt, "dg" if dg else "fwd"), dg=dg, N=64, batch=2,
                            planes=[p(C, -12, 400, step=2)],
                            classes=[dict(m=(0, 380), terms=taps(0, -12, nt), saved=dg)]))
    # row ranges: 1, 127, 128, 129, 255 rows and a large one, m_lo != 0; classes of different lengths in one launch
    cs.append(conv_desc(name="rows_1_127_128_129", dg=False, N=48, batch=3, planes=[p(16, 0, 2000)],
                        classes=[dict(m=(7, 8), terms=taps(0, -2, 5)), dict(m=(3, 130), terms=taps(0, -1, 3)),
                                 dict(m=(11, 139), terms=taps(0, 0, 2)), dict(m=(1, 130), terms=taps(0, 1, 2))]))
    cs.append(conv_desc(name="rows_255_large_dg", dg=True, N=32, batch=1, planes=[p(32, 0, 4100), p(16, 3, 500)],
                        classes=[dict(m=(33, 288), terms=taps(0, -1, 3) + taps(1, 0, 2), saved=True, acc=(100, 200)),
                                 dict(m=(1, 4001), terms=taps(0, -2, 5), acc=(0, 1000))]))
    # planes cut mid-tile (r_lo > 0, r_hi inside a tile), negative shifts, 4 planes / groups per class, groups empty for
    # whole tiles (the plane holds only rows [0, 60)), a class whose every group is empty on some tiles
    cs.append(conv_desc(name="four_groups_empty_tiles", dg=False, N=64, batch=3,
                        planes=[p(16, 37, 301), p(24, 0, 60), p(8, -5, 190), p(32, 200, 700)],
                        classes=[dict(m=(0, 640), terms=taps(0, -3, 3) + taps(1, -1, 2) + taps(2, 0, 4) + taps(3, -7, 3)),
                                 dict(m=(0, 520), terms=taps(1, 0, 2))]))
    cs.append(conv_desc(name="two_planes_dg_plain", dg=True, epi=2, N=40, batch=3, planes=[p(24, 10, 250), p(24, 0, 131), p(24, -4, 90)],
                        classes=[dict(m=(0, 260), terms=taps(0, -2, 3) + taps(1, -9, 2) + taps(2, -1, 2), acc=(40, 200)),
                                 dict(m=(2, 140), terms=taps(1, 2, 3))]))
    # MID planes at the tensor's last row: valid / clamp / zero, with and without blend weights
    for mode in (0, 1, 2):
        for blend in (False, True):
            for dg in ((False, True) if mode == 2 else (False,)):
                cs.append(conv_desc(name="mid%d_blend%d_%s" % (mode, blend, "dg" if dg else "fwd"), dg=dg, N=32, batch=3,
                                    planes=[p(24, 0, 261, kind=1, mid_mode=mode, blend=blend), p(16, 0, 262)],
                                    classes=[dict(m=(0, 262), terms=taps(0, -1, 3) + taps(1, 0, 2), saved=dg,
                                                  acc=(200, 262) if dg else (0, 0))]))
    # no bias; batch 16
    cs.append(conv_desc(name="no_bias_b16_one_tap", dg=False, N=24, batch=16, bias=False, planes=[p(16, 0, 200)],
                        classes=[dict(m=(0, 200), terms=taps(0, 0, 1))]))
    # pair-merged classes: unequal half row ranges, taps present in one half only (woff / woff2 = -1)
    cs.append(conv_desc(name="pair_fwd", dg=False, N=48, batch=3, planes=[p(24, -3, 300)],
                        classes=[dict(m=None, terms=taps(0, -3, 6))],
                        pair=dict(h=[(0, 290), (1, 300)], missing=[(0, 1), (5, 0)])))
    cs.append(conv_desc(name="pair_dg", dg=True, N=64, batch=16, planes=[p(32, 0, 200), p(32, 0, 199)],
                        classes=[dict(m=None, terms=taps(0, -2, 3) + taps(1, -3, 3), saved=True, acc=(30, 120))],
                        pair=dict(h=[(0, 200), (5, 199)], missing=[(1, 0), (4, 1)], acc2=(0, 100), saved2=True)))
    return cs


# ------------------------------------------------------------------------------------------------
# synthetic weight-gradient layers
# ------------------------------------------------------------------------------------------------
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


def wgrad_cases():
    cs = []
    # every NT, both orientations (swap = 1: the gradient side is the wider one)
    for NT in (16, 32, 48, 64, 80, 96, 112, 128):
        cs.append(wgrad_layer(name="nt%d_swap0" % NT, batch=2, cout=NT, planes=[p(128, -2, 300)], classes=[(0, 300)],
                              groups=[(0, 0, [(0, -2), (1, -1), (2, 0)])]))
        cs.append(wgrad_layer(name="nt%d_swap1" % NT, batch=3, cout=136, planes=[p(NT, 0, 200)], classes=[(3, 203)],
                              groups=[(0, 0, [(0, -1), (1, 0), (2, 1)])]))
    # several M and N tiles, tap sets, odd row counts, CTAs whose chunks cross batch items, many CTAs along x
    cs.append(wgrad_layer(name="mtiles_ntiles", batch=3, cout=200, planes=[p(200, 0, 333)], classes=[(0, 333)],
                          groups=[(0, 0, [(0, -2), (1, -1), (2, 0), (3, 1), (4, 2)])]))
    cs.append(wgrad_layer(name="tapsets_8taps", batch=5, cout=64, planes=[p(64, -8, 4 * 64 + 17)], classes=[(0, 4 * 64 + 17)],
                          groups=[(0, 0, [(j, j - 8) for j in range(8)])]))
    cs.append(wgrad_layer(name="nt128_3tapsets_m264", batch=2, cout=128, planes=[p(264, -3, 700, step=2)], classes=[(0, 650)],
                          groups=[(0, 0, [(j, j - 3) for j in range(5)])]))
    cs.append(wgrad_layer(name="long_rows_b16", batch=16, cout=24, planes=[p(16, 0, 1000)], classes=[(0, 999)],
                          groups=[(0, 0, [(0, 0), (1, 1)])]))
    # a down block: two classes (even / odd rows) x two planes, shared taps (2 sums per dW element), MID activation planes
    cs.append(wgrad_layer(name="two_classes_two_planes", batch=3, cout=48,
                          planes=[p(24, 0, 330), p(32, 0, 329, kind=1, mid_mode=2, blend=True)], classes=[(0, 300), (20, 250)],
                          groups=[(0, 0, [(0, -2), (1, -1), (2, 0)]), (0, 1, [(0, -1), (1, 0), (2, 1)]),
                                  (1, 0, [(0, -1), (1, 0), (2, 1)]), (1, 1, [(0, -2), (1, -1), (2, 0)])]))
    cs.append(wgrad_layer(name="mid_valid_linear", batch=2, cout=32, planes=[p(40, 0, 260, kind=1, mid_mode=0)], classes=[(0, 250)],
                          groups=[(0, 0, [(0, -1), (1, 0), (2, 1), (3, 2)])]))
    cs.append(wgrad_layer(name="mid_clamp_last_row", batch=3, cout=16, planes=[p(16, 0, 200, kind=1, mid_mode=1)], classes=[(0, 200)],
                          groups=[(0, 0, [(0, 0), (1, 1)])]))
    # 8 groups (2 classes x 4 planes) of 1..8 taps
    cs.append(wgrad_layer(name="eight_groups", batch=2, cout=32, planes=[p(16 + 8 * (j % 3), -j, 180 + j) for j in range(4)],
                          classes=[(0, 150), (1, 171)],
                          groups=[(j // 4, j % 4, [(t, t - j) for t in range(1 + j)]) for j in range(8)]))
    return cs


def fill_wgrad(W, rng, regime):
    S, B = W["synth"], W["batch"]
    ws = np.full(S.n["ws"] + GUARD, np.nan, np.float32)
    seen = set()
    for G in W["groups"]:
        for P in (G["plane"], G["dpre"]):
            if P["base"] in seen:
                continue
            seen.add(P["base"])
            idx = plane_reads(P, B)
            ws[idx] = data(rng, idx.size, regime)
            if P["blend"] >= 0:
                b0 = (P["blend"] - WS_BASE) // 4
                ws[b0:b0 + P["C"]] = data(rng, P["C"], regime, "blend")
    grads = np.full(W["grads_n"], SENTINEL, np.float32)
    out = wgrad_outputs(W["groups"])
    grads[out] = data(rng, out.size, "exact") if regime == "exact" else 0.0
    return {"ws": ws, "par": np.zeros(64, np.float32), "mix": np.zeros(64, np.float32)}, grads


# ------------------------------------------------------------------------------------------------
# running one launch
# ------------------------------------------------------------------------------------------------
def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _arena(nbytes):
    import torch
    return torch.empty(max(int(nbytes), 256) + 256, dtype=torch.uint8, device="cuda")


def check_float(family, got, ref, ref_abs, what):
    err = np.abs(got.astype(np.float64) - ref)
    bad = ~(err <= TAU * ref_abs)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError("%s: %d of %d elements beyond %.1e * ref_abs; first: got %r ref %r ref_abs %r"
                             % (what, int(bad.sum()), got.size, TAU, got[i], ref[i], ref_abs[i]))
    nz = ref_abs > 0
    if nz.any():
        WORST[family] = max(WORST[family], float((err[nz] / ref_abs[nz]).max()))


def run_conv_case(D, kernel, regime, seed):
    """Runs one conv description on the GPU and checks every output element and the bits of everything else."""
    import torch
    family = ("simt " if kernel else "wgmma ") + ("dgrad" if D["launch"]["pass"] else "fwd")
    rng = np.random.default_rng(seed)
    mem = fill_conv(D, rng, regime)
    text = H.conv_text(D)
    plan = H.plan_conv(text)
    ws_d, par_d, mix_d = _dev(mem["ws"]), _dev(mem["par"]), _dev(mem["mix"])
    arena = _arena(plan["pack_bytes"])
    H.run_conv(text, ws_d.data_ptr(), par_d.data_ptr(), mix_d.data_ptr(), kernel, arena.data_ptr(), arena.numel() - 256, _stream())
    torch.cuda.synchronize()
    got = ws_d.cpu().numpy()
    out, _, _ = conv_outputs(D)
    keep = np.ones(got.size, bool)
    keep[out] = False
    assert np.array_equal(got.view(np.uint32)[keep], mem["ws"].view(np.uint32)[keep]), \
        "%s: %d elements outside the output views changed" % (D["name"], int((got.view(np.uint32)[keep] != mem["ws"].view(np.uint32)[keep]).sum()))
    m64 = {k: v.astype(np.float64) for k, v in mem.items()}
    if regime == "exact":
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
        check_float(family, got[out], m64["ws"][out], mabs["ws"][out], D["name"])
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
    import torch
    family = ["wgrad bulk+fused colsum", "wgrad bulk+colsum", "wgrad converter-fed", "wgrad simt"][mode]
    rng = np.random.default_rng(seed)
    mem, grads = fill_wgrad(W, rng, regime)
    text = H.wgrad_text(W["groups"])
    plan = H.plan_wgrad(text)
    ws_d = _dev(mem["ws"])
    arena = _arena(plan["arena_bytes"])
    results = []
    for rep in range(2 if mode in (0, 1) else 1):
        g_d = _dev(grads)
        H.run_wgrad(text, ws_d.data_ptr(), ws_d.data_ptr(), ws_d.data_ptr(), g_d.data_ptr(), scale, mode, arena.data_ptr(),
                    arena.numel() - 256, _stream())
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
    if regime == "exact":
        g, r = got[out], ref[out]
        ok = g.astype(np.float64) == r
        assert ok.all(), "%s (%s): %d of %d gradient elements differ; first: got %r want %r" % (
            W["name"], family, int((~ok).sum()), ok.size, g[~ok][0], r[~ok][0])
        EXACT[family] += 1
    else:
        rabs = np.zeros_like(ref)
        run_wgrad_layer(m64, W["groups"], rabs, "abs", scale)
        check_float(family, got[out], ref[out], rabs[out], W["name"])
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


# ------------------------------------------------------------------------------------------------
# host tests (no GPU)
# ------------------------------------------------------------------------------------------------
def _lib_or_skip():
    if H.stale() and not os.path.exists(H.NVCC):
        pytest.skip("no nvcc to build tests/kernels")
    return H.load()


def test_harness_builds_and_plans_host_only():
    """The harness links the product's kernel sources, and its plan-only entry points run the product's planner without a GPU."""
    _lib_or_skip()
    D = conv_cases()[0]
    pc = H.plan_conv(H.conv_text(D))
    assert pc["eligible"] and pc["NPAD"] == 16 and pc["nsplit"] == 1 and pc["pack_bytes"] > 0
    W = wgrad_cases()[0]
    pw = H.plan_wgrad(H.wgrad_text(W["groups"]))
    assert pw["eligible"] and pw["bulk"] and pw["groups"][0]["NT"] == 16 and pw["arena_bytes"] > pw["split_bytes"]


def _conv_coverage(cs):
    seen = defaultdict(set)
    for D in cs:
        L = D["launch"]
        pc = H.plan_conv(H.conv_text(D))
        assert pc["eligible"], D["name"]
        npad_total = (L["N"] + 15) // 16 * 16
        last = L["N"] - (pc["nsplit"] - 1) * pc["NPAD"]
        seen["npad_pass"].add((pc["NPAD"], L["pass"]))
        seen["nsplit"].add(pc["nsplit"])
        if pc["nsplit"] > (npad_total + 127) // 128:
            seen["doubled"].add(True)
        if last < pc["NPAD"]:
            seen["partial_last_split"].add(True)
        for q in D["cls"]:
            vec = last % 4 == 0 and q["rstride"] % 4 == 0 and ((q["base"] - WS_BASE) % 16) == 0 and q["bstride"] % 4 == 0
            seen["epilogue"].add("vector" if vec else "scalar")
            seen["rows"].add(q["m_hi"] - q["m_lo"])
            if q["m_lo"]:
                seen["m_lo>0"].add(True)
            if q["saved"] >= 0:
                seen["saved"].add(True)
            if L["pass"] and q["saved"] < 0:
                seen["no_saved"].add(True)
            if q["acc_hi"] > q["acc_lo"]:
                seen["accumulate"].add(True)
            planes = {t["plane"] for t in D["terms"][q["term_begin"]:q["term_end"]]}
            seen["planes_per_class"].add(len(planes))
        if len({(q["m_hi"] - q["m_lo"] + 127) // 128 for q in D["cls"]}) > 1:
            seen["unequal_classes"].add(True)
        seen["rows_alloc"].add(pc["rows_alloc"])
        seen["batch"].add(L["batch"])
        seen["epi"].add(L["epilogue"])
        seen["bias"].add(L["bias"] >= 0)
        for P in D["planes"]:
            seen["cin"].add(P["C"])
            if P["r_lo"] > 0:
                seen["r_lo>0"].add(True)
            if P["kind"] == 1:
                seen["mid"].add((P["mid_mode"], P["blend"] >= 0))
        if any(t["d"] < 0 for t in D["terms"]):
            seen["negative_d"].add(True)
        if L["pairC"]:
            seen["pair"].add(L["pass"])
            q = D["cls"][0]
            if (q["lo0"], q["hi0"]) != (q["lo1"], q["hi1"]):
                seen["pair_unequal_halves"].add(True)
            if any(t["woff"] < 0 for t in D["terms"]) and any(t["woff2"] < 0 for t in D["terms"]):
                seen["pair_missing_taps"].add(True)
    return seen


def test_case_table_reaches_every_kernel_variant():
    """Host only: the planner's choices for the whole synthetic case table reach every variant the GPU tests are meant to cover,
    so that a planner change cannot quietly drop one from them."""
    _lib_or_skip()
    s = _conv_coverage(conv_cases())
    assert s["npad_pass"] == {(n, ps) for n in range(16, 129, 16) for ps in (0, 1)}, sorted(s["npad_pass"])
    assert s["nsplit"] >= {1, 2, 3, 4} and s["doubled"] and s["partial_last_split"]
    assert s["epilogue"] == {"vector", "scalar"}
    assert {8, 24} <= s["cin"] and max(s["cin"]) > 128
    assert s["planes_per_class"] >= {1, 2, 3, 4}
    assert max(s["rows_alloc"]) == 152 and min(s["rows_alloc"]) == 128
    assert {1, 127, 128, 129, 255} <= s["rows"] and max(s["rows"]) > 1000 and s["m_lo>0"] and s["r_lo>0"] and s["negative_d"]
    assert s["unequal_classes"] and s["accumulate"] and s["saved"] and s["no_saved"] and s["bias"] == {True, False}
    assert s["mid"] == {(m, b) for m in (0, 1, 2) for b in (False, True)}
    assert s["epi"] == {0, 1, 2} and s["batch"] >= {1, 3, 16}
    assert s["pair"] == {0, 1} and s["pair_unequal_halves"] and s["pair_missing_taps"]
    seen = defaultdict(set)
    for W in wgrad_cases():
        pw = H.plan_wgrad(H.wgrad_text(W["groups"]))
        assert pw["eligible"] and pw["bulk"], W["name"]
        seen["ngroups"].add(pw["ngroups"])
        for G, g in zip(W["groups"], pw["groups"]):
            seen["nt_swap"].add((g["NT"], g["swap"]))
            seen["ntaps"].add(len(G["terms"]))
            if g["n_mtiles"] > 1:
                seen["mtiles"].add(True)
            if g["n_ntiles"] > 1:
                seen["ntiles"].add(True)
            if g["n_tapsets"] > 1:
                seen["tapsets"].add(True)
            if g["n_ctas_x"] > 1:
                seen["ctas_x"].add(True)
            if g["n_ctas_x"] > 1 and g["chunks_per_batch"] % g["chunks_per_cta"]:
                seen["cross_batch"].add(True)
            if (G["wgrad"]["m_hi"] - G["wgrad"]["m_lo"]) % 64:
                seen["odd_rows"].add(True)
            if G["plane"]["kind"] == 1:
                seen["mid"].add(G["plane"]["mid_mode"])
            if any(t["d"] < 0 for t in G["terms"]):
                seen["negative_d"].add(True)
    assert seen["nt_swap"] == {(n, s_) for n in range(16, 129, 16) for s_ in (0, 1)}, sorted(seen["nt_swap"])
    assert seen["mtiles"] and seen["ntiles"] and seen["tapsets"] and seen["ctas_x"] and seen["cross_batch"] and seen["odd_rows"]
    assert seen["mid"] == {0, 1, 2} and seen["negative_d"] and 1 in seen["ngroups"] and 8 in seen["ngroups"]
    assert seen["ntaps"] >= set(range(1, 9))


def test_sixteen_views_is_the_most_a_layer_has_and_fits_one_split_pass():
    """umma_plan_wgrad_split returns 0 (-> the converter-fed wgrad) only above kSplitMaxJobs = 16 distinct operand views, but a
    launch has at most kWgMaxGroups = 8 groups of two views each: the layer with 8 groups and 16 distinct views still takes the
    bulk path, so the converter-fed kernel runs only when WUN_BULK_WGRAD=0 asks for it (its GPU test calls it directly)."""
    _lib_or_skip()
    W = wgrad_layer(name="sixteen_views", batch=2, cout=32, planes=[p(16 + 8 * (j % 3), -j, 180 + j) for j in range(8)],
                    classes=[(j, 150 + j) for j in range(8)], groups=[(j, j, [(t, t - j) for t in range(1 + j)]) for j in range(8)])
    views = {(G["plane"]["base"], G["plane"]["r_lo"], G["plane"]["r_hi"]) for G in W["groups"]} | {class_key(G) for G in W["groups"]}
    assert len(views) == 16
    pw = H.plan_wgrad(H.wgrad_text(W["groups"]))
    assert pw["eligible"] and pw["bulk"] and pw["ngroups"] == 8


PREMISE = [(n, ov) for n in ("baseline", "baseline_diff", "baseline_context", "baseline_stereo", "full", "full_multi_instrument")
           for ov in (dict(num_layers=5),)] + [
    ("baseline_diff", dict(num_layers=4, upsampling="learned", mono_downmix=False)),
    ("baseline", dict(num_layers=4, upsampling="learned")),
    ("full", dict(num_layers=4, context=False)),
]


@pytest.mark.parametrize("batch", [1, 16])
@pytest.mark.parametrize("named,ov", PREMISE, ids=["%s_%s" % (n, "_".join("%s%s" % kv for kv in sorted(o.items()))) for n, o in PREMISE])
def test_each_gradient_element_receives_at_most_two_sums(named, ov, batch):
    """launch_wgrad_reduce is reproducible bit for bit only because every dW / bias element receives at most 2 partial sums (two
    float additions onto zero commute, three do not): per layer, the groups' tap slices cover each dW element at most twice and
    at most 2 distinct class-gradient views feed each bias."""
    cfg = Config.build_config([named], ov, experiment_id=0)["model_config"]
    t_in, _ = O.get_padding(cfg, 512)
    eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
    eng.launch_descriptions(batch)
    by_layer = defaultdict(list)
    for G in eng.wgrad_groups:
        by_layer[G["wgrad"]["layer"]].append(G)
    assert by_layer
    for layer, groups in by_layer.items():
        cnt = np.zeros(eng.param_numel + 64, np.int32)
        for G in groups:
            g = G["wgrad"]
            for t in G["terms"]:
                idx = g["dW"] + t["woff"] + np.arange(G["plane"]["C"])[:, None] * g["w_sk"] + np.arange(g["N"])[None, :] * g["w_sn"]
                np.add.at(cnt, idx.reshape(-1), 1)
        assert cnt.max() <= 2, (layer, int(cnt.max()))
        assert len({class_key(G) for G in groups}) <= 2, layer


# ------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------
def _gpu_lib():
    import torch
    assert torch.cuda.is_available()
    assert os.path.exists(H.LIB) or os.path.exists(H.NVCC), "tests/kernels/_build/libwun_kernels.so is missing and there is no nvcc"
    return H.load()


CONV = conv_cases()
WGRAD = wgrad_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
@pytest.mark.parametrize("kernel", [0, 1], ids=["wgmma", "simt"])
def test_conv_launches_match_float64(kernel, regime):
    _gpu_lib()
    for k, D in enumerate(CONV):
        if kernel == 1 and D["launch"]["pairC"]:
            continue                                  # pair-merged classes exist only for the tensor-core conv (merge_pair)
        run_conv_case(D, kernel, regime, 1000 + k)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
@pytest.mark.parametrize("mode", [0, 1, 2, 3], ids=["bulk_fused", "bulk_colsum", "converter", "simt"])
def test_wgrad_layers_match_float64(mode, regime):
    _gpu_lib()
    for k, W in enumerate(WGRAD):
        if mode == 3 and any(len(G["terms"]) > 8 for G in W["groups"]):
            continue
        run_wgrad_case(W, mode, regime, 2000 + k, 0.5 if k % 2 else 2.0)


# replays: every conv and wgrad launch the planner emits for real configurations, alone, on random workspace contents
MID = [("m4_like_L5", ["baseline_stereo"], dict(num_layers=5), 3, 200, {}),
       ("m5_like_L4", ["full"], dict(num_layers=4, num_initial_filters=16), 2, 123, {}),
       ("m6_like_L4", ["full_multi_instrument"], dict(num_layers=4), 2, 77, {}),
       ("m1_like_L5", ["baseline"], dict(num_layers=5), 3, 256, {}),
       ("same_learned_stereo", ["baseline_diff"], dict(num_layers=4, upsampling="learned", mono_downmix=False), 2, 128, {}),
       ("odd_filters", ["baseline_context"], dict(num_layers=3, filter_size=9, input_filter_size=9, merge_filter_size=3,
                                                   num_initial_filters=10, output_filter_size=3), 2, 50, {})]
FORCE = {"WUN_PAIR_MIN_CTAS": "1", "WUN_PAIR_DGRAD": "1"}
FORCED = [("forced_m4_like_L5", ["baseline_stereo"], dict(num_layers=5), 3, 2000, FORCE),
          ("forced_m5_like_L4", ["full"], dict(num_layers=4, num_initial_filters=16), 2, 1500, FORCE),
          ("forced_m6_like_L4", ["full_multi_instrument"], dict(num_layers=4), 2, 1200, FORCE),
          ("forced_m1_like_L5", ["baseline"], dict(num_layers=5), 3, 4096, FORCE),
          ("forced_same_learned_stereo", ["baseline_diff"], dict(num_layers=4, upsampling="learned", mono_downmix=False), 2, 2048, FORCE)]
FULL = [("M1_full", ["baseline"], {}, 1, None, {}), ("M4_full", ["baseline_stereo"], {}, 1, None, {}),
        ("M5_full", ["full"], {}, 1, None, {}), ("M6_full", ["full_multi_instrument"], {}, 1, None, {}),
        ("M4_full_b16", ["baseline_stereo"], {}, 16, None, {})]
REPLAYS = MID + FORCED + FULL


@pytest.mark.gpu
@pytest.mark.parametrize("name,named,ov,batch,nf,env", REPLAYS, ids=[r[0] for r in REPLAYS])
def test_replayed_launches_match_float64(name, named, ov, batch, nf, env, monkeypatch):
    import torch
    _gpu_lib()
    for k in [k for k in os.environ if k.startswith("WUN_")]:
        monkeypatch.delenv(k)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = Config.build_config(named, ov, experiment_id=0)["model_config"]
    t_in, _ = O.get_padding(cfg, nf or cfg["num_frames"])
    eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
    descs = eng.launch_descriptions(batch)
    layers = defaultdict(list)
    for G in eng.wgrad_groups:
        layers[G["wgrad"]["layer"]].append(G)
    margin = 1 << 16
    n_ws = eng.workspace_bytes(batch, True) // 4 + 2 * margin
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
        H.run_conv(text, ws.data_ptr(), par.data_ptr(), mix.data_ptr(), kernel, arena.data_ptr(), arena.numel() - 256, _stream())
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
        got = ws[out_t].double()
        err = (got - ref[out_t]).abs()
        rabs = mem["ws"][out_t]
        bad = ~(err <= TAU * rabs)
        assert not bad.any(), (name, D["launch"]["layer"], D["launch"]["pass"], int(bad.sum()))
        fam = "replay " + ("wgmma " if kernel == 0 else "simt ") + ("dgrad" if D["launch"]["pass"] else "fwd")
        nz = rabs > 0
        if nz.any():
            WORST[fam] = max(WORST[fam], float((err[nz] / rabs[nz]).max()))
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
                    arena.numel() - 256, _stream())
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
        err = (grads[out].double() - ref[out]).abs()
        bad = ~(err <= TAU * rabs[out])
        assert not bad.any(), (name, layer, "wgrad", int(bad.sum()))
        fam = "replay wgrad"
        nz = rabs[out] > 0
        if nz.any():
            WORST[fam] = max(WORST[fam], float((err[nz] / rabs[out][nz]).max()))
        COUNTS[fam] += 1
        ran += 1
    assert ran > 0


@pytest.mark.gpu
def test_zz_report():
    """Prints the case count per kernel family, the worst err / ref_abs of the float regime and the exact-regime matches."""
    print("\nkernel family                   cases  exact(bit for bit)  worst err/ref_abs (bound %.2e)" % TAU)
    for fam in sorted(COUNTS):
        print("%-30s %6d %10s %22s" % (fam, COUNTS[fam], EXACT.get(fam, "-"), ("%.2e" % WORST[fam]) if fam in WORST else "-"))
    assert COUNTS
