"""The tensor-core (wgmma) conv / dgrad, weight pack, split pass, wgrad and fixed-order reduction kernels - and their CUDA-core
fallbacks - launch by launch against a float64 interpreter of the same launch (tests/launch_interp.py), element by element.

One launch at a time runs through tests/kernels/harness.cu (libwun_kernels.so: the product's planner and launchers, fed the
text that wun_debug_launches writes).  Synthetic launches reach the edges no configuration does (every NPAD / NT, partly filled
last splits, the scalar epilogue, MID boundary rows, empty groups, ...); the planner must accept each one and choose the variant
the case is for.  Replays run every conv and wgrad launch the planner emits for real configurations.  The launch builders and
runners are in tests/conv_launches.py, the bound TAU and the checks in tests/launch_checks.py.

The conv table has, per NPAD and pass, tiles whose K loops leave the weight ring unrefilled, wrap it once and cycle its mbarrier
phases at least twice, and tiles that skip groups; the wgrad table has CTAs of 1 to past 2 * nstages + 1 chunks per stage ring
and orientation.  The host test checks both against the product's own step walk (kernels_umma.h next_step) and planner.

Four input regimes:
  exact      - activations k/4 in [-4, 4], weights integers in [-3, 3], MID blend weights in {1/4, 1/2, 3/4}, power-of-two
               scales: the bf16 hi/lo split and every product are exact and every sum stays below 2^24, so the fp32 result must
               equal the float64 sums bit for bit whatever the MMA order; the epilogue is applied in float32 in the kernels'
               order.  Any indexing error (tap, row, chunk, split column, class, batch item, MID neighbour, accumulate range) is a
               mismatch.  Every lo half is zero here.
  exact_lo_x - activations (wgrad: plane rows) j/2^10 with up to 12 significant bits, most with a non-zero bf16 lo half, against
               exact weights (wgrad: gradient rows); exact_lo_w - the reverse.  One side of each product is exact in bf16, so
               hi*hi + hi*lo + lo*hi is the product; the exact side is sparse enough that the sum of |terms| stays below 2^23
               units of the product grid (MID grid included), so the bits are again those of the float64 sums.  A kernel that
               drops or misplaces a lo half, or reads it from the wrong slab or weight block, is a mismatch.
  float      - random data over a wide dynamic range with mixed signs: |got - ref| <= TAU * ref_abs at every element, ref_abs
               the same launch on |x| and |w|.  A power check proves the bound sees one dropped tap of a boundary row (conv) and
               one dropped 64-row chunk (wgrad).
Memory the contract says is never read holds NaN (rows outside [r_lo, r_hi), gaps between weight slices, rows around views);
every workspace / gradient element outside the launch's outputs must keep its bits; weight and bias gradients are pre-filled
(the contract is +=); every bulk-fed wgrad runs twice and must give the same bits (the fixed-order reduction).

Run with -s to see the case count per kernel family, the worst err / ref_abs of the float regime and the exact matches.
"""
from collections import defaultdict

import numpy as np
import pytest

from configurations import REPLAYS
from conv_launches import LO_REGIMES, conv_desc, lo_fits, p, replay_conv_and_wgrad, run_conv_case, run_wgrad_case, wgrad_layer
from launch_checks import COUNTS, H, engine, gpu_lib, lib_or_skip, print_report, set_env
from launch_interp import WS_BASE, class_key


# ------------------------------------------------------------------------------------------------
# the conv case table
# ------------------------------------------------------------------------------------------------
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
    return cs + schedule_cases()


# ------------------------------------------------------------------------------------------------
# conv cases driven by the K-loop schedule: the weight ring (nbs stages of TB taps) filled, refilled and wrapped
# ------------------------------------------------------------------------------------------------
# N per NPAD: with the 36 row tiles of a schedule launch the planner neither doubles the splits of N <= 94 nor those of
# N = 224 / 256 (two splits of 112 / 128 columns)
SCHED_N = {16: 16, 32: 32, 48: 48, 64: 64, 80: 80, 96: 88, 112: 224, 128: 256}
SCHED_ROWS = [(0, 300), (7, 390), (0, 384), (2, 259)]        # three row tiles per class, the last one partly filled
SCHED_BATCH = 3


def ring(N, rows=SCHED_ROWS, batch=SCHED_BATCH):
    """(NPAD, TB, nbs) the planner chooses for N output columns and these classes (TB and nbs depend on NPAD alone)."""
    probe = conv_desc(dg=False, N=N, batch=batch, planes=[p(16, -3, 400)],
                      classes=[dict(m=m, terms=taps(0, 0, 1)) for m in rows])
    pc = H.plan_conv(H.conv_text(probe))
    return pc["NPAD"], pc["TB"], pc["nbs"]


def k_loop(S, TB, w, odd):
    """Taps per plane of a class whose K loop is exactly S steps, for the planes [16 * w channels, 8 channels, 16 channels]
    (w, 1 and 1 chunks): w * kw + k8 + kn = S steps at kw / k8 / kn steps per chunk, with the 8-channel group between the
    other two whenever S allows.  A group of k steps per chunk takes k * TB taps (a full last step) or (k - 1) * TB + 1 (a
    last step of one tap); `odd` picks which groups end in one tap."""
    if S <= 2:
        kw, k8, kn = 0, 0, S
    else:
        kw = (S - 2) // w
        k8, kn = 1, S - w * kw - 1
    def nt(k, one):
        return 0 if k == 0 else (k - 1) * TB + 1 if one else k * TB
    return [nt(kw, odd), nt(k8, not odd), nt(kn, odd)]


def sched_desc(name, dg, N, planes, class_taps, rows=SCHED_ROWS, pair=None):
    classes = []
    for m, ns in zip(rows, class_taps):
        terms = [tp for pl, n in enumerate(ns) if n for tp in taps(pl, -(n // 2), n)]
        classes.append(dict(m=m, terms=terms, saved=dg, acc=(100, 200) if dg else (0, 0)))
    return conv_desc(name=name, dg=dg, N=N, batch=SCHED_BATCH if pair is None else 2, planes=planes, classes=classes, pair=pair)


def schedule_cases():
    """Per NPAD and pass, tiles of 1, nbs - 1, nbs, nbs + 1, 2 nbs + 1, 3 nbs + 1 and 4 nbs + 1 K steps (the ring is never
    refilled, refilled, wrapped once, and wrapped until its mbarrier phases have cycled twice), a run of nbs + 1 one-step chunks,
    chunks ending in a one-tap step and in a full one, an 8-channel group between wider ones; per NPAD one launch whose tiles
    skip their first, a middle, their last or every group next to tiles of long step runs; pair-merged classes past 2 nbs steps."""
    cs = []
    for npad, N in SCHED_N.items():
        got, TB, nbs = ring(N)
        assert got == npad, (N, got)
        R = max(hi for _, hi in SCHED_ROWS) + 12
        for dg in (False, True):
            sfx = "npad%d_%s" % (npad, "dg" if dg else "fwd")
            for part, w, steps in (("a", 2, (1, nbs - 1, nbs, nbs + 1)), ("b", nbs + 1, (2 * nbs + 1, 3 * nbs + 1, 4 * nbs + 1))):
                planes = [p(16 * w, -12, R), p(8, -12, R), p(16, -12, R)]
                class_taps = [k_loop(S, TB, w, i % 2 == 0) for i, S in enumerate(steps)]
                if part == "b":
                    class_taps.append([1, 0, 0])                  # nbs + 1 one-step chunks and nothing else
                cs.append(sched_desc("sched_%s_%s" % (part, sfx), dg, N, planes, class_taps))
        # plane rows chosen so that in the first class (rows [0, 384)) tile 0 skips the 48-channel group, tile 1 the 8-channel
        # one in the middle and tile 2 the last two, next to tiles of 9 - 13 steps; the second class's tile 2 skips both groups
        planes = [p(48, 200, 400), p(8, -2, 120), p(32, -2, 250)]
        long_ = [2 * TB + 1, 2, TB + 1]
        cs.append(sched_desc("sched_skip_npad%d_%s" % (npad, "dg" if npad % 32 else "fwd"), npad % 32 != 0, N, planes,
                             [long_, [0, 2, TB + 1], [2 * TB + 1, 0, TB + 1], long_],
                             rows=[(0, 384), (0, 384), (100, 390), (5, 300)]))
    # pair-merged classes (one class, two output views): 3 nbs + 1 and 4 nbs + 1 steps
    for N, dg in ((64, False), (80, True)):
        _, TB, nbs = ring(N, rows=[(0, 260)], batch=2)
        w = nbs + 1
        S = 3 * nbs + 1 if dg else 4 * nbs + 1
        ns = k_loop(S, TB, w, dg)
        planes = [p(16 * w, -12, 272), p(8, -12, 272), p(16, -12, 272)]
        nterm = sum(ns)
        cs.append(sched_desc("sched_pair_N%d_%s" % (N, "dg" if dg else "fwd"), dg, N, planes, [ns], rows=[None],
                             pair=dict(h=[(0, 250), (3, 260)], missing=[(0, 1), (nterm - 1, 0)], acc2=(0, 100) if dg else (0, 0),
                                       saved2=dg)))
    return cs


# ------------------------------------------------------------------------------------------------
# the weight-gradient case table
# ------------------------------------------------------------------------------------------------
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
    return cs + ring_wgrad_cases()


# (name, Cp, Cg, groups of the long class): the 2-stage ring of N tiles of 128 (Cg or Cp 128) and the 3-stage one of N tiles of
# 80 (Cg 80 / Cp 80), each side on M and on N; 256-channel M sides (two M tiles), 8 taps (tap sets of 2 or 3) and several
# planes multiply the work of a short reduction, so that chunks_per_cta grows past 2 * nstages + 1 over at most 2048 rows.
RING_LAYERS = [("ns2_swap0", 256, 128, 4), ("ns2_swap1", 128, 256, 4), ("ns3_swap0", 256, 80, 7), ("ns3_swap1", 80, 256, 7)]


def ring_layer(name, Cp, Cg, ngroups, rows_long, rows_short):
    """A long class (rows_long rows, ngroups planes of 8 taps) and a short one (one plane, 2 taps), batch 1."""
    planes = [p(Cp, -4, rows_long + 4) for _ in range(ngroups)] + [p(Cp, -1, rows_short + 1)]
    groups = [(0, j, [(t, t - 4) for t in range(8)]) for j in range(ngroups)] + [(1, ngroups, [(0, -1), (1, 0)])]
    return wgrad_layer(name=name, batch=1, cout=Cg, planes=planes, classes=[(0, rows_long), (0, rows_short)], groups=groups)


def ring_wgrad_cases():
    """Per ring (nstages 2 / 3) and orientation, CTAs of 1, 2, nstages, nstages + 1 and >= 2 nstages + 1 chunks: in one launch
    chunks_per_cta >= 2 nstages + 1 with a shorter last CTA, next to a class of one chunk; in another chunks_per_cta =
    nstages + 1 with a last CTA of nstages chunks, next to a class of 2 chunks.  The long class's length is searched through
    the planner, which sets chunks_per_cta from the launch's work."""
    cs = []
    for name, Cp, Cg, ng in RING_LAYERS:
        for part, short in (("long", 1), ("wrap", 2)):
            for chunks in range(2, 33):
                W = ring_layer("ring_%s_%s" % (part, name), Cp, Cg, ng, 64 * chunks - 5, 64 * short - 3)
                pw = H.plan_wgrad(H.wgrad_text(W["groups"]))
                cpc, ns = pw["groups"][0]["chunks_per_cta"], pw["nstages"]
                if (cpc >= 2 * ns + 1 and chunks % cpc) if part == "long" else (cpc == ns + 1 and chunks % cpc == ns):
                    cs.append(W)
                    break
            else:
                raise AssertionError("no length of the long class gives the %s CTAs of %s" % (part, name))
    return cs


# ------------------------------------------------------------------------------------------------
# host tests (no GPU)
# ------------------------------------------------------------------------------------------------
def test_harness_builds_and_plans_host_only():
    """The harness links the product's kernel sources, and its plan-only entry points run the product's planner without a GPU."""
    lib_or_skip()
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
    lib_or_skip()
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
    _assert_rings_wrap(conv_cases(), wgrad_cases())
    assert [W["name"] for W in wgrad_cases() if not lo_fits(W)] == ["long_rows_b16"]


STEP_CLASSES = ("1", "nbs-1", "nbs", "nbs+1", "2nbs+1", ">=3nbs+1")        # K steps of a conv row tile
CHUNK_CLASSES = ("1", "2", "ns", "ns+1", ">=2ns+1")                      # 64-row chunks of a wgrad CTA


def _step_classes(n, nbs):
    hits = (n == 1, n == nbs - 1, n == nbs, n == nbs + 1, n == 2 * nbs + 1, n >= 3 * nbs + 1)
    return {k for k, hit in zip(STEP_CLASSES, hits) if hit}


def _conv_schedule(cs):
    """What the conv K loops of a case table do with the weight ring, per NPAD, from the steps the product's next_step walks."""
    seen = defaultdict(set)
    for D in cs:
        text = H.conv_text(D)
        npad, ps = H.plan_conv(text)["NPAD"], D["launch"]["pass"]
        st = H.conv_steps(text)
        TB, nbs = st["TB"], st["nbs"]
        tiles = [(qi, t) for qi, q in enumerate(st["cls"]) for t in q["tiles"]]
        longest = max(len(t) for _, t in tiles)
        for qi, t in tiles:
            seen[("steps", ps)].update((npad, k) for k in _step_classes(len(t), nbs))
            if len(t) >= 4 * nbs + 1:                      # the ring's mbarrier phases return to their start twice
                seen["two_phase_cycles"].add(npad)
            if D["launch"]["pairC"] and len(t) > 2 * nbs:
                seen["pair_past_2nbs"].add(ps)
            run = best = 0                                 # consecutive chunks of one step each
            for j, (g, c, t0, nt, _) in enumerate(t):
                last = j + 1 == len(t) or t[j + 1][:2] != (g, c)
                run = run + 1 if t0 == 0 and last else 0
                best = max(best, run)
                if last and t0 > 0 and nt == 1:
                    seen["last_step_one_tap"].add(npad)
                elif last and t0 > 0 and nt == TB:
                    seen["last_step_full"].add(npad)
            if best > nbs:
                seen["one_step_run_past_nbs"].add(npad)
            ng = st["cls"][qi]["ngroups"]
            present = {s[0] for s in t}
            if longest > 2 * nbs:                          # a group skipped next to tiles of long step runs
                if not present:
                    seen["skip_every"].add(npad)
                elif 0 not in present:
                    seen["skip_first"].add(npad)
                if present and ng - 1 not in present:
                    seen["skip_last"].add(npad)
                if {0, ng - 1} <= present and len(present) < ng:
                    seen["skip_middle"].add(npad)
        for q in D["cls"]:
            Cs = [D["planes"][tm["plane"]]["C"] for tm in D["terms"][q["term_begin"]:q["term_end"]]]
            Cs = [c for j, c in enumerate(Cs) if j == 0 or c != Cs[j - 1]]
            if any(Cs[j] == 8 and Cs[j - 1] > 8 and Cs[j + 1] > 8 for j in range(1, len(Cs) - 1)):
                seen["c8_between"].add(npad)
    return seen


def _wgrad_rings(cs):
    """(nstages, swap, chunk class) of every CTA of a wgrad case table, and whether a last CTA along x is shorter."""
    seen = defaultdict(set)
    for W in cs:
        pw = H.plan_wgrad(H.wgrad_text(W["groups"]))
        ns = pw["nstages"]
        for g in pw["groups"]:
            total, cpc, nx = W["batch"] * g["chunks_per_batch"], g["chunks_per_cta"], g["n_ctas_x"]
            last = total - (nx - 1) * cpc
            if last < cpc:
                seen["short_last_cta"].add(ns)
            for n in {cpc, last}:
                hits = (n == 1, n == 2, n == ns, n == ns + 1, n >= 2 * ns + 1)
                seen["chunks"].update((ns, g["swap"], k) for k, hit in zip(CHUNK_CLASSES, hits) if hit)
    return seen


def _assert_rings_wrap(conv, wgrad):
    """The conv weight ring and the wgrad stage ring are filled, refilled and wrapped at every NPAD / nstages: each step-count
    class per NPAD and pass, two full mbarrier phase cycles, a run of one-step chunks past the ring, chunks ending in a one-tap and
    in a full step, an 8-channel group between wider ones, the four group-skip patterns next to long tiles, pair-merged classes
    past 2 nbs steps; each chunks-per-CTA class per nstages and orientation."""
    s = _conv_schedule(conv)
    npads = set(range(16, 129, 16))
    for ps in (0, 1):
        missing = {(n, k) for n in npads for k in STEP_CLASSES} - s[("steps", ps)]
        assert not missing, ("pass", ps, sorted(missing))
    for key in ("two_phase_cycles", "one_step_run_past_nbs", "last_step_one_tap", "last_step_full", "c8_between", "skip_first",
                "skip_middle", "skip_last", "skip_every"):
        assert s[key] >= npads, (key, sorted(npads - s[key]))
    assert s["pair_past_2nbs"] == {0, 1}
    w = _wgrad_rings(wgrad)
    missing = {(ns, sw, k) for ns in (2, 3) for sw in (0, 1) for k in CHUNK_CLASSES} - w["chunks"]
    assert not missing, sorted(missing)
    assert w["short_last_cta"] >= {2, 3}


def test_sixteen_views_is_the_most_a_layer_has_and_fits_one_split_pass():
    """umma_plan_wgrad_split returns 0 (-> the converter-fed wgrad) only above kSplitMaxJobs = 16 distinct operand views, but a
    launch has at most kWgMaxGroups = 8 groups of two views each: the layer with 8 groups and 16 distinct views still takes the
    bulk path, so the converter-fed kernel runs only when WUN_BULK_WGRAD=0 asks for it (its GPU test calls it directly)."""
    lib_or_skip()
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
    eng = engine([named], ov, batch, 512)[2]
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


REGIMES = ["exact", "exact_lo_x", "exact_lo_w", "float"]


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("kernel", [0, 1], ids=["wgmma", "simt"])
def test_conv_launches_match_float64(kernel, regime):
    gpu_lib()
    for k, D in enumerate(conv_cases()):
        if kernel == 1 and D["launch"]["pairC"]:
            continue                                  # pair-merged classes exist only for the tensor-core conv (merge_pair)
        run_conv_case(D, kernel, regime, 1000 + k)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("mode", [0, 1, 2, 3], ids=["bulk_fused", "bulk_colsum", "converter", "simt"])
def test_wgrad_layers_match_float64(mode, regime):
    gpu_lib()
    for k, W in enumerate(wgrad_cases()):
        if mode == 3 and any(len(G["terms"]) > 8 for G in W["groups"]):
            continue
        if regime in LO_REGIMES and not lo_fits(W):
            continue                                  # long_rows_b16: 16k-row bias sums of 12-bit rows would round
        run_wgrad_case(W, mode, regime, 2000 + k, 0.5 if k % 2 else 2.0)


# replays: every conv and wgrad launch the planner emits for real configurations, alone, on random workspace contents
@pytest.mark.gpu
@pytest.mark.parametrize("name,named,ov,batch,nf,env", REPLAYS, ids=[r[0] for r in REPLAYS])
def test_replayed_launches_match_float64(name, named, ov, batch, nf, env, monkeypatch):
    gpu_lib()
    set_env(monkeypatch, env)
    replay_conv_and_wgrad(name, named, ov, batch, nf)


@pytest.mark.gpu
def test_zz_report():
    """Prints the case count per kernel family, the worst err / ref_abs of the float regime and the exact-regime matches."""
    print_report("kernel family")
    assert COUNTS
