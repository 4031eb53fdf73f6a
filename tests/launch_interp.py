"""A float64 interpreter of the engine's exported launch descriptions (wun_debug_launches: planes, classes, terms - csrc/launch.h;
the weight-gradient groups of each layer).  It follows the exact-fp32 reference kernels (plane_conv_kernel, plane_wgrad_kernel,
colsum_kernel in csrc/kernels_simt.cu) and works on numpy arrays and, for the full-size replays, on torch tensors (float64 on
the GPU: cuBLAS DGEMM is an implementation independent of the kernels under test) - one code path for both.

mem = {"ws", "par", "mix"}: the buffers the exported addresses point into (decode); conv writes go to mem["ws"].
Modes of run_launch / run_wgrad_layer:
  "f64" - the operation in float64 (epilogue included);
  "f32" - the float64 sums, then the kernels' epilogue in float32 in their order (v + bias, fmaxf(0.2f * v, v), v * slope,
          v + old): with inputs whose products and sums are exact in fp32 this is what the kernels must produce bit for bit;
  "abs" - |x| and |w| everywhere and no sign-changing epilogue (bias and the accumulated destination enter as magnitudes,
          LeakyReLU slopes are <= 1 and left out): the per-element magnitude the error bound of the float regime scales with.
"""
import numpy as np

WS_BASE, PAR_BASE, MIX_BASE = 1 << 40, 1 << 41, 1 << 42
SLACK = 1 << 38


def decode(addr):
    """raw exported address -> (buffer name, element offset); offsets may be negative (views that start before their tensor)."""
    if addr >= MIX_BASE - SLACK:
        return "mix", (addr - MIX_BASE) // 4
    if addr >= PAR_BASE - SLACK:
        return "par", (addr - PAR_BASE) // 4
    return "ws", (addr - WS_BASE) // 4


class _Numpy(object):
    def ix(self, a):
        return a

    def arange(self, n):
        return np.arange(n)

    def zeros(self, shape):
        return np.zeros(shape)

    def where(self, c, a, b):
        return np.where(c, a, b)

    def abs(self, a):
        return np.abs(a)


class _Torch(object):
    def __init__(self, like):
        import torch
        self.t, self.dev, self.dtype = torch, like.device, like.dtype

    def ix(self, a):
        return a if isinstance(a, self.t.Tensor) else self.t.as_tensor(a, device=self.dev)

    def arange(self, n):
        return self.t.arange(n, device=self.dev)

    def zeros(self, shape):
        return self.t.zeros(shape, dtype=self.dtype, device=self.dev)

    def where(self, c, a, b):
        return self.t.where(self.ix(c), a, b)

    def abs(self, a):
        return a.abs()


def _be(buf):
    return _Numpy() if isinstance(buf, np.ndarray) else _Torch(buf)


def plane_rows(mem, P, b, rows, mode="f64"):
    """[len(rows), C] float64: plane rows `rows` (numpy ints) of batch item b, zero outside [r_lo, r_hi); MID planes blend two
    tensor rows (plane_load, kernels_simt.cu)."""
    name, base = decode(P["base"])
    buf = mem[name]
    be = _be(buf)
    C = P["C"]
    out = be.zeros((len(rows), C))
    ok = (rows >= P["r_lo"]) & (rows < P["r_hi"])
    r = be.ix(rows[ok])
    idx = base + b * P["bstride"] + r[:, None] * P["rstride"] + be.arange(C)[None, :]
    x = buf[idx]
    absolute = mode == "abs"
    if P["kind"] == 1:                                   # PLANE_MID
        if P["mid_mode"] == 0:                           # MID_VALID: r + 1 always exists
            nx = buf[idx + P["rstride"]]
        else:
            has_next = (rows[ok] + 1 < P["xrows"])[:, None]
            nxt = buf[be.where(has_next, idx + P["rstride"], idx)]
            nx = be.where(has_next, nxt, x if P["mid_mode"] == 1 else 0.0 * x)      # MID_CLAMP / MID_ZERO
        if P["blend"] >= 0:
            bname, boff = decode(P["blend"])
            w = mem[bname][boff + be.arange(C)][None, :]
            x = be.abs(w) * be.abs(x) + be.abs(1.0 - w) * be.abs(nx) if absolute else w * x + (1.0 - w) * nx
        else:
            x = (be.abs(x) + be.abs(nx)) * 0.5 if absolute else x + (nx - x) * 0.5
    elif absolute:
        x = be.abs(x)
    out[be.ix(ok)] = x
    return out


def run_launch(mem, D, mode="f64", fma=None):
    """Execute one exported ConvLaunch on mem = {"ws", "par", "mix"} (float64 arrays); writes go to mem["ws"].  mode "f32": `fma`
    (a bool array like mem["ws"], optional) is set where the kernel may fuse the 0.2 slope and the accumulation into one FMA."""
    L, planes, classes, terms = D["launch"], D["planes"], D["cls"], D["terms"]
    N, pairC = L["N"], L["pairC"]
    wname, wbase = decode(L["W"])
    W = mem[wname]
    ws = mem["ws"]
    be = _be(ws)
    absolute, f32 = mode == "abs", mode == "f32"
    for q in classes:
        if q["m_hi"] <= q["m_lo"]:
            continue
        rows = np.arange(q["m_lo"], q["m_hi"])
        for b in range(L["batch"]):
            acc = be.zeros((len(rows), N))
            for t in terms[q["term_begin"]:q["term_end"]]:
                P = planes[t["plane"]]
                X = plane_rows(mem, P, b, rows + t["d"], mode)
                Wt = be.zeros((P["C"], N))
                c = be.arange(P["C"])[:, None]
                if pairC == 0:
                    Wt[:] = W[wbase + t["woff"] + c * L["w_sk"] + be.arange(N)[None, :] * L["w_sn"]]
                else:
                    n = be.arange(pairC)[None, :]
                    if t["woff"] >= 0:
                        Wt[:, :pairC] = W[wbase + t["woff"] + c * L["w_sk"] + n * L["w_sn"]]
                    if t["woff2"] >= 0:
                        Wt[:, pairC:] = W[wbase + t["woff2"] + c * L["w_sk"] + n * L["w_sn"]]
                acc += X @ (be.abs(Wt) if absolute else Wt)
            halves = [(0, N, q["base"], q["bstride"], q["rstride"], q["saved"], q["acc_lo"], q["acc_hi"], q["m_lo"], q["m_hi"])]
            if pairC > 0:
                assert q["pairC"] == pairC and N == 2 * pairC
                halves = [(0, pairC, q["base"], q["bstride"], q["rstride"], q["saved"], q["acc_lo"], q["acc_hi"], q["lo0"], q["hi0"]),
                          (pairC, N, q["base2"], q["bstride2"], q["rstride2"], q["saved2"], q["acc_lo2"], q["acc_hi2"], q["lo1"], q["hi1"])]
            for (n0, n1, base, bstride, rstride, saved, acc_lo, acc_hi, lo, hi) in halves:
                sel = (rows >= lo) & (rows < hi)
                m = rows[sel]
                v = acc[be.ix(sel)][:, n0:n1]
                if f32:
                    v = v.astype(np.float32)
                    assert np.array_equal(v.astype(np.float64), acc[sel][:, n0:n1]), "mode f32: the sums are not exact in fp32"
                else:
                    v = v.clone() if not isinstance(v, np.ndarray) else v.copy()
                _, dbase = decode(base)
                didx = dbase + b * bstride + be.ix(m)[:, None] * rstride + be.arange(n1 - n0)[None, :]
                slope = None
                if L["epilogue"] == 0:                                   # EPI_BIAS_LRELU
                    if L["bias"] >= 0:
                        bname, boff = decode(L["bias"])
                        bias = mem[bname][boff + be.arange(n1 - n0)][None, :]      # pair: the bias repeats per half
                        v = v + (be.abs(bias) if absolute else bias.astype(np.float32) if f32 else bias)
                    if f32:
                        v = np.maximum(np.float32(0.2) * v, v)
                    elif not absolute:
                        v = be.where(0.2 * v > v, 0.2 * v, v)
                elif L["epilogue"] == 1 and saved >= 0 and not absolute:  # EPI_SLOPE
                    sname, sbase = decode(saved)
                    sidx = sbase + b * bstride + be.ix(m)[:, None] * rstride + be.arange(n1 - n0)[None, :]
                    pos = mem[sname][sidx] > 0.0
                    if f32:
                        slope = ~pos
                        v = np.where(pos, v, v * np.float32(0.2))
                    else:
                        v = v * be.where(pos, 1.0 + 0.0 * v, 0.2 + 0.0 * v)
                accum = ((m >= acc_lo) & (m < acc_hi))[:, None]
                old = ws[didx]
                if f32:
                    v = np.where(accum, v + old.astype(np.float32), v).astype(np.float64)
                    if fma is not None and slope is not None:
                        fma[didx] = accum & slope
                else:
                    v = be.where(accum, v + (be.abs(old) if absolute else old), v)
                ws[didx] = v


def run_wgrad_group(mem, G, dW, mode="f64", scale=1.0):
    """One exported (class, plane) weight-gradient group (launch.h WgradLaunch; plane_wgrad_kernel, kernels_simt.cu):
    dW[dW + woff_t + c * w_sk + n * w_sn] += scale * sum_{b, m in [m_lo, m_hi)} plane[b, m + d_t, c] * dpre[b, m, n]."""
    g = G["wgrad"]
    be = _be(dW)
    rows = np.arange(g["m_lo"], g["m_hi"])
    C, N = G["plane"]["C"], g["N"]
    c, n = be.arange(C)[:, None], be.arange(N)[None, :]
    s = abs(scale) if mode == "abs" else scale
    for t in G["terms"]:
        acc = be.zeros((C, N))
        for b in range(g["batch"]):
            Y = plane_rows(mem, G["dpre"], b, rows, mode)[:, :N]
            X = plane_rows(mem, G["plane"], b, rows + t["d"], mode)
            acc += X.T @ Y
        dW[g["dW"] + t["woff"] + c * g["w_sk"] + n * g["w_sn"]] += s * acc


def class_key(G):
    """The class-gradient view of a group: groups of one forward class share it (and its bias contribution)."""
    P = G["dpre"]
    return (G["wgrad"]["layer"], P["base"], P["bstride"], P["rstride"], P["r_lo"], P["r_hi"], P["C"])


def run_wgrad_layer(mem, groups, grads, mode="f64", scale=1.0):
    """A layer's weight gradient (every group) and bias gradient (the column sums of each distinct class-gradient view, once):
    grads[db + n] += scale * sum_{b, m} dpre[b, m, n]."""
    be = _be(grads)
    s = abs(scale) if mode == "abs" else scale
    seen = set()
    for G in groups:
        run_wgrad_group(mem, G, grads, mode, scale)
        if class_key(G) in seen:
            continue
        seen.add(class_key(G))
        g = G["wgrad"]
        rows = np.arange(g["m_lo"], g["m_hi"])
        tot = be.zeros((g["N"],))
        for b in range(g["batch"]):
            tot += plane_rows(mem, G["dpre"], b, rows, mode)[:, :g["N"]].sum(0)
        grads[g["db"] + be.arange(g["N"])] += s * tot
