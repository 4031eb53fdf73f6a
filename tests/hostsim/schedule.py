"""Host-side racecheck of the engine's multi-stream schedule (TEST INFRASTRUCTURE; no GPU).

build()  - compiles tests/hostsim/fake_cudart.cpp (a recording stand-in for the CUDA runtime) and a second build of the engine's
           sources with `nvcc --cudart none` linked against it, under tests/hostsim/_build/ (git-ignored).
trace()  - runs the engine's real host code for a scenario in a subprocess (run_trace.py) and returns the parsed trace.
check()  - replays the trace: vector clocks over streams and events give the happens-before relation of the launches; a shadow
           memory at 4-byte granularity remembers, per word, the last writer and the last reader / atomic-accumulator of every
           stream.  A launch that reads a word must be ordered after its last writer and after the last atomic accumulation of every
           stream; a write after all of those and after the last read of every stream; an atomic accumulation (red.add - they
           commute with each other) after the last writer and the last readers.  Anything else is a race, reported with both launches.
           The same pass checks that every access lies inside its buffer (Shadow.locate) and that no launch reads a workspace /
           gradient / loss word before some launch has written it (an initcheck at launch granularity).
"""
import json
import os
import shutil
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
PKG = os.path.join(REPO, "wave-u-net_b200")
BUILD = os.path.join(HERE, "_build")
SOURCES = ["plan.cpp", "crc32c.cpp", "kernels_simt.cu", "kernels_first.cu", "kernels_feed.cu", "kernels_umma.cu", "engine.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build():
    """Returns the path of the simulated engine library, or None when there is no nvcc / g++ to build it with."""
    if not (os.path.exists(NVCC) and shutil.which("g++")):
        return None
    global BUILD
    try:
        os.makedirs(BUILD, exist_ok=True)
        with open(os.path.join(BUILD, ".writable"), "w"):
            pass
    except OSError:                                          # read-only checkout: build under the temp directory instead
        import tempfile
        BUILD = os.path.join(tempfile.gettempdir(), "wun_hostsim_build")
        os.makedirs(BUILD, exist_ok=True)
    csrc = os.path.join(PKG, "csrc")
    headers = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")]
    fake = os.path.join(BUILD, "libfakecudart.so")
    fake_srcs = [os.path.join(HERE, "fake_cudart.cpp"), os.path.join(HERE, "cpu_kernels.cpp")]
    if _newer(fake, fake_srcs + headers):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, "-I", "/usr/local/cuda/include",
                               "-o", fake] + fake_srcs)
    sim = os.path.join(BUILD, "libwun_sim.so")
    srcs = [os.path.join(csrc, s) for s in SOURCES]
    if _newer(sim, srcs + headers):                          # (the runtime is linked dynamically: no relink when only it changes)
        # the device code is never executed: lowest optimisation levels, the host code is what runs
        subprocess.check_call([NVCC, "--cudart", "none", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-Xptxas", "-O0",
                               "-std=c++17", "-diag-suppress", "177", "-Xcompiler", "-fPIC", "-shared", "-o", sim] + srcs +
                              ["-L" + BUILD, "-lfakecudart", "-Xlinker", "-rpath=$ORIGIN"], cwd=PKG)
    return sim


def trace(scenario, named, overrides, batch, num_frames, env=None):
    """-> (meta, ops): meta = regions / stream handles; ops = parsed trace lines in issue order."""
    sim = build()
    assert sim is not None
    e = dict(os.environ)
    for k in [k for k in e if k.startswith("WUN_")]:
        del e[k]
    e.update(env or {})
    e["WUN_LIB"] = sim
    out = subprocess.run([sys.executable, os.path.join(HERE, "run_trace.py"), scenario, str(batch), str(num_frames),
                          json.dumps(overrides)] + list(named), env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    if out.returncode != 0:
        raise RuntimeError("run_trace.py failed:\n" + out.stderr[-3000:])
    lines = out.stdout.splitlines()
    meta = json.loads(lines[0])
    ops = []
    for ln in lines[1:]:
        f = ln.split(" ")
        if f[0] in ("C", "N"):
            ops.append((f[0], int(f[1])))
        elif f[0] == "E":
            ops.append(("E", int(f[1]), int(f[2])))
        elif f[0] == "S":
            ops.append(("S", int(f[1]), int(f[2])))
        elif f[0] == "L":
            acc = []
            geo = None
            for a in f[3:]:
                p = a.split(":")
                if p[0] == "G":
                    geo = tuple(int(x) for x in p[1:])
                    continue
                if p[0] == "V":
                    acc.append(("V", p[1]) + tuple(int(x) for x in p[2:]))
                elif p[0] == "F":
                    acc.append(("F", p[1], int(p[2]), int(p[3])))
                else:                                   # part of a kernel name that contained a blank
                    raise ValueError("bad access token %r in %r" % (a, ln[:200]))
            ops.append(("L", int(f[1]), f[2], acc, geo))
        elif ln.strip():
            raise ValueError("bad trace line %r" % ln[:200])
    return meta, ops


class Shadow(object):
    """Per region: last writer (stream, seq) and per stream the seq of its last read / atomic accumulation, per 4-byte word."""

    def __init__(self, meta, n_streams):
        self.base = {}
        self.regions = []
        for name, (addr, size) in meta["regions"].items():
            n = (size + 3) // 4 + 64
            self.regions.append((addr, addr + size, name, {
                "w_stream": np.full(n, -1, np.int8), "w_seq": np.zeros(n, np.int16),
                "r": np.zeros((n_streams, n), np.int16), "a": np.zeros((n_streams, n), np.int16)}))

    def locate(self, addr, nbytes):
        for lo, hi, name, st in self.regions:
            if lo <= addr < hi:
                if addr + nbytes > hi:
                    raise AssertionError("access [%d, +%d) runs past region %s" % (addr - lo, nbytes, name))
                return name, st, (addr - lo) // 4
        raise AssertionError("address %d is in no region" % addr)

    def windows(self, acc):
        """-> list of (region name, state, index) where index selects the words of the access (slice or strided-view spec)."""
        out = []
        if acc[0] == "F":
            _, _, addr, nbytes = acc
            name, st, w0 = self.locate(addr, nbytes)
            out.append((name, st, ("s", w0, w0 + (nbytes + 3) // 4)))
        else:
            _, _, base, batch, bstride, rlo, rhi, rstride, C = acc
            for b in range(batch):
                first = base + 4 * (b * bstride + rlo * rstride)
                last = base + 4 * (b * bstride + (rhi - 1) * rstride + C)
                name, st, w0 = self.locate(first, last - first)
                if rstride == C or rhi - rlo == 1:
                    out.append((name, st, ("s", w0, w0 + (rhi - rlo - 1) * rstride + C)))
                else:
                    out.append((name, st, ("v", w0, rhi - rlo, rstride, C)))
        return out


def _sel(arr, idx):
    """View of the selected words of a 1-D state array (no copy)."""
    if idx[0] == "s":
        return arr[idx[1]:idx[2]]
    _, w0, rows, rstride, C = idx
    assert rstride >= C
    return np.lib.stride_tricks.as_strided(arr[w0:], shape=(rows, C), strides=(rstride * arr.itemsize, arr.itemsize))


def check(meta, ops, max_reports=20, init_regions=("ws", "ws_infer", "grads", "loss")):
    """-> (violations, stats).  A violation: dict(op, name, stream, mode, region, other_stream, other_seq, other_name, words).
    Reads of words of `init_regions` that no launch has written yet are violations too (mode "uninitialised": the workspace,
    the gradient buffer and the loss are produced by the library itself - everything else is the caller's input)."""
    streams = {}

    def sid(handle):
        if handle not in streams:
            streams[handle] = len(streams)
        return streams[handle]

    for op in ops:                                          # number the streams first: the shadow needs their count
        if op[0] in ("C",):
            sid(op[1])
        elif op[0] == "E":
            sid(op[2])
        elif op[0] in ("S", "L"):
            sid(op[1])
    S = len(streams)
    shadow = Shadow(meta, S)
    clk = np.zeros((S, S), np.int64)                        # clk[s] = vector clock of the next operation on stream s
    seq = np.zeros(S, np.int64)
    events = {}
    names = {}
    violations = []
    n_launch = 0
    for i, op in enumerate(ops):
        if op[0] in ("C", "N"):
            continue
        if op[0] == "E":
            s = sid(op[2])
            events[op[1]] = clk[s].copy()
            continue
        if op[0] == "S":
            s = sid(op[1])
            if op[2] not in events:
                raise AssertionError("stream waits for event %d that was never recorded (trace line %d)" % (op[2], i))
            clk[s] = np.maximum(clk[s], events[op[2]])
            continue
        _, handle, name, accs = op[:4]
        if name.startswith("UNKNOWN:"):
            raise AssertionError("fake_cudart.cpp cannot decode kernel %s" % name)
        s = sid(handle)
        seq[s] += 1
        assert seq[s] < 32000, "int16 sequence numbers in the shadow memory"
        clk[s, s] = seq[s]
        vc = clk[s].copy()
        names[(s, int(seq[s]))] = (i, name)
        n_launch += 1
        vc_ext = np.concatenate([vc, [np.iinfo(np.int64).max]])      # slot -1: never written
        by_mode = {"R": [], "A": [], "W": []}
        for acc in accs:
            by_mode[acc[1]].append(acc)

        def report(mode, region, other_stream, bad_seq_values, nwords):
            if len(violations) < max_reports:
                oseq = int(bad_seq_values.max())
                other = names.get((other_stream, oseq), (None, "?"))
                violations.append({"op": i, "name": name, "stream": s, "mode": mode, "region": region, "other_stream": other_stream,
                                   "other_op": other[0], "other_name": other[1], "words": int(nwords)})

        for mode in ("R", "A", "W"):                         # all reads of the launch first, its writes last
            for acc in by_mode[mode]:
                for region, st, idx in shadow.windows(acc):
                    ws, wq = _sel(st["w_stream"], idx), _sel(st["w_seq"], idx)
                    if mode in ("R", "A") and region in init_regions:
                        never = ws < 0
                        if never.any() and len(violations) < max_reports:
                            violations.append({"op": i, "name": name, "stream": s, "mode": "uninitialised-" + mode, "region": region,
                                               "other_stream": None, "other_op": None, "other_name": "(no launch wrote these words)",
                                               "words": int(never.sum())})
                    bad = wq > vc_ext[ws]
                    if bad.any():
                        o = int(ws[bad].max())
                        report(mode, region, o, wq[bad & (ws == o)], int(bad.sum()))
                    for t in range(S):
                        if t == s:
                            continue
                        if mode in ("R", "W"):               # vs atomic accumulations of the other streams
                            aq = _sel(st["a"][t], idx)
                            bad = aq > vc[t]
                            if bad.any():
                                report(mode + "-after-A", region, t, aq[bad], int(bad.sum()))
                        if mode in ("A", "W"):               # vs reads of the other streams
                            rq = _sel(st["r"][t], idx)
                            bad = rq > vc[t]
                            if bad.any():
                                report(mode + "-after-R", region, t, rq[bad], int(bad.sum()))
            for acc in by_mode[mode]:                        # then record this launch
                for region, st, idx in shadow.windows(acc):
                    if mode == "R":
                        _sel(st["r"][s], idx)[...] = seq[s]
                    elif mode == "A":
                        _sel(st["a"][s], idx)[...] = seq[s]
                    else:
                        _sel(st["w_stream"], idx)[...] = s
                        _sel(st["w_seq"], idx)[...] = seq[s]
    main = streams.get(meta["main"], 0)
    # fork / join discipline (what CUDA-graph capture of the step requires): when the trace ends, everything every other
    # stream has been given happens-before the caller's stream position
    stats = {"launches": n_launch, "streams": {h: k for h, k in streams.items()}, "per_stream": [int(x) for x in seq],
             "joined_into_caller": bool((clk[main] >= seq).all())}
    return violations, stats


def launch_limit_violations(ops):
    """Launch geometry against the sm_90 limits (the real values the engine passes to the runtime, not the planner's audit):
    <= 1024 threads per CTA, grid y / z <= 65535, dynamic shared memory <= 227 KB and - above the 48 KB default - within what the
    kernel opted in to with cudaFuncSetAttribute, cluster width <= 8 dividing grid.x, non-empty grids."""
    bad = []
    for op in ops:
        if op[0] != "L" or len(op) < 5 or op[4] is None:
            continue
        gx, gy, gz, bx, by, bz, smem, opted, cluster = op[4]
        why = []
        if min(gx, gy, gz, bx, by, bz) < 1:
            why.append("empty grid or block")
        if bx * by * bz > 1024:
            why.append("%d threads per CTA" % (bx * by * bz))
        if gy > 65535 or gz > 65535 or gx > 2147483647:
            why.append("grid (%d, %d, %d)" % (gx, gy, gz))
        if smem > 232448:
            why.append("%d B of dynamic shared memory" % smem)
        if smem > 49152 and opted < smem:
            why.append("%d B of dynamic shared memory but the kernel opted in to %d" % (smem, opted))
        if cluster < 1 or cluster > 8 or gx % max(cluster, 1) != 0:
            why.append("cluster width %d on grid.x %d" % (cluster, gx))
        if why:
            bad.append((op[2].split("(")[0], op[4], why))
    return bad
