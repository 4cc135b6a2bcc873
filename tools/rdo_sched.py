#!/usr/bin/env python
"""Where the time of one rdo_batch_kernel launch goes, from its per-super-block timeline (tb_rdo_batch_trace; tools/rdo_profile.py --trace FILE writes one).

  python tools/rdo_sched.py TRACE.npz [--sm-mhz 1980]

Reports, on the measured durations:
  busy        sum of super-block time / (CTAs x launch time); the launch runs from the first start to the last end
  idle        split per CTA into ramp-up (before its first super block: no row was ready for it yet), dependency waits (between two of its super
              blocks) and tail (after its last super block: no more work came)
  lower bound max(total super-block time / CTAs, longest dependency chain of any frame)
  longest idle stretch of any CTA, against the kernel's watchdog (6e10 SM clocks without work)
  by frame type (traces that record each frame's type and qp): frames, qps, longest dependency chain and mean super-block time of each type,
              which shows the frames that set the lower bound
  replay      the same durations re-scheduled by an event model of the kernel's claim rule, for several claim policies

The event model: a super block (r, c) is ready when (r, c-1) and (r-1, min(c+1, nsbx-1)) have ended (row r-1 has published min(c+2, nsbx)); an idle
CTA claims the best ready row under the policy and runs its super blocks while the next one is ready (continue-in-row) or, with "-each", only one;
claiming takes no time.  CPU only: no GPU and no library needed."""
import argparse
import heapq
import json
import sys

import numpy as np

WATCHDOG_CLOCKS = 60_000_000_000  # rdo_batch_kernel: a CTA without work for this many SM clocks while work remains ends the launch
TRACE_FIELDS = ("frame", "row", "col", "cta", "t_start", "t_end")
FRAME_TYPES = {0: "I", 1: "P", 2: "B"}
# index: lowest row index (frame-major); longest: longest remaining dependency path (nsbx - p) + 2 (nsby - 1 - row), ties to the lower index;
# weighted: that path times the frame's running mean super-block time.  "-each": one super block per claim (what rdo_batch_kernel does).
POLICIES = ("index", "longest", "longest-each", "weighted", "weighted-each")


def load(path):
    z = np.load(path)
    return {k: z[k] for k in z.files}


def durations(tr):
    """per frame, a (nsby, nsbx) array of the super blocks' measured durations (seconds)"""
    d = [np.zeros((int(tr["nsby"][f]), int(tr["nsbx"][f]))) for f in range(len(tr["nsbx"]))]
    for f, r, c, a, b in zip(tr["frame"], tr["row"], tr["col"], tr["t_start"], tr["t_end"]):
        d[f][r, c] = (int(b) - int(a)) * 1e-9
    return d


def chain(d):
    """length of the longest dependency chain of one frame: F(r, c) = max(F(r, c-1), F(r-1, min(c+1, nsbx-1))) + d(r, c)"""
    nsby, nsbx = d.shape
    F = np.zeros_like(d)
    for r in range(nsby):
        for c in range(nsbx):
            F[r, c] = max(F[r, c - 1] if c else 0.0, F[r - 1, min(c + 1, nsbx - 1)] if r else 0.0) + d[r, c]
    return float(F[-1, -1])


def replay(d, ctas, policy="longest"):
    """schedule the super blocks of the frames d (list of (nsby, nsbx) duration arrays) on `ctas` CTAs; returns a trace dict (times in seconds)"""
    each = policy.endswith("-each")
    base = policy[:-5] if each else policy
    if base not in ("index", "longest", "weighted"):
        raise ValueError("unknown policy %r" % policy)
    rows = [(f, r) for f in range(len(d)) for r in range(d[f].shape[0])]
    nsbx = [d[f].shape[1] for f, _ in rows]
    path = [d[f].shape[1] + 2 * (d[f].shape[0] - 1 - r) for f, r in rows]
    prog = [0] * len(rows)
    claimed = [False] * len(rows)
    fsum = [0.0] * len(d)
    fcnt = [0] * len(d)

    def ready(g):
        p = prog[g]
        return not claimed[g] and p < nsbx[g] and (rows[g][1] == 0 or prog[g - 1] >= min(p + 2, nsbx[g]))

    def key(g):
        if base == "index":
            return (0.0, -g)
        rem = path[g] - prog[g]
        if base == "weighted":  # remaining path x the frame's running mean super-block time (all frames alike until one has finished something)
            f = rows[g][0]
            tot = sum(fcnt)
            mean = fsum[f] / fcnt[f] if fcnt[f] else (sum(fsum) / tot if tot else 1.0)
            return (rem * mean, -g)
        return (float(rem), -g)

    out = {k: [] for k in TRACE_FIELDS}
    idle = list(range(ctas))
    heapq.heapify(idle)
    ev = []

    def start(t, cta, g):
        f, r = rows[g]
        c = prog[g]
        claimed[g] = True
        heapq.heappush(ev, (t + float(d[f][r, c]), cta, g, t))

    def dispatch(t):
        while idle:
            cand = [g for g in range(len(rows)) if ready(g)]
            if not cand:
                return
            start(t, heapq.heappop(idle), max(cand, key=key))

    dispatch(0.0)
    while ev:
        t, cta, g, t0 = heapq.heappop(ev)
        f, r = rows[g]
        for k, v in zip(TRACE_FIELDS, (f, r, prog[g], cta, t0, t)):
            out[k].append(v)
        fsum[f] += t - t0
        fcnt[f] += 1
        prog[g] += 1
        claimed[g] = False
        if not each and ready(g):
            start(t, cta, g)
        else:
            heapq.heappush(idle, cta)
        dispatch(t)
    res = {k: np.array(v) for k, v in out.items()}
    res["nsbx"] = np.array([x.shape[1] for x in d])
    res["nsby"] = np.array([x.shape[0] for x in d])
    res["ctas"] = ctas
    return res


def analyse(tr, ctas, scale=1e-9):
    """busy fraction, idle split and longest idle stretch of a trace; scale converts its times to seconds"""
    t0, t1 = float(tr["t_start"].min()), float(tr["t_end"].max())
    T = (t1 - t0) * scale
    dur = (tr["t_end"].astype(np.float64) - tr["t_start"].astype(np.float64)) * scale
    ramp = dep = tail = longest = 0.0
    for c in range(ctas):
        m = tr["cta"] == c
        if not m.any():  # never got work
            ramp += T
            longest = max(longest, T)
            continue
        s = (tr["t_start"][m].astype(np.float64) - t0) * scale
        e = (tr["t_end"][m].astype(np.float64) - t0) * scale
        o = np.argsort(s)
        s, e = s[o], e[o]
        gaps = s[1:] - e[:-1]
        ramp += s[0]
        dep += float(gaps.sum())
        tail += T - e[-1]
        longest = max(longest, s[0], T - e[-1], float(gaps.max()) if gaps.size else 0.0)
    work = float(dur.sum())
    total = ctas * T
    return {"launch_s": round(T, 4), "super_blocks": int(dur.size), "ctas": ctas, "busy": round(work / total, 4),
            "idle_share": {"ramp_up": round(ramp / total, 4), "dependency_wait": round(dep / total, 4), "tail": round(tail / total, 4)},
            "longest_idle_s": round(longest, 4), "work_s": round(work, 4)}


def report(tr, sm_mhz=1980.0):
    ctas = int(tr["ctas"])
    d = durations(tr)
    out = analyse(tr, ctas)
    work = sum(float(x.sum()) for x in d)
    chains = [chain(x) for x in d]
    lb = max(work / ctas, max(chains))
    out["lower_bound_s"] = {"value": round(lb, 4), "work_over_ctas": round(work / ctas, 4), "longest_frame_chain": round(max(chains), 4),
                            "bound": "work" if work / ctas >= max(chains) else "chain"}
    out["launch_over_lower_bound"] = round(out["launch_s"] / lb, 4)
    sb = np.concatenate([x.reshape(-1) for x in d])
    out["super_block_s"] = {"mean": round(float(sb.mean()), 5), "cv": round(float(sb.std() / sb.mean()), 4), "min": round(float(sb.min()), 5), "max": round(float(sb.max()), 5)}
    if "frame_type" in tr:
        out["by_frame_type"] = {}
        for ft in sorted(set(int(v) for v in tr["frame_type"])):
            fs = [f for f in range(len(d)) if int(tr["frame_type"][f]) == ft]
            out["by_frame_type"][FRAME_TYPES.get(ft, str(ft))] = {
                "frames": len(fs), "qp": sorted(set(int(tr["qp"][f]) for f in fs)), "longest_chain_s": round(max(chains[f] for f in fs), 4),
                "mean_super_block_s": round(float(np.concatenate([d[f].reshape(-1) for f in fs]).mean()), 5)}
    out["watchdog_s"] = round(WATCHDOG_CLOCKS / (sm_mhz * 1e6), 1)
    out["replay"] = {}
    for p in POLICIES:
        r = analyse(replay(d, ctas, p), ctas, scale=1.0)
        out["replay"][p] = {"launch_s": r["launch_s"], "busy": r["busy"], "idle_share": r["idle_share"], "over_lower_bound": round(r["launch_s"] / lb, 4)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("trace", help=".npz written by tools/rdo_profile.py --trace")
    ap.add_argument("--sm-mhz", type=float, default=1980.0, help="SM clock that converts the watchdog's clocks to seconds")
    args = ap.parse_args()
    print(json.dumps(report(load(args.trace), args.sm_mhz)))


if __name__ == "__main__":
    sys.exit(main())
