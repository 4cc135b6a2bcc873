#!/usr/bin/env python
"""One launch of rdo_batch_kernel over the inter frames of a captured clip, for ncu / compute-sanitizer:
  ncu --set full --import-source on --clock-control none -k regex:rdo_batch -c 1 -o rdo python tools/rdo_profile.py --size 640x384
Prints the kernel's own counters (cycles per primitive class, work executed).  --copies 5 --size 1920x1080 is the launch bench.py times;
--trace FILE writes the per-super-block timeline of the last launch (tb_rdo_batch_trace) as .npz for tools/rdo_sched.py, with each frame's type and qp."""
import argparse
import ctypes as C
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

# the counters behind bench.py's (include/thor_b200.h TB_RDO_NSTATS): the search phase of an overlapped block decision (tb_rdo.cu ST_X), warp 0 and the last
# warp, each {own searches, (unused), wait at the barrier that ends the phase}; its bi-prediction phase (ST_XB), warp 0 {chain, inter candidates, barrier
# wait} and the last warp {joint search as the helper, inter candidates, barrier wait}; the B-frame decisions whose joint search ran on the helper / warp 0
SEARCH_PHASE_NAMES = ["w0_own_searches", "w0_barrier_wait", "wlast_own_searches", "wlast_barrier_wait"]
BIPRED_PHASE_NAMES = ["w0_chain", "w0_inter_cands", "w0_barrier_wait", "wlast_joint_search", "wlast_inter_cands", "wlast_barrier_wait"]
STAT_NAMES = bench.STAT_NAMES + ["x_w0_own_searches", "x_unused_1", "x_w0_barrier_wait", "x_wlast_own_searches", "x_unused_4", "x_wlast_barrier_wait"] + \
    ["xb_" + n for n in BIPRED_PHASE_NAMES] + ["joint_on_helper", "joint_on_warp0"]
NSTATS = int(re.search(r"#define TB_RDO_NSTATS (\d+)", open(os.path.join(ROOT, "include", "thor_b200.h")).read()).group(1))
assert len(STAT_NAMES) == NSTATS, (len(STAT_NAMES), NSTATS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="hdb")
    ap.add_argument("--size", default="640x384")
    ap.add_argument("--frames", type=int, default=0)
    ap.add_argument("--copies", type=int, default=1)
    ap.add_argument("--launches", type=int, default=1)
    ap.add_argument("--cache", default="/tmp/thor_b200_bench")
    ap.add_argument("--trace", default=None, metavar="FILE", help="write the per-super-block timeline of the last launch (.npz)")
    args = ap.parse_args()
    cfg = bench.Cfg(args.config, tuple(int(v) for v in args.size.split("x")), args.frames or None)
    os.makedirs(args.cache, exist_ok=True)
    jobdir, meta = bench.capture_jobs(cfg, args.cache)
    import thor_b200 as tb
    from thor_b200 import rdo_jobs as RJ
    L = tb.lib
    tb.init(0)
    L.tb_rdo_batch_create.restype = C.c_void_p
    L.tb_rdo_batch_create.argtypes = [C.c_int, C.c_int]
    L.tb_rdo_batch_upload.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.tb_rdo_batch_run.argtypes = [C.c_void_p, C.c_int]
    L.tb_rdo_batch_download.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.tb_rdo_batch_sync.argtypes = [C.c_void_p]
    L.tb_rdo_batch_grid.argtypes = [C.c_void_p]
    L.tb_rdo_batch_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.tb_rdo_batch_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.tb_rdo_last_error.restype = C.c_char_p
    jobs = [j for j in RJ.load_jobs(jobdir) if j.hdr.frame_type != 0]
    keep = []

    def alloc(n):
        a = np.zeros(max(n, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    base = [RJ.HostFrame(j, alloc) for j in jobs]  # copies upload from the same input planes
    hosts = base + [RJ.HostFrame(j, alloc, share_inputs=hf) for _ in range(args.copies - 1) for j, hf in zip(jobs, base)]
    b = L.tb_rdo_batch_create(len(hosts), cfg.ESZ)
    for s, hf in enumerate(hosts):
        assert L.tb_rdo_batch_upload(b, s, C.byref(hf.desc)) == 0, L.tb_rdo_last_error()
    for _ in range(args.launches):
        t = time.time()
        assert L.tb_rdo_batch_run(b, len(hosts)) == 0, L.tb_rdo_last_error()
        for s, hf in enumerate(hosts):
            assert L.tb_rdo_batch_download(b, s, C.byref(hf.desc)) == 0
        assert L.tb_rdo_batch_sync(b) == 0, L.tb_rdo_last_error()
        dt = time.time() - t
    st = (C.c_uint64 * NSTATS)()
    assert L.tb_rdo_batch_stats(b, st, NSTATS) == NSTATS
    d = dict(zip(STAT_NAMES, [int(v) for v in st]))
    px = sum(hf.job.pixels for hf in hosts)
    ok = all(all(hf.check().values()) for hf in hosts)
    out = {"size": args.size, "frames": len(hosts), "ctas": int(L.tb_rdo_batch_grid(b)), "seconds": round(dt, 3), "mpixel_s": round(px / dt / 1e6, 4), "parity_ok": ok,
           "cycles_per_search": round(d["cyc_me"] / max(1, d["searches"])), "cycles_per_txfm_chain": round(d["cyc_tx_chain"] / max(1, d["txfm_chains"])),
           "cycles_per_prediction": round(d["cyc_interp"] / max(1, d["predictions"])), "cycles_per_intra": round(d["cyc_intra"] / max(1, d["intra_predictions"])),
           "warp_cycles_per_super_block": round(d["cyc_total"] * (1 - d["cyc_idle"] / max(1, d["cyc_total"])) / max(1, d["super_blocks"])),
           "share": {k[4:]: round(d[k] / max(1, d["cyc_total"]), 4) for k in bench.STAT_NAMES[:10] + bench.STAT_NAMES[23:40]}, "phase": {k[3:]: round(d[k] / max(1, sum(d[n] for n in bench.STAT_NAMES[40:49])), 4) for k in bench.STAT_NAMES[40:49]}, "me_stage": {k[9:]: round(d[k] / max(1, sum(d[n] for n in bench.STAT_NAMES[49:])), 4) for k in bench.STAT_NAMES[49:]}, "work": {k: d[k] for k in bench.STAT_NAMES[11:23]},
           "search_phase_mcycles": {n: round(d["x_" + n] / 1e6) for n in SEARCH_PHASE_NAMES},
           "bipred_phase_mcycles": {n: round(d["xb_" + n] / 1e6) for n in BIPRED_PHASE_NAMES},
           "joint_search": {"on_helper": d["joint_on_helper"], "on_warp0": d["joint_on_warp0"],
                            "helper_hit_rate": round(d["joint_on_helper"] / max(1, d["joint_on_helper"] + d["joint_on_warp0"]), 4)}}
    if args.trace:
        n = L.tb_rdo_batch_trace(b, None, 0)
        tr = np.zeros(n, [(k, np.int32) for k in ("frame", "row", "col", "cta")] + [("t_start", np.uint64), ("t_end", np.uint64)])
        assert L.tb_rdo_batch_trace(b, tr.ctypes.data, n) == n, L.tb_rdo_last_error()
        sb = [1 << hf.desc.log2_sb_size for hf in hosts]
        np.savez(args.trace, **{k: tr[k] for k in tr.dtype.names}, nsbx=np.array([-(-hf.desc.width // s) for hf, s in zip(hosts, sb)]),
                 nsby=np.array([-(-hf.desc.height // s) for hf, s in zip(hosts, sb)]), ctas=out["ctas"],
                 frame_type=np.array([hf.desc.frame_type for hf in hosts]), qp=np.array([hf.desc.qp for hf in hosts]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
