"""Time me_batch_kernel per coding-block size class of the bench workload (needs a GPU; writes a small table to stdout)."""
import ctypes as C, json, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench as B
import thor_b200 as tb

tb.init(0)
L = tb.lib
rng = np.random.default_rng(2026)
fr = B.synth_frames(rng, B.NREF + 1)
cur = tb.Frame(B.W, B.H, B.ESZ); cur.upload(*fr[0])
refs = []; tmp = tb.Frame(B.W, B.H, B.ESZ)
for k in range(B.NREF):
    tmp.upload(*fr[k + 1]); r = tb.Frame(B.W, B.H, B.ESZ); tb.check(L.tb_create_reference_frame(r.h, tmp.h)); refs.append(r)
blocks = B.block_grid()
items, cands = B.build_me(tb, blocks, cur.plane(0)[0], cur.plane(0)[1], [r.plane(0)[0] for r in refs], refs[0].plane(0)[1], rng)
d_cand = tb.DevBuf.from_array(cands)
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream); tb.check(L.tb_set_stream(C.c_void_p(stream.cuda_stream)))
rows = []
def run(name, sel):
    it = np.ascontiguousarray(items[sel]); d = tb.DevBuf.from_array(it); out = tb.DevBuf(8 * len(it))
    st = tb.DevBuf.from_array(np.zeros(5, np.uint64))
    for _ in range(2):
        tb.check(L.tb_motion_estimate_batch(d.ptr, len(it), d_cand.ptr, B.ESZ, B.BD, 0, 1, B.W, B.H, out.ptr))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(3):
        tb.check(L.tb_motion_estimate_batch(d.ptr, len(it), d_cand.ptr, B.ESZ, B.BD, 0, 1, B.W, B.H, out.ptr))
    b.record(stream); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / 3
    L.tb_me_set_stats(st.ptr)
    tb.check(L.tb_motion_estimate_batch(d.ptr, len(it), d_cand.ptr, B.ESZ, B.BD, 0, 1, B.W, B.H, out.ptr)); torch.cuda.synchronize()
    L.tb_me_set_stats(None)
    s = st.download(np.uint64, 5)
    px = float((it["width"].astype(np.int64) * it["height"]).sum())
    print("%-14s n=%8d  %7.3f ms  %7.1f ns/search  %6.3f ns/px  n_int/search %.1f" % (name, len(it), ms, ms * 1e6 / len(it), ms * 1e6 / px, float(s[1]) / len(it)))
run("all", slice(None))
for s in B.SIZES:
    run("cb%d" % s, items["size"] == s)
for s in (8, 16, 64):
    for (w, h) in ((s, s), (s, s // 2), (s // 2, s), (s // 2, s // 2)):
        run("cb%d pb%dx%d" % (s, w, h), (items["size"] == s) & (items["width"] == w) & (items["height"] == h))
