"""Time interp_batch_kernel and intra_batch_kernel on the bench workload (needs a GPU)."""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench as B
import thor_b200 as tb

tb.init(0)
L = tb.lib
rng = np.random.default_rng(2026)
fr = B.synth_frames(rng, B.NREF + 1)
refs = []; tmp = tb.Frame(B.W, B.H, B.ESZ)
for k in range(B.NREF):
    tmp.upload(*fr[k + 1]); r = tb.Frame(B.W, B.H, B.ESZ); tb.check(L.tb_create_reference_frame(r.h, tmp.h)); refs.append(r)
blocks = B.block_grid()
planes = [[r.plane(p) for p in range(3)] for r in refs]
_, total = B.build_interp(tb, blocks, planes, 0, np.random.default_rng(1), 1)
buf = tb.DevBuf(total * B.ESZ + 64)
items, _ = B.build_interp(tb, blocks, planes, buf.ptr, rng)
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream); tb.check(L.tb_set_stream(C.c_void_p(stream.cuda_stream)))
def run(name, sel):
    it = np.ascontiguousarray(items[sel]); d = tb.DevBuf.from_array(it)
    for _ in range(2):
        tb.check(L.tb_interp_batch(d.ptr, len(it), B.ESZ, B.BD, 1))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(3):
        tb.check(L.tb_interp_batch(d.ptr, len(it), B.ESZ, B.BD, 1))
    b.record(stream); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / 3
    px = float((it["width"].astype(np.int64) * it["height"]).sum())
    print("%-16s n=%8d  %7.3f ms  %7.2f ns/item  %7.4f ns/px" % (name, len(it), ms, ms * 1e6 / len(it), ms * 1e6 / px))
area = items["width"].astype(np.int64) * items["height"]
run("all", slice(None))
run("luma", items["chroma"] == 0)
run("chroma", items["chroma"] == 1)
run("<=64 px", area <= 64)
run("65..255 px", (area > 64) & (area < 256))
run(">=256 px", area >= 256)
