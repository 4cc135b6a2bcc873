"""Time txfm_chain_kernel per transform size of the bench workload (needs a GPU)."""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench as B
import thor_b200 as tb

tb.init(0)
L = tb.lib
rng = np.random.default_rng(2026)
fr = B.synth_frames(rng, 2)
cur = tb.Frame(B.W, B.H, B.ESZ); cur.upload(*fr[0])
tmp = tb.Frame(B.W, B.H, B.ESZ); tmp.upload(*fr[1]); ref = tb.Frame(B.W, B.H, B.ESZ); tb.check(L.tb_create_reference_frame(ref.h, tmp.h))
rec = tb.Frame(B.W, B.H, B.ESZ)
tus = B.tu_list(B.block_grid())
items = B.build_txfm(tb, tus, [cur.plane(0), cur.plane(1)], [ref.plane(0), ref.plane(1)], [rec.plane(0), rec.plane(1)], rng)
if '--bits' in sys.argv:
    items['fast'] |= tb.TXFM_BITS  # also count the write_coeff bits (SURVEY 8f.2)
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream); tb.check(L.tb_set_stream(C.c_void_p(stream.cuda_stream)))
def run(name, sel):
    it = np.ascontiguousarray(items[sel]); d = tb.DevBuf.from_array(it); out = tb.DevBuf(16 * len(it))
    for _ in range(2):
        tb.check(L.tb_txfm_chain_batch(d.ptr, len(it), B.ESZ, B.BD, out.ptr))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(3):
        tb.check(L.tb_txfm_chain_batch(d.ptr, len(it), B.ESZ, B.BD, out.ptr))
    b.record(stream); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / 3
    px = float((it["size"].astype(np.int64) ** 2).sum())
    res = out.download(tb.TXFM_RESULT, len(it))
    print("%-10s n=%9d  %7.3f ms  %8.2f ns/chain  %7.4f ns/px  cbp!=0: %.2f" % (name, len(it), ms, ms * 1e6 / len(it), ms * 1e6 / px, float((res["cbp"] != 0).mean())))
run("all", slice(None))
for s in (4, 8, 16, 32, 64, 128):
    run("size%d" % s, items["size"] == s)
