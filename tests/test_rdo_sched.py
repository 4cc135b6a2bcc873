"""The RD-loop scheduler: the event model of tools/rdo_sched.py (CPU) and the per-super-block timeline rdo_batch_kernel records (GPU)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import rdo_sched as S  # noqa: E402


def check_dependencies(tr):
    """every super block exactly once; (r, c) starts after (r, c-1) and (r-1, min(c+1, nsbx-1)) have ended"""
    end = {}
    for f, r, c, e in zip(tr["frame"], tr["row"], tr["col"], tr["t_end"]):
        assert (f, r, c) not in end, ("twice", f, r, c)
        end[(int(f), int(r), int(c))] = e
    assert len(end) == sum(int(x) * int(y) for x, y in zip(tr["nsbx"], tr["nsby"]))
    for f, r, c, s in zip(tr["frame"], tr["row"], tr["col"], tr["t_start"]):
        f, r, c = int(f), int(r), int(c)
        nsbx = int(tr["nsbx"][f])
        if c:
            assert s >= end[(f, r, c - 1)], ("left", f, r, c)
        if r:
            assert s >= end[(f, r - 1, min(c + 1, nsbx - 1))], ("up-right", f, r, c)


def frames(rng, shapes, sigma):
    return [np.exp(rng.normal(0, sigma, (h, w))) for w, h in shapes]


@pytest.mark.parametrize("policy", S.POLICIES)
def test_model_respects_dependencies(policy):
    rng = np.random.default_rng(3)
    d = frames(rng, [(15, 9), (4, 3), (1, 5), (7, 1), (15, 9)], 0.7)
    tr = S.replay(d, 6, policy)
    check_dependencies(tr)
    for c in range(6):  # a CTA runs one super block at a time
        m = tr["cta"] == c
        s, e = tr["t_start"][m], tr["t_end"][m]
        o = np.argsort(s)
        assert (s[o][1:] >= e[o][:-1] - 1e-12).all()


@pytest.mark.parametrize("policy", [p for p in S.POLICIES if not p.endswith("-each")])  # continue-in-row: a lone CTA never leaves its row
def test_model_one_frame_one_cta_is_raster_order(policy):
    d = frames(np.random.default_rng(4), [(6, 4)], 0.5)
    tr = S.replay(d, 1, policy)
    assert list(zip(tr["row"], tr["col"])) == [(r, c) for r in range(4) for c in range(6)]
    assert np.isclose(tr["t_end"].max(), d[0].sum())


@pytest.mark.parametrize("nfr,w,h,ctas", [(40, 15, 9, 132), (8, 15, 9, 132), (16, 4, 3, 10), (5, 8, 6, 7), (64, 15, 9, 132)])
def test_longest_path_never_worse_than_lowest_index_on_uniform_costs(nfr, w, h, ctas):
    d = [np.ones((h, w)) for _ in range(nfr)]
    lo = S.replay(d, ctas, "index")["t_end"].max()
    for p in ("longest", "longest-each"):
        lp = S.replay(d, ctas, p)["t_end"].max()
        assert lp <= lo, p
        assert lp >= max(nfr * w * h / ctas, S.chain(d[0])) - 1e-9  # never below the lower bound


def test_idle_split_adds_up():
    d = frames(np.random.default_rng(5), [(15, 9)] * 12, 0.5)
    a = S.analyse(S.replay(d, 20, "longest"), 20, scale=1.0)
    assert np.isclose(a["busy"] + sum(a["idle_share"].values()), 1.0, atol=1e-3)
    assert 0 < a["longest_idle_s"] < a["launch_s"]


def test_trace_entry_point_is_exported():
    import thor_b200 as t
    assert hasattr(t.lib, "tb_rdo_batch_trace")


@pytest.mark.gpu
def test_trace_of_one_launch_over_golden_jobs(tmp_path):
    """four copies of the committed golden jobs in one launch: the trace holds every super block once, in dependency order, and the decisions
    still equal the reference's"""
    import thor_b200 as tb
    from thor_b200 import rdo_jobs as RJ
    from test_rdo_jobs import golden_jobs
    golden_jobs(str(tmp_path))
    jobs = RJ.load_jobs(str(tmp_path))
    L = tb.lib
    L.tb_rdo_batch_create.restype = C.c_void_p
    L.tb_rdo_batch_create.argtypes = [C.c_int, C.c_int]
    L.tb_rdo_batch_upload.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.tb_rdo_batch_run.argtypes = [C.c_void_p, C.c_int]
    L.tb_rdo_batch_download.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.tb_rdo_batch_sync.argtypes = [C.c_void_p]
    L.tb_rdo_batch_grid.argtypes = [C.c_void_p]
    L.tb_rdo_batch_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.tb_rdo_batch_destroy.argtypes = [C.c_void_p]
    L.tb_rdo_last_error.restype = C.c_char_p
    keep = []

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    hosts = [RJ.HostFrame(j, alloc) for _ in range(4) for j in jobs]
    tb.init(0)
    b = L.tb_rdo_batch_create(len(hosts), jobs[0].hdr.sample_bytes)
    assert b, L.tb_rdo_last_error()
    try:
        for s, hf in enumerate(hosts):
            assert L.tb_rdo_batch_upload(b, s, C.byref(hf.desc)) == 0, L.tb_rdo_last_error()
        assert L.tb_rdo_batch_run(b, len(hosts)) == 0, L.tb_rdo_last_error()
        for s, hf in enumerate(hosts):
            assert L.tb_rdo_batch_download(b, s, C.byref(hf.desc)) == 0, L.tb_rdo_last_error()
        assert L.tb_rdo_batch_sync(b) == 0, L.tb_rdo_last_error()
        nsb = sum(hf.job.nsb for hf in hosts)
        assert L.tb_rdo_batch_trace(b, None, 0) == nsb
        rec = np.zeros(nsb, [(k, np.int32) for k in ("frame", "row", "col", "cta")] + [("t_start", np.uint64), ("t_end", np.uint64)])
        assert L.tb_rdo_batch_trace(b, rec.ctypes.data, nsb) == nsb
        grid = int(L.tb_rdo_batch_grid(b))
    finally:
        L.tb_rdo_batch_destroy(b)
    sb = [1 << hf.desc.log2_sb_size for hf in hosts]
    tr = {k: rec[k] for k in rec.dtype.names}
    tr["nsbx"] = np.array([-(-hf.desc.width // s) for hf, s in zip(hosts, sb)])
    tr["nsby"] = np.array([-(-hf.desc.height // s) for hf, s in zip(hosts, sb)])
    assert ((tr["cta"] >= 0) & (tr["cta"] < grid)).all()
    assert (tr["t_end"] >= tr["t_start"]).all()
    check_dependencies(tr)
    for hf in hosts:
        assert hf.check() == {"rec": True, "blk": True, "sb_cost": True}, ("frame", hf.job.frame_num)
