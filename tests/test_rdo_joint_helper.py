"""The joint bi-prediction search of an overlapped B-frame block decision on a helper warp.

In B frames at encoder_speed 0, mode_decision_rdo (thor_b200/csrc/tb_rdo.h) hands the joint search (motion_estimate_bi) and its candidate to the last
warp, beside warp 0's bi-prediction chain, when candidate list r0 already holds four entries at the start of the phase; otherwise warp 0 runs it after
the chain, as the reference does.  Both schedules must decide every block as the reference does:
  CPU  every super block decided by tb_rdo.h over the oracle with 1, 3, 4 and 8 simulated warps (TBR_HOST_WARPS) must equal the reference's
       process_block(), on moving synthetic content (the list is usually long enough: mostly the helper) and on flat content with a scene cut (the
       vectors are few and alike, so the list is often short: warp 0); the host build's counters (TBR_HOST_STATS) show that each schedule ran;
  GPU  one launch of the same frames must return the reference's reconstruction, block state and cost per super block, and the leaf lists and
       coefficients of oracle/librdo_hostcheck.so for the same jobs; the kernel's counters show that each schedule ran."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from test_dropin_link import HDB, REF, synth_yuv
from test_rdo_intra_ties import flat_yuv

FLAGS = HDB + ["-cdef", "0"]  # tiny frames + CDEF corrupt the reference's header (SURVEY §8c.3)
CONTENT = {  # name: (clip writer, width, height, frames)
    "synthetic": (synth_yuv, 256, 136, 9),
    "flat": (flat_yuv, 128, 136, 9),
}
# tb_rdo.cu ST_JOINT: the overlapped B-frame decisions whose joint search ran on the helper warp, on warp 0 (include/thor_b200.h TB_RDO_NSTATS)
ST_JOINT = 66

needs_check = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_rdocheck")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                                 reason="oracle/_ref/Thorenc_rdocheck not built (make -C oracle ref rdocheck)")
needs_capture = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_capture")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                                   reason="oracle/_ref (reference objects + capture link) not built")


@needs_check
@pytest.mark.parametrize("warps", [1, 3, 4, 8])
@pytest.mark.parametrize("content", sorted(CONTENT))
def test_every_super_block_matches_reference_process_block(tmp_path, content, warps):
    from test_rdo_host import enc
    make_clip, w, h, n = CONTENT[content]
    tmp = str(tmp_path)
    make_clip(os.path.join(tmp, "in.yuv"), w, h, n)
    _, _, err = enc("Thorenc_rdocheck", FLAGS, w, h, n, "chk", tmp, (),
                    {"TB_RDO_VERIFY": "1", "TB_RDO_VERBOSE": "1", "TBR_HOST_WARPS": str(warps), "TBR_HOST_STATS": "1"})
    m = re.search(r"verify: (\d+) super blocks compared with the reference's process_block, (\d+) differ", err)
    assert m, err[-1500:]
    assert (int(m.group(1)), int(m.group(2))) == (((w + 127) // 128) * ((h + 127) // 128) * n, 0), err[-3000:]
    m = re.search(r"joint bi-prediction searches of overlapped decisions: (\d+) on the helper warp, (\d+) on warp 0", err)
    assert m, err[-1500:]
    on_helper, on_warp0 = int(m.group(1)), int(m.group(2))
    if warps == 1:  # one warp: no overlapped schedule
        assert (on_helper, on_warp0) == (0, 0)
    else:
        assert on_helper > 0 and on_warp0 > 0, (content, warps, on_helper, on_warp0)


@pytest.mark.gpu
@needs_capture
@pytest.mark.parametrize("content", sorted(CONTENT))
def test_one_launch_equals_reference_and_host_decisions(tmp_path, content):
    import thor_b200 as tb
    from test_rdo_jobs import capture
    from thor_b200 import rdo_jobs as RJ
    from _libs import host_decisions_of_dir
    make_clip, w, h, n = CONTENT[content]
    jobdir = capture(str(tmp_path), FLAGS, w, h, n, 8, 32, make_clip)
    jobs = RJ.load_jobs(jobdir)
    keep = []

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    L = tb.lib
    tb.init(0)
    L.tb_rdo_batch_create.restype = C.c_void_p
    L.tb_rdo_batch_create.argtypes = [C.c_int, C.c_int]
    L.tb_rdo_batch_upload.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.tb_rdo_batch_run.argtypes = [C.c_void_p, C.c_int]
    L.tb_rdo_batch_download.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.tb_rdo_batch_sync.argtypes = [C.c_void_p]
    L.tb_rdo_batch_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.tb_rdo_batch_destroy.argtypes = [C.c_void_p]
    L.tb_rdo_last_error.restype = C.c_char_p
    hosts = [RJ.HostFrame(j, alloc) for j in jobs]
    b = L.tb_rdo_batch_create(len(hosts), 1)
    assert b, L.tb_rdo_last_error()
    try:
        for s, hf in enumerate(hosts):
            assert L.tb_rdo_batch_upload(b, s, C.byref(hf.desc)) == 0, L.tb_rdo_last_error()
        assert L.tb_rdo_batch_run(b, len(hosts)) == 0, L.tb_rdo_last_error()
        for s, hf in enumerate(hosts):
            assert L.tb_rdo_batch_download(b, s, C.byref(hf.desc)) == 0, L.tb_rdo_last_error()
        assert L.tb_rdo_batch_sync(b) == 0, L.tb_rdo_last_error()
        st = (C.c_uint64 * (ST_JOINT + 2))()
        assert L.tb_rdo_batch_stats(b, st, len(st)) == len(st)
    finally:
        L.tb_rdo_batch_destroy(b)
    bad = [(hf.job.frame_num, r) for hf in hosts for r in [hf.check()] if not all(r.values())]
    assert not bad, "%d of %d frames differ from the reference: %s" % (len(bad), len(hosts), bad)
    want = host_decisions_of_dir(jobdir)
    assert len(want) == len(hosts)
    for g, (check, leaves, count, coeffs) in zip(hosts, want):
        assert check == {"rec": True, "blk": True, "sb_cost": True}, ("frame", g.job.frame_num, "host decisions differ from the reference's")
        d = RJ.leaf_differences(g.leaves, g.leaf_count, g.coeffs, leaves, count, coeffs)
        assert not d, ("frame", g.job.frame_num, d)
    assert st[ST_JOINT] > 0 and st[ST_JOINT + 1] > 0, (content, st[ST_JOINT], st[ST_JOINT + 1])
