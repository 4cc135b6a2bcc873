"""Intra candidates with exact ties between intra modes.

With intra_rdo 1 the items of a block's intra-mode search, every (intra mode, tb_param) pair, are its intra candidates, each with index
IDX_INTRA + intra_mode * max_tb + tb_param (thor_b200/csrc/tb_rdo.h, mode_decision_rdo).  On flat content several intra modes predict the same
samples and cost the same, so only that index makes min (cost, index) pick the reference's intra mode, whichever warp evaluated which item.
The content here is flat rectangles with a scene cut, so that intra also wins inside P and B frames:
  CPU  every super block decided by tb_rdo.h over the oracle and by the reference's process_block() must be identical, with one and with eight
       simulated warps (with eight, the items of one block are spread over warps, which is where a wrong tie rule shows);
  GPU  every frame decided in one tb_rdo_encode_frames() launch must return the reference's reconstruction, block state and cost per super block,
       and the leaf lists and coefficients of oracle/librdo_hostcheck.so for the same jobs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from test_dropin_link import HDB, REF

FLAGS = HDB + ["-cdef", "0"]  # tiny frames + CDEF corrupt the reference's header (SURVEY §8c.3)
W, H, N, QP = 128, 136, 9, 32


def flat_yuv(path, w, h, n, bitdepth=8, seed=23):
    """Seeded 4:2:0 content where intra wins with exact ties between intra modes:
      * every plane: large constant rectangles at a few levels, with hard edges between them (on a flat block DC, horizontal, vertical, planar and
        most angular modes predict the same samples, so their RD costs are equal);
      * frame n // 2 + 1 (when n > 2) and the frames after it: a different layout of rectangles, a scene cut, so that intra also wins inside P and
        B frames."""
    rng = np.random.default_rng(seed)
    maxv = (1 << bitdepth) - 1
    levels = [0, maxv // 5, maxv // 2, maxv - maxv // 7, maxv]
    cut = n // 2 + 1 if n > 2 else -1

    def layout():
        planes = []
        for ph, pw in ((h, w), (h // 2, w // 2), (h // 2, w // 2)):
            p = np.full((ph, pw), levels[rng.integers(len(levels))])
            for _ in range(6):
                y0, x0 = int(rng.integers(0, ph)), int(rng.integers(0, pw))
                p[y0:y0 + int(rng.integers(ph // 4, ph)), x0:x0 + int(rng.integers(pw // 4, pw))] = levels[rng.integers(len(levels))]
            planes.append(p)
        return planes
    before, after = layout(), layout()
    with open(path, "wb") as f:
        for k in range(n):
            for p in (after if 0 <= cut <= k else before):
                f.write(p.astype(np.uint8 if bitdepth == 8 else "<u2").tobytes())


needs_check = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_rdocheck")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                                 reason="oracle/_ref/Thorenc_rdocheck not built (make -C oracle ref rdocheck)")
needs_capture = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_capture")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                                   reason="oracle/_ref (reference objects + capture link) not built")


@needs_check
@pytest.mark.parametrize("warps", [1, 8])
def test_flat_content_every_super_block_matches_reference_process_block(tmp_path, warps):
    from test_rdo_host import enc
    tmp = str(tmp_path)
    flat_yuv(os.path.join(tmp, "in.yuv"), W, H, N)
    _, _, err = enc("Thorenc_rdocheck", FLAGS, W, H, N, "chk", tmp, (), {"TB_RDO_VERIFY": "1", "TB_RDO_VERBOSE": "1", "TBR_HOST_WARPS": str(warps)}, qp=QP)
    m = re.search(r"verify: (\d+) super blocks compared with the reference's process_block, (\d+) differ", err)
    assert m, err[-1500:]
    assert (int(m.group(1)), int(m.group(2))) == (((W + 127) // 128) * ((H + 127) // 128) * N, 0), err[-3000:]


@pytest.mark.gpu
@needs_capture
def test_flat_content_on_the_device_equals_reference_and_host_decisions(tmp_path):
    import thor_b200 as tb
    from test_rdo_jobs import capture
    from thor_b200 import rdo_jobs as RJ
    from _libs import host_decisions_of_dir
    jobdir = capture(str(tmp_path), FLAGS, W, H, N, 8, QP, flat_yuv)
    jobs = RJ.load_jobs(jobdir)
    keep = []

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    hosts = [RJ.HostFrame(j, alloc) for j in jobs]
    descs = (RJ.RdoFrame * len(hosts))(*[hf.desc for hf in hosts])
    tb.lib.tb_rdo_encode_frames.argtypes = [C.c_void_p, C.c_int]
    tb.lib.tb_rdo_last_error.restype = C.c_char_p
    assert tb.lib.tb_rdo_encode_frames(descs, len(hosts)) == 0, tb.lib.tb_rdo_last_error()
    bad = [(hf.job.frame_num, r) for hf in hosts for r in [hf.check()] if not all(r.values())]
    assert not bad, "%d of %d frames differ from the reference: %s" % (len(bad), len(hosts), bad)
    want = host_decisions_of_dir(jobdir)
    assert len(want) == len(hosts)
    for g, (check, leaves, count, coeffs) in zip(hosts, want):
        assert check == {"rec": True, "blk": True, "sb_cost": True}, ("frame", g.job.frame_num, "host decisions differ from the reference's")
        d = RJ.leaf_differences(g.leaves, g.leaf_count, g.coeffs, leaves, count, coeffs)
        assert not d, ("frame", g.job.frame_num, d)
