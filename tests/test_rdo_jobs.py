"""RD-loop jobs (SURVEY §8f.1): the capture link (oracle/_ref/Thorenc_capture = the all-reference CPU encoder + the observing shim) and the batched
device RD loop on its jobs.
CPU: the capture encoder's stream equals the plain reference encoder's, its job files parse, and the captured reconstruction is consistent.
GPU: tb_rdo_encode_frames() on ALL frames of a real encode in ONE launch returns, for every frame, the reference's reconstruction, block state and
RD cost per super block (bit-exact)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_dropin_link import HDB, LDB, REF, synth_yuv

needs = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_capture")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                           reason="oracle/_ref (reference objects + capture link) not built")


def capture(tmp, flags, w, h, n, bitdepth=8, qp=32, make_clip=synth_yuv):
    """encode make_clip(path, w, h, n, bitdepth) with the reference encoder and with the capture link; returns the directory of the captured jobs"""
    clip = os.path.join(tmp, "in.yuv")
    make_clip(clip, w, h, n, bitdepth)
    jobs = os.path.join(tmp, "jobs")
    os.makedirs(jobs, exist_ok=True)
    extra = ["-bitdepth", str(bitdepth), "-input_bitdepth", str(bitdepth)] if bitdepth != 8 else []
    common = ["-if", clip, "-width", str(w), "-height", str(h), "-n", str(n), "-qp", str(qp), "-f", "30"] + extra
    r0 = subprocess.run([os.path.join(REF, "Thorenc")] + flags + common + ["-of", os.path.join(tmp, "a.bit"), "-rf", os.path.join(tmp, "a.yuv")], capture_output=True, text=True)
    r1 = subprocess.run([os.path.join(REF, "Thorenc_capture")] + flags + common + ["-of", os.path.join(tmp, "b.bit"), "-rf", os.path.join(tmp, "b.yuv")], capture_output=True,
                        text=True, env=dict(os.environ, TB_RDO_DUMP=jobs, TB_RDO_STATS="1"))
    assert r0.returncode == 0 and r1.returncode == 0, (r0.stderr[-500:], r1.stderr[-500:])
    assert open(os.path.join(tmp, "a.bit"), "rb").read() == open(os.path.join(tmp, "b.bit"), "rb").read(), "the observing shim changed the stream"
    assert "in the reference's process_block" in r1.stderr
    return jobs


@needs
def test_capture_link_is_transparent_and_jobs_parse(tmp_path):
    from thor_b200 import rdo_jobs as RJ  # importing the package needs the built library, not a GPU
    jobs = RJ.load_jobs(capture(str(tmp_path), HDB + ["-cdef", "0"], 256, 136, 9))
    assert len(jobs) == 9
    types = [j.hdr.frame_type for j in jobs]
    assert types[0] == 0 and 1 in types and types.count(2) == 7           # I, P, seven B frames
    for j in jobs:
        assert j.hdr.width == 256 and j.hdr.height == 136 and j.nsb == 4 and len(j.refs) == j.hdr.num_ref
        assert j.blk.shape[0] == (136 // 4) * (256 // 4) and (j.sb_cost > 0).all()
        assert (j.blk["size"] >= 8).all()                                   # every 4x4 cell belongs to a coded block
    b = [j for j in jobs if j.hdr.frame_type == 2][0]
    assert b.hdr.interp_ref == 1 and b.hdr.enable_bipred == 1 and b.hdr.num_ref >= 3
    # a P frame's first reference is the previous reconstruction AFTER the in-loop filters; the job's rec is BEFORE them: only shapes are comparable
    assert b.refs[0][0].shape == (136 + 2 * b.hdr.ref_pad, b.hdr.ref_stride[0])


@pytest.mark.gpu
@needs
@pytest.mark.parametrize("name,flags,w,h,n,bd", [
    ("hdb_8bit", HDB + ["-cdef", "0"], 320, 200, 9, 8),
    ("ldb_8bit", LDB, 320, 200, 4, 8),
    ("hdb_10bit", HDB + ["-cdef", "0"], 256, 136, 9, 10),
])
def test_batched_rd_loop_equals_reference_decisions(tmp_path, name, flags, w, h, n, bd):
    import thor_b200 as tb
    from thor_b200 import rdo_jobs as RJ
    jobs = RJ.load_jobs(capture(str(tmp_path), flags, w, h, n, bd))
    L = tb.lib
    L.tb_rdo_encode_frames.argtypes = [C.c_void_p, C.c_int]
    L.tb_rdo_last_error.restype = C.c_char_p
    keep = []

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    # the whole sequence twice over in one launch: 2 n independent frames (the second copy exercises slots with equal geometry)
    hosts = [RJ.HostFrame(j, alloc) for j in jobs] + [RJ.HostFrame(j, alloc) for j in jobs]
    descs = (RJ.RdoFrame * len(hosts))(*[hf.desc for hf in hosts])
    rc = L.tb_rdo_encode_frames(descs, len(hosts))
    assert rc == 0, L.tb_rdo_last_error()
    for k, hf in enumerate(hosts):
        r = hf.check()
        assert r == {"rec": True, "blk": True, "sb_cost": True}, (name, "frame", hf.job.frame_num, "copy", k // len(jobs), r)


# ---- committed golden jobs (tests/golden/rdo_jobs_*.xz, generated from the reference by tests/golden/make_golden_rdo.py):
#   hdb_128x136        9 frames of 128x136 HDB at qp 32 on smooth content (I, P, seven hierarchical B frames)
#   hdb_hard_q4_10bit  5 frames of 128x136 10-bit HDB at qp 4 on tests/test_rdo_matrix.py:hard_yuv (large coefficients, saturated samples)
#   hdb_q51_12bit      3 frames of 128x136 12-bit HDB at qp 51 on smooth content (an unsplit 128x128 block in every frame)
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_FRAMES = {"hdb_128x136": 9, "hdb_hard_q4_10bit": 5, "hdb_q51_12bit": 3}


def golden_module():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_rdo", os.path.join(GOLDEN_DIR, "make_golden_rdo.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def golden_jobs(tmp, case="hdb_128x136"):
    m = golden_module()
    n = m.unpack(open(m.path(case), "rb").read(), tmp)
    return m, n


def decide_and_check(jobs):
    """all jobs in one tb_rdo_encode_frames() launch; every frame must return the reference's reconstruction, block state and cost per super block,
    and code exactly as oracle/librdo_hostcheck.so's decisions on the same job (leaf lists and coefficients, RJ.leaf_differences)"""
    import thor_b200 as tb
    from thor_b200 import rdo_jobs as RJ
    from _libs import host_decisions
    L = tb.lib
    L.tb_rdo_encode_frames.argtypes = [C.c_void_p, C.c_int]
    L.tb_rdo_last_error.restype = C.c_char_p
    keep = []

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    hosts = [RJ.HostFrame(j, alloc) for j in jobs]
    descs = (RJ.RdoFrame * len(hosts))(*[hf.desc for hf in hosts])
    assert L.tb_rdo_encode_frames(descs, len(hosts)) == 0, L.tb_rdo_last_error()
    for hf in hosts:
        assert hf.check() == {"rec": True, "blk": True, "sb_cost": True}, ("frame", hf.job.frame_num, hf.check())
    for hf, want in zip(hosts, host_decisions(jobs, alloc)):
        assert want.check() == {"rec": True, "blk": True, "sb_cost": True}, ("frame", hf.job.frame_num, "host decisions differ from the reference's")
        d = hf.leaf_differences(want)
        assert not d, ("frame", hf.job.frame_num, d)


def rederive(tmp_path, case):
    m, n = golden_jobs(str(tmp_path), case)
    fresh_dir = tmp_path / "fresh"
    fresh_dir.mkdir()
    fresh = m.capture(str(fresh_dir), case)
    assert n == len(fresh) == GOLDEN_FRAMES[case]
    for k in range(n):
        assert open(os.path.join(str(tmp_path), "frame_%03d.job" % k), "rb").read() == fresh[k], "job %d differs from a fresh capture" % k


@needs
def test_golden_rdo_jobs_are_what_the_reference_writes_today(tmp_path):
    """the fixture is pinned: a fresh capture with the compiled reference reproduces it byte for byte"""
    rederive(tmp_path, "hdb_128x136")


@needs
def test_hard_low_qp_golden_rdo_jobs_are_what_the_reference_writes_today(tmp_path):
    rederive(tmp_path, "hdb_hard_q4_10bit")


@needs
def test_12bit_golden_rdo_jobs_are_what_the_reference_writes_today(tmp_path):
    rederive(tmp_path, "hdb_q51_12bit")


@pytest.mark.parametrize("case", sorted(GOLDEN_FRAMES))
def test_host_decisions_of_the_golden_jobs_code_alike_with_any_warp_count(tmp_path, case):
    """oracle/librdo_hostcheck.so (tb_rdo.h over the oracle; no reference needed) returns the reference's decisions on the committed jobs, and
    its leaf lists and coefficients code identically with one and with eight simulated warps: what RJ.leaf_differences compares does not depend on
    which warp evaluated which candidate, so it can compare the device's eight-warp decisions with the host's"""
    from thor_b200 import rdo_jobs as RJ
    from _libs import host_decisions
    golden_jobs(str(tmp_path), case)
    jobs = RJ.load_jobs(str(tmp_path))
    keep = []

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    one, eight = host_decisions(jobs, alloc, warps=1), host_decisions(jobs, alloc, warps=8)
    for a, b in zip(one, eight):
        assert a.check() == b.check() == {"rec": True, "blk": True, "sb_cost": True}, ("frame", a.job.frame_num)
        assert a.leaf_count.sum() > 0
        assert not b.leaf_differences(a), ("frame", a.job.frame_num, b.leaf_differences(a))


@pytest.mark.gpu
def test_batched_rd_loop_on_the_golden_jobs(tmp_path):
    """the device RD loop against the committed decisions of the reference (no oracle/_ref needed on the GPU box): all nine frames in one launch"""
    from thor_b200 import rdo_jobs as RJ
    golden_jobs(str(tmp_path))
    jobs = RJ.load_jobs(str(tmp_path))
    assert len(jobs) == 9 and [j.hdr.frame_type for j in jobs].count(2) == 7
    decide_and_check(jobs)


@pytest.mark.gpu
def test_batched_rd_loop_on_the_hard_low_qp_golden_jobs(tmp_path):
    """the same on the 10-bit qp 4 hard-content fixture: large coefficients, saturated samples, a scene cut and local motion"""
    from thor_b200 import rdo_jobs as RJ
    golden_jobs(str(tmp_path), "hdb_hard_q4_10bit")
    jobs = RJ.load_jobs(str(tmp_path))
    assert len(jobs) == 5 and all(j.hdr.bitdepth == 10 and j.hdr.qp <= 8 for j in jobs)
    decide_and_check(jobs)


@pytest.mark.gpu
def test_batched_rd_loop_on_the_12bit_golden_jobs(tmp_path):
    """the same on the 12-bit qp 51 fixture: every frame holds an unsplit 128x128 block, and the first frame's is an intra block whose transform's
    box sum wraps in int16 (common/common_kernels.c:1544-1549)"""
    from thor_b200 import rdo_jobs as RJ
    golden_jobs(str(tmp_path), "hdb_q51_12bit")
    jobs = RJ.load_jobs(str(tmp_path))
    assert len(jobs) == 3 and all(j.hdr.bitdepth == 12 and (j.blk["size"] == 128).any() for j in jobs)
    decide_and_check(jobs)
