"""The RD loop across the quantiser range, hard content and encoder options.

One table of cases (CASES) drives every test here:
  CPU  oracle/_ref/Thorenc_rdocheck with TB_RDO_VERIFY=1: every super block of every case, decided by thor_b200/csrc/tb_rdo.h over the plain-C
       oracle and by the reference's process_block() on the same encoder state, must be identical; five cases also run with eight simulated warps.
  GPU  every case captured with the reference (oracle/_ref/Thorenc_capture); all 8-bit frames of all cases decided in ONE tb_rdo_encode_frames()
       launch, the 8-bit frames held in 16-bit samples (-frame_bitdepth 16) in a second, all 10-bit frames in a third, all 12-bit frames in a
       fourth.  Frames of one launch differ in size, qp, speed, options and (8 bits) super-block size.  Every
       frame must return the reference's reconstruction, block state and cost per super block, and the leaf lists and coefficients that
       oracle/librdo_hostcheck.so (tb_rdo.h over the oracle, itself checked against the reference first) returns for the same job: everything the
       bit writer reads.
The cases reach what qp 32 on smooth content does not: large coefficients and saturation in the transform chain (low qp), frames that are nearly
all skipped (qp 51), samples at 0 and 2^bd-1 in prediction, bipred average and reconstruction, intra blocks in inter frames (a scene cut), local
motion, cfl_inter, encoder speeds 1 and 3, block contexts off, no tb split, intra_rdo 0, no early skip, two references, and 12 bits, where the box
sum of a 128x128 transform can wrap in int16 (hdb_q51_12 codes an unsplit 128x128 block in every frame).  Further cases take 64x64 super blocks,
8-bit content in 16-bit frames (where the reference's SIMD edge filters predict 0), B frames without an interpolated reference, the other reorder
structures, a second P frame, P-frame bi-prediction over four references, CfL intra off and pb split off.  The two fast pans hold vectors of 80
samples and more, the first of them negative on both axes, and predict thousands of 4x4 cells from wholly outside the picture (split_mv's clamps).
clip_mv's own limit, 144 samples outside the picture, stays out of the RD loop's reach: a block's search starts from its neighbours' vectors and
extends them by at most the telescope and hexagon range, and tracked motion does not build up to 144 samples in clips of this length.  The
motion searches are tested at that limit on their own (test_oracle_vs_ref.py, test_gpu_parity.py)."""
import ctypes as C
import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from test_dropin_link import HDB, LDB, REF, synth_yuv


def hard_yuv(path, w, h, n, bitdepth=8, seed=11):
    """Seeded 4:2:0 content at the edges of the RD loop:
      * luma: a uniform-noise texture that pans by one row and one column per frame (motion search finds it; every residual is large);
      * the bottom-right quadrant: a second noise texture moving by (-3, +2) per frame, against the background;
      * a 24x24 block at (16, 16) that alternates between 0 and 2^bd-1 every frame;
      * frame n // 2 + 1 (when n > 2): fresh noise everywhere, a scene cut;
      * U: uniform noise; V: every sample either 0 or 2^bd-1."""
    rng = np.random.default_rng(seed)
    maxv = (1 << bitdepth) - 1
    m = 4 * n + 8
    bg = rng.integers(0, maxv + 1, (h + m, w + m))
    fg = rng.integers(0, maxv + 1, (h + m, w + m))
    cut = n // 2 + 1 if n > 2 else -1
    qy, qx = h // 2, w // 2
    with open(path, "wb") as f:
        for k in range(n):
            y = bg[k:k + h, k:k + w].copy()
            y[qy:, qx:] = fg[3 * k:3 * k + h - qy, 2 * (n - k):2 * (n - k) + w - qx]
            y[16:40, 16:40] = maxv if k % 2 else 0
            if k == cut:
                y = rng.integers(0, maxv + 1, (h, w))
            u = rng.integers(0, maxv + 1, (h // 2, w // 2))
            v = rng.integers(0, 2, (h // 2, w // 2)) * maxv
            for p in (y, u, v):
                f.write(p.astype(np.uint8 if bitdepth == 8 else "<u2").tobytes())


def pan_yuv(path, w, h, n, bitdepth=8, seed=13, pan=(-20, -12)):
    """Seeded 4:2:0 content panning by `pan` = (x, y) samples per frame: a smooth, aperiodic field (a ramp plus low-pass noise) that holds
    motion vectors of some 80 samples, negative on both axes for a negative pan, and predicts thousands of 4x4 cells from wholly outside the
    picture.  (Periodic content aliases: vectors then stop at a fraction of the pan.)"""
    rng = np.random.default_rng(seed)
    maxv = (1 << bitdepth) - 1
    fh, fw = h + abs(pan[1]) * n + 16, w + abs(pan[0]) * n + 16
    noise = np.fft.ifft2(np.fft.fft2(rng.normal(0, 1, (fh, fw))) * np.exp(-(np.fft.fftfreq(fh)[:, None] ** 2 + np.fft.fftfreq(fw)[None, :] ** 2) * 2000)).real
    yy, xx = np.mgrid[0:fh, 0:fw]
    field = 0.25 * xx + 0.15 * yy + noise * (60 / noise.std())
    field = (field - field.min()) / (field.max() - field.min()) * (maxv - 32) + 16
    y0, x0 = (abs(pan[1]) * n if pan[1] < 0 else 0), (abs(pan[0]) * n if pan[0] < 0 else 0)
    with open(path, "wb") as f:
        for k in range(n):
            y = field[y0 + pan[1] * k:y0 + pan[1] * k + h, x0 + pan[0] * k:x0 + pan[0] * k + w] + rng.normal(0, 1, (h, w))
            u = field[y0 + pan[1] * k:y0 + pan[1] * k + h:2, x0 + pan[0] * k:x0 + pan[0] * k + w:2] * 0.5 + maxv / 4
            v = maxv - u
            for p in (y, u, v):
                f.write(np.clip(np.rint(p), 0, maxv).astype(np.uint8 if bitdepth == 8 else "<u2").tobytes())


CONTENT = {"synth": synth_yuv, "hard": hard_yuv, "pan_neg": pan_yuv, "pan_pos": lambda path, w, h, n, bitdepth=8: pan_yuv(path, w, h, n, bitdepth, pan=(22, 14))}
HDB0 = HDB + ["-cdef", "0"]   # tiny frames + CDEF corrupt the reference's header (SURVEY §8c.3)
FB16 = ["-frame_bitdepth", "16"]   # 16-bit frames; with 8-bit input the internal bit depth stays 8
SB64 = ["-log2_sb_size", "6"]
CASES = [
    # name               flags                                                         w    h    frames qp bitdepth content
    ("hdb_q4",           HDB0,                                                         128, 136, 9, 4,  8,  "synth"),
    ("hdb_q51",          HDB0,                                                         128, 136, 9, 51, 8,  "synth"),
    ("hdb_q12_hard",     HDB0,                                                         128, 136, 9, 12, 8,  "hard"),
    ("hdb_q4_hard_10",   HDB0,                                                         128, 136, 5, 4,  10, "hard"),
    ("hdb_q51_hard_10",  HDB0,                                                         128, 136, 5, 51, 10, "hard"),
    ("hdb_q32_hard",     HDB0,                                                         128, 136, 9, 32, 8,  "hard"),
    ("cfl_inter",        HDB0 + ["-enable_cfl_inter", "1"],                            128, 136, 9, 32, 8,  "synth"),
    ("cfl_inter_hard",   HDB0 + ["-enable_cfl_inter", "1"],                            128, 136, 5, 22, 8,  "hard"),
    ("speed1",           HDB0 + ["-encoder_speed", "1"],                               128, 136, 9, 32, 8,  "synth"),
    ("speed1_hard_rect", HDB0 + ["-encoder_speed", "1"],                               200, 72,  5, 8,  8,  "hard"),
    ("speed3",           HDB0 + ["-encoder_speed", "3"],                               128, 136, 9, 32, 8,  "synth"),
    ("no_ctx_no_tbsplit", HDB0 + ["-use_block_contexts", "0", "-enable_tb_split", "0"], 128, 136, 9, 32, 8,  "synth"),
    ("intra_rdo0",       HDB0 + ["-intra_rdo", "0"],                                   128, 136, 9, 32, 8,  "synth"),
    ("no_bipred_hard",   HDB0 + ["-enable_bipred", "0"],                               128, 136, 9, 32, 8,  "hard"),
    ("max_ref2",         HDB0 + ["-max_num_ref", "2"],                                 128, 136, 9, 32, 8,  "synth"),
    ("no_early_skip",    HDB0 + ["-early_skip_thr", "0"],                              128, 136, 9, 32, 8,  "synth"),
    ("ldb_q45_hard",     LDB,                                                          256, 136, 4, 45, 8,  "hard"),
    # fast pans, (-20, -12) and (+22, +14) samples per frame: the reference's block state holds vectors of up to 80 / 88 samples and predicts
    # 8916 / 8658 4x4 cells from wholly outside the picture (split_mv's clamps)
    ("hdb_pan_neg",      HDB0,                                                         384, 256, 9, 32, 8,  "pan_neg"),
    ("hdb_pan_pos",      HDB0,                                                         384, 256, 9, 32, 8,  "pan_pos"),
    # 12 bits: box sums of 16 residuals leave int16 (128x128 transforms wrap), the inverse transform's second stage can saturate
    ("hdb_q51_12",       HDB0,                                                         128, 136, 5, 51, 12, "synth"),
    ("hdb_q4_hard_12",   HDB0,                                                         128, 136, 5, 4,  12, "hard"),
    ("hdb_q32_hard_12",  HDB0,                                                         128, 136, 5, 32, 12, "hard"),
    ("speed1_hard_12",   HDB0 + ["-encoder_speed", "1"],                               128, 136, 5, 45, 12, "hard"),
    # 8-bit content in 16-bit frames: the reference's SIMD edge filters predict 0 there (see DESIGN.md §5)
    ("hdb_fb16",         HDB0 + FB16,                                                  128, 136, 5, 32, 8,  "synth"),
    ("hdb_hard_fb16",    HDB0 + FB16,                                                  128, 136, 5, 22, 8,  "hard"),
    ("ldb_fb16",         LDB + FB16,                                                   256, 136, 4, 32, 8,  "synth"),
    # 64x64 super blocks: partial 64-wide columns, speed 2's top-down partition, speed 3's early skip of whole super blocks, 10 bits
    ("hdb_sb64_rect",    HDB0 + SB64,                                                  200, 136, 9, 32, 8,  "synth"),
    ("ldb_sb64",         LDB + SB64,                                                   256, 136, 5, 32, 8,  "synth"),
    ("speed3_sb64_hard", HDB0 + SB64 + ["-encoder_speed", "3"],                        128, 136, 5, 32, 8,  "hard"),
    ("hdb_sb64_10",      HDB0 + SB64,                                                  128, 136, 5, 32, 10, "synth"),
    # other GOP structures: B frames without an interpolated reference, the non-dyadic layout with three reorder pictures (four references with
    # an interpolated one), two reorder pictures (the first two references swapped), and 17 frames (a second P frame, with several references)
    ("hdb_no_interp",    HDB0 + ["-interp_ref", "0"],                                  128, 136, 9, 32, 8,  "synth"),
    ("reorder3_nd",      HDB0 + ["-num_reorder_pics", "3", "-dyadic_coding", "0"],     128, 136, 9, 32, 8,  "synth"),
    ("reorder3_nd_no_interp", HDB0 + ["-num_reorder_pics", "3", "-dyadic_coding", "0", "-interp_ref", "0"], 128, 136, 9, 32, 8, "synth"),
    ("reorder2",         HDB0 + ["-num_reorder_pics", "2"],                            128, 136, 7, 32, 8,  "synth"),
    ("reorder2_no_interp", HDB0 + ["-num_reorder_pics", "2", "-interp_ref", "0"],      128, 136, 7, 32, 8,  "synth"),
    ("hdb_17",           HDB0,                                                         128, 72,  17, 32, 8, "synth"),
    # P frames with bi-prediction over four references, at speeds 2 and 0
    ("ldb_bipred4",      LDB + ["-enable_bipred", "1", "-max_num_ref", "4"],           128, 136, 6, 32, 8,  "synth"),
    ("ldb_bipred4_s0",   LDB + ["-enable_bipred", "1", "-max_num_ref", "4", "-encoder_speed", "0"], 128, 136, 6, 32, 8, "synth"),
    ("no_cfl_intra",     HDB0 + ["-enable_cfl_intra", "0"],                            128, 136, 5, 32, 8,  "synth"),
    ("no_pb_split",      HDB0 + ["-enable_pb_split", "0"],                             128, 136, 5, 32, 8,  "synth"),
]
BY_NAME = {c[0]: c for c in CASES}


def write_clip(tmp, case):
    name, flags, w, h, n, qp, bd, content = case
    CONTENT[content](os.path.join(tmp, "in.yuv"), w, h, n, bd)
    return ("-bitdepth", str(bd), "-input_bitdepth", str(bd)) if bd != 8 else ()


def sb_size(flags):
    return 1 << int(flags[flags.index("-log2_sb_size") + 1]) if "-log2_sb_size" in flags else 128


def super_blocks(w, h, n, sb=128):
    return ((w + sb - 1) // sb) * ((h + sb - 1) // sb) * n


def launch_key(case):
    """(sample bytes, bit depth) of a case's frames: one device launch per key"""
    flags, bd = case[1], case[6]
    return (2 if bd > 8 or "-frame_bitdepth" in flags else 1), bd


LAUNCHES = [(1, 8), (2, 8), (2, 10), (2, 12)]
LAUNCH_IDS = ["8", "8_in_16bit", "10", "12"]   # by bit depth; 8_in_16bit: -frame_bitdepth 16 with 8-bit input


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# CPU: tb_rdo.h over the oracle against the reference's process_block, super block by super block
# ---------------------------------------------------------------------------------------------------------------------------------------------------
needs_check = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_rdocheck")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                                 reason="oracle/_ref/Thorenc_rdocheck not built (make -C oracle ref rdocheck)")


def verify(tmp, case, env=()):
    from test_rdo_host import enc
    name, flags, w, h, n, qp, bd, content = case
    extra = write_clip(tmp, case)
    _, _, err = enc("Thorenc_rdocheck", flags, w, h, n, "chk", tmp, extra, dict({"TB_RDO_VERIFY": "1", "TB_RDO_VERBOSE": "1"}, **dict(env)), qp=qp)
    m = re.search(r"verify: (\d+) super blocks compared with the reference's process_block, (\d+) differ", err)
    assert m, err[-1500:]
    assert (int(m.group(1)), int(m.group(2))) == (super_blocks(w, h, n, sb_size(flags)), 0), err[-3000:]


@needs_check
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_every_super_block_matches_reference_process_block(tmp_path, case):
    verify(str(tmp_path), case)


@needs_check
@pytest.mark.parametrize("name", ["cfl_inter_hard", "hdb_q4_hard_10", "hdb_q51_12", "speed1_hard_12", "hdb_pan_neg", "hdb_sb64_rect", "reorder3_nd"])
def test_overlapped_decision_with_the_device_warp_count(tmp_path, name):
    """the device decides with eight warps per CTA; host threads stand in for them (TBR_HOST_WARPS), see tests/test_rdo_host.py"""
    verify(str(tmp_path), BY_NAME[name], {"TBR_HOST_WARPS": "8"})


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: all cases in one launch per sample size
# ---------------------------------------------------------------------------------------------------------------------------------------------------
needs_capture = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_capture")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                                   reason="oracle/_ref (reference objects + capture link) not built")


def alloc_into(keep):
    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    return alloc


@pytest.fixture(scope="module")
def matrix_jobs(tmp_path_factory):
    """every case captured with the reference encoder: {name: (job directory, jobs)}"""
    from test_rdo_jobs import capture
    from thor_b200 import rdo_jobs as RJ

    def one(case):
        name, flags, w, h, n, qp, bd, content = case
        d = str(tmp_path_factory.mktemp(name))
        jobdir = capture(d, flags, w, h, n, bd, qp, CONTENT[content])
        return name, (jobdir, RJ.load_jobs(jobdir))
    tmp_path_factory.getbasetemp()  # created lazily: threads that create it at once get different ones, and mktemp then refuses the name
    with ThreadPoolExecutor(min(8, os.cpu_count() or 1)) as ex:
        return dict(ex.map(one, CASES))


@pytest.fixture(scope="module")
def launches(matrix_jobs):
    """launch((sample bytes, bit depth)) -> (return code, [(case name, device HostFrame)]): the frames of every case with that sample size and bit
    depth in one tb_rdo_encode_frames() call, each launch made once per module"""
    import thor_b200 as tb
    from thor_b200 import rdo_jobs as RJ
    L = tb.lib
    L.tb_rdo_encode_frames.argtypes = [C.c_void_p, C.c_int]
    L.tb_rdo_last_error.restype = C.c_char_p
    done, keep = {}, []

    def launch(key):
        if key not in done:
            hosts = [(c[0], RJ.HostFrame(j, alloc_into(keep))) for c in CASES if launch_key(c) == key for j in matrix_jobs[c[0]][1]]
            assert all((hf.job.hdr.sample_bytes, hf.job.hdr.bitdepth) == key for _, hf in hosts)
            descs = (RJ.RdoFrame * len(hosts))(*[hf.desc for _, hf in hosts])
            rc = L.tb_rdo_encode_frames(descs, len(hosts))
            done[key] = (rc, hosts, L.tb_rdo_last_error() if rc else b"")
        return done[key]
    return launch


@pytest.mark.gpu
@needs_capture
@pytest.mark.parametrize("key", LAUNCHES, ids=LAUNCH_IDS)
def test_matrix_in_one_launch_equals_reference_decisions(launches, key):
    rc, hosts, err = launches(key)
    assert rc == 0, err
    assert len({(hf.job.hdr.width, hf.job.hdr.height, hf.job.hdr.qp, hf.job.hdr.encoder_speed) for _, hf in hosts}) > 1  # parameters differ within the launch
    bad = [(name, hf.job.frame_num, r) for name, hf in hosts for r in [hf.check()] if not all(r.values())]
    assert not bad, "%d of %d frames differ from the reference: %s" % (len(bad), len(hosts), bad[:8])


@pytest.mark.gpu
@needs_capture
@pytest.mark.parametrize("key", LAUNCHES, ids=LAUNCH_IDS)
def test_matrix_leaf_lists_and_coefficients_equal_host_decisions(launches, matrix_jobs, key):
    import multiprocessing
    from concurrent.futures import ProcessPoolExecutor
    from _libs import host_decisions_of_dir
    from thor_b200 import rdo_jobs as RJ
    rc, hosts, err = launches(key)
    assert rc == 0, err
    names = [c[0] for c in CASES if launch_key(c) == key]
    # the host decisions of each case in a process of its own (the CPU side takes about a second per frame)
    with ProcessPoolExecutor(min(8, os.cpu_count() or 1), mp_context=multiprocessing.get_context("spawn")) as ex:
        want = dict(zip(names, ex.map(host_decisions_of_dir, [matrix_jobs[n][0] for n in names])))
    bad = []
    for name in names:
        got = [hf for n, hf in hosts if n == name]
        assert len(got) == len(want[name])
        for g, (check, leaves, count, coeffs) in zip(got, want[name]):
            assert check == {"rec": True, "blk": True, "sb_cost": True}, (name, "frame", g.job.frame_num, "host decisions differ from the reference's")
            d = RJ.leaf_differences(g.leaves, g.leaf_count, g.coeffs, leaves, count, coeffs)
            if d:
                bad.append((name, g.job.frame_num, d))
    assert not bad, "%d frames code differently from the host decisions; first: %s" % (len(bad), bad[:3])
