#!/usr/bin/env python
"""Generates the committed RD-loop jobs (SURVEY §8f.1) of tests/golden: every frame's RD-loop inputs of a small real encode WITH the decisions of the
reference's own process_block(), written by the reference encoder + observing shim (oracle/_ref/Thorenc_capture, TB_RDO_DUMP).  The frame_NNN.job
files are concatenated (8-byte length prefix each) and xz-compressed.  CDEF is off in every case: tiny frames + CDEF corrupt the reference's header,
SURVEY §8c.3.  The cases (CASES):
  hdb_128x136          rdo_jobs_hdb_128x136.xz: 9 frames of 128x136 HDB at qp 32 on tests/test_dropin_link.py:synth_yuv (I, P, seven
                       hierarchical B frames with interpolated reference and bipred)
  hdb_hard_q4_10bit    rdo_jobs_hdb_hard_q4_10bit.xz: 5 frames of 128x136 10-bit HDB at qp 4 on tests/test_rdo_matrix.py:hard_yuv (large
                       coefficients, saturated samples, local motion)
  hdb_q51_12bit        rdo_jobs_hdb_q51_12bit.xz: 3 frames of 128x136 12-bit HDB at qp 51 on synth_yuv (an unsplit 128x128 block in each, one
                       of them an intra block whose transform's box sum wraps in int16)
Run in the development container (needs /root/reference compiled into oracle/_ref):  python tests/golden/make_golden_rdo.py [case ...]"""
import lzma
import os
import struct
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from test_dropin_link import HDB, REF, synth_yuv  # noqa: E402

CASES = {
    # name: (flags, width, height, frames, qp, bitdepth, clip writer name, output file)
    "hdb_128x136": (HDB + ["-cdef", "0"], 128, 136, 9, 32, 8, "synth", "rdo_jobs_hdb_128x136.xz"),
    "hdb_hard_q4_10bit": (HDB + ["-cdef", "0"], 128, 136, 5, 4, 10, "hard", "rdo_jobs_hdb_hard_q4_10bit.xz"),
    "hdb_q51_12bit": (HDB + ["-cdef", "0"], 128, 136, 3, 51, 12, "synth", "rdo_jobs_hdb_q51_12bit.xz"),
}


def path(case):
    return os.path.join(HERE, CASES[case][7])


def capture(tmp, case="hdb_128x136"):
    flags, w, h, n, qp, bd, content, _ = CASES[case]
    if content == "hard":
        from test_rdo_matrix import hard_yuv as make_clip
    else:
        make_clip = synth_yuv
    make_clip(os.path.join(tmp, "in.yuv"), w, h, n, bd)
    extra = ["-bitdepth", str(bd), "-input_bitdepth", str(bd)] if bd != 8 else []
    r = subprocess.run([os.path.join(REF, "Thorenc_capture")] + flags + ["-if", os.path.join(tmp, "in.yuv"), "-of", os.path.join(tmp, "o.bit"), "-width", str(w),
                                                                         "-height", str(h), "-n", str(n), "-qp", str(qp), "-f", "30"] + extra, capture_output=True,
                       text=True, env=dict(os.environ, TB_RDO_DUMP=tmp))
    assert r.returncode == 0, r.stderr[-800:]
    return [open(os.path.join(tmp, f), "rb").read() for f in sorted(os.listdir(tmp)) if f.endswith(".job")]


def pack(jobs):
    return lzma.compress(b"".join(struct.pack("<Q", len(j)) + j for j in jobs), preset=9 | lzma.PRESET_EXTREME)


def unpack(blob, directory):
    raw, o, k = lzma.decompress(blob), 0, 0
    while o < len(raw):
        n = struct.unpack_from("<Q", raw, o)[0]
        open(os.path.join(directory, "frame_%03d.job" % k), "wb").write(raw[o + 8:o + 8 + n])
        o += 8 + n
        k += 1
    return k


if __name__ == "__main__":
    for case in sys.argv[1:] or ["hdb_128x136"]:
        with tempfile.TemporaryDirectory() as tmp:
            jobs = capture(tmp, case)
        blob = pack(jobs)
        open(path(case), "wb").write(blob)
        print("%s: %d jobs, %d bytes raw, %d bytes compressed" % (path(case), len(jobs), sum(len(j) for j in jobs), len(blob)))
