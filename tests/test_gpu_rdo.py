"""SURVEY §8f.1 on the GPU: oracle/_ref/Thorenc_b200_rdo = the reference's unmodified HOST objects + thor_b200/csrc/tb_rdo_shim.c
(--wrap=process_block_*) + libthor_b200.so.  Every frame's RD loop runs in rdo_batch_kernel (tb_rdo_encode_frame), the in-loop filters and
the temporal interpolation run through the drop-in CUDA symbols, and the host only drives the sequence and writes bits.  The .bit file and
the reconstruction must equal the all-reference encoder's — with B frames, interpolated references, bipred and (one case) CDEF on."""
import os
import subprocess

import pytest

from test_dropin_link import HDB, LDB, REF, synth_yuv
from test_rdo_matrix import hard_yuv

needs = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_b200_rdo")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                           reason="oracle/_ref (reference objects + drop-in links) not built")


def enc(exe, flags, w, h, n, tag, tmp, extra, env=None, qp=32):
    """encode tmp/in.yuv (written by the caller) with oracle/_ref/<exe>"""
    bit, rec = os.path.join(tmp, tag + ".bit"), os.path.join(tmp, tag + "_rec.yuv")
    cmd = [os.path.join(REF, exe)] + flags + ["-if", os.path.join(tmp, "in.yuv"), "-of", bit, "-rf", rec, "-width", str(w), "-height", str(h), "-n", str(n), "-qp", str(qp),
                                              "-f", "30"] + list(extra)
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=e)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-2000:])
    return open(bit, "rb").read(), open(rec, "rb").read(), r.stderr, bit


# qp and clip of the cases that do not encode synth_yuv at qp 32: low qp on 10-bit hard content (large coefficients, saturation), nearly everything
# skipped (qp 51), cfl_inter, encoder speed 1 on a frame narrower than two super blocks, 12 bits at qp 51 (a 128x128 intra block whose transform's
# box sum wraps in int16)
CLIPS = {"hdb_10bit_q4_hard": (4, hard_yuv), "hdb_8bit_q51": (51, synth_yuv), "hdb_8bit_cfl_inter_hard": (22, hard_yuv), "hdb_8bit_speed1_rect_hard": (8, hard_yuv),
         "hdb_12bit_q51": (51, synth_yuv)}


@pytest.mark.gpu
@needs
@pytest.mark.parametrize("name,flags,w,h,n,extra,decode", [
    ("hdb_8bit_B", HDB + ["-cdef", "0"], 256, 136, 9, (), True),      # I, P, 7 hierarchical B frames: interp_ref, bipred, early skip, tb/pb split
    ("ldb_8bit", LDB, 320, 200, 5, (), True),                         # speed 2: top-down 16x16, SAD-based intra, best_ref
    ("hdb_10bit_B", HDB + ["-cdef", "0"], 128, 136, 9, ("-bitdepth", "10", "-input_bitdepth", "10"), True),
    ("hdb_8bit_rect", HDB + ["-cdef", "0"], 200, 136, 3, (), True),   # widths that are not a multiple of the super block: rectangular skips
    ("hdb_8bit_cdef", HDB, 256, 192, 9, (), False),                   # CDEF on (tiny-frame streams are undecodable in the reference, SURVEY §8c.3: encoder outputs only)
    # cases of tests/test_rdo_matrix.py, with their qp and clip in CLIPS
    ("hdb_10bit_q4_hard", HDB + ["-cdef", "0"], 128, 136, 5, ("-bitdepth", "10", "-input_bitdepth", "10"), True),
    ("hdb_8bit_q51", HDB + ["-cdef", "0"], 128, 136, 9, (), True),
    ("hdb_8bit_cfl_inter_hard", HDB + ["-cdef", "0", "-enable_cfl_inter", "1"], 128, 136, 5, (), True),
    ("hdb_8bit_speed1_rect_hard", HDB + ["-cdef", "0", "-encoder_speed", "1"], 200, 72, 5, (), True),
    ("hdb_12bit_q51", HDB + ["-cdef", "0"], 128, 136, 5, ("-bitdepth", "12", "-input_bitdepth", "12"), True),
    ("hdb_8bit_sb64_rect", HDB + ["-cdef", "0", "-log2_sb_size", "6"], 200, 136, 5, (), True),   # 64x64 super blocks, a partial last column
    ("hdb_8bit_no_interp", HDB + ["-cdef", "0", "-interp_ref", "0"], 128, 136, 9, (), True),     # B frames without an interpolated reference
    # 8-bit content in 16-bit frames, where the reference's encoder predicts 0 at one-axis fractions (DESIGN.md §5).  Its decoder filters
    # these normally, so it does not reconstruct the encoder's frames: encoder outputs only
    ("hdb_8bit_fb16", HDB + ["-cdef", "0"], 128, 136, 5, ("-frame_bitdepth", "16"), False),
])
def test_device_rd_loop_encode_is_bit_exact(tmp_path, name, flags, w, h, n, extra, decode):
    tmp = str(tmp_path)
    qp, make_clip = CLIPS.get(name, (32, synth_yuv))
    make_clip(os.path.join(tmp, "in.yuv"), w, h, n, 12 if "12bit" in name else 10 if "10bit" in name else 8)
    bit_ref, rec_ref, _, _ = enc("Thorenc", flags, w, h, n, "ref", tmp, extra, qp=qp)
    bit, rec, err, bitfile = enc("Thorenc_b200_rdo", flags, w, h, n, "gpu", tmp, extra, {"TB_RDO_STATS": "1"}, qp=qp)
    assert "frames decided by tb_rdo_encode_frame: %d," % n in err, err[-800:]   # every frame went through the device RD loop (no host-loop frames)
    assert bit == bit_ref, "bitstream differs"
    assert rec == rec_ref, "reconstruction differs"
    if decode:
        out = os.path.join(tmp, "dec.yuv")
        r = subprocess.run(["timeout", "600", os.path.join(REF, "Thordec_b200"), bitfile, out], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        assert open(out, "rb").read() == rec_ref, "decoder output differs from the encoder's reconstruction"
