"""SURVEY §8f.1 on the CPU: the RD-loop control flow of thor_b200/csrc/tb_rdo.h (process_block, early skip, mode_decision_rdo,
encode_block, the bit counts of write_block, MV predictors / skip / merge candidates, block contexts) pinned against the compiled
reference.  oracle/_ref/Thorenc_rdocheck = the reference's unmodified objects + thor_b200/csrc/tb_rdo_shim.c (--wrap=process_block_*) +
oracle/librdo_hostcheck.so (tb_rdo.h over the plain-C oracle's primitives; test infrastructure).

  * verify mode (TB_RDO_VERIFY=1): every super block of a real encode is decided by tb_rdo.h AND by the reference's process_block()
    on the same encoder state; bits, reconstruction and deblock_data must be identical;
  * frame mode: every frame goes through tb_rdo_encode_frame() (the C ABI the CUDA library implements) and the .bit file and the
    reconstruction must equal the all-reference encoder's.
The CUDA build of the same header differs only in its backend (tests/test_gpu_rdo.py runs the same comparison on the GPU)."""
import os
import re
import subprocess

import pytest

from test_dropin_link import HDB, LDB, REF, synth_yuv

needs = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_rdocheck")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                           reason="oracle/_ref/Thorenc_rdocheck not built (make -C oracle ref rdocheck)")

CASES = [
    # name, flags, w, h, frames, extra   (9 frames of HDB = I, P and 7 hierarchical B frames with interpolated references and bipred)
    ("hdb_8bit_B", HDB + ["-cdef", "0"], 256, 136, 9, ()),
    ("hdb_8bit_odd", HDB + ["-cdef", "0"], 200, 136, 3, ()),
    ("ldb_8bit", LDB, 320, 200, 5, ()),
    ("hdb_10bit_B", HDB + ["-cdef", "0"], 128, 136, 9, ("-bitdepth", "10", "-input_bitdepth", "10")),
    ("ldb_10bit", LDB, 256, 200, 4, ("-bitdepth", "10", "-input_bitdepth", "10")),
    ("hdb_8bit_fb16", HDB + ["-cdef", "0"], 128, 136, 5, ("-frame_bitdepth", "16")),   # 8-bit content in 16-bit frames (DESIGN.md §5)
]


def enc(exe, flags, w, h, n, tag, tmp, extra, env=None, qp=32):
    """encode tmp/in.yuv (written by the caller) with oracle/_ref/<exe>"""
    bit, rec = os.path.join(tmp, tag + ".bit"), os.path.join(tmp, tag + "_rec.yuv")
    cmd = [os.path.join(REF, exe)] + flags + ["-if", os.path.join(tmp, "in.yuv"), "-of", bit, "-rf", rec, "-width", str(w), "-height", str(h), "-n", str(n), "-qp", str(qp),
                                              "-f", "30"] + list(extra)
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=e)
    assert r.returncode == 0, r.stderr[-2000:]
    return open(bit, "rb").read(), open(rec, "rb").read(), r.stderr


@needs
@pytest.mark.parametrize("name,flags,w,h,n,extra", CASES)
def test_every_super_block_matches_reference_process_block(tmp_path, name, flags, w, h, n, extra):
    tmp = str(tmp_path)
    synth_yuv(os.path.join(tmp, "in.yuv"), w, h, n, 10 if "10bit" in name else 8)
    _, _, err = enc("Thorenc_rdocheck", flags, w, h, n, "chk", tmp, extra, {"TB_RDO_VERIFY": "1", "TB_RDO_VERBOSE": "1"})
    m = re.search(r"verify: (\d+) super blocks compared with the reference's process_block, (\d+) differ", err)
    assert m, err[-1500:]
    nsb = ((w + 127) // 128) * ((h + 127) // 128) * n
    assert int(m.group(1)) == nsb and int(m.group(2)) == 0, err[-3000:]


@needs
@pytest.mark.parametrize("name,flags,w,h,n,extra", CASES[:1] + CASES[2:3] + CASES[5:6])
def test_whole_encode_through_the_c_abi_is_bit_exact(tmp_path, name, flags, w, h, n, extra):
    tmp = str(tmp_path)
    synth_yuv(os.path.join(tmp, "in.yuv"), w, h, n, 10 if "10bit" in name else 8)
    bit_ref, rec_ref, _ = enc("Thorenc", flags, w, h, n, "ref", tmp, extra)
    bit, rec, err = enc("Thorenc_rdocheck", flags, w, h, n, "chk", tmp, extra, {"TB_RDO_STATS": "1"})
    assert "frames decided by tb_rdo_encode_frame: %d," % n in err, err[-500:]
    assert bit == bit_ref, "bitstream differs"
    assert rec == rec_ref, "reconstruction differs"


@needs
@pytest.mark.parametrize("nw", [3, 8])
def test_overlapped_decision_with_simulated_warps(tmp_path, nw):
    """The device runs the control flow SPMD over the warps of a CTA; with more than one warp mode_decision_rdo overlaps the bi-prediction chain, the
    inter candidates and the intra-mode search (shared work counters).  Host threads stand in for the warps (TBR_HOST_WARPS): every super block must
    still equal the reference's process_block, whichever warp evaluated which candidate."""
    name, flags, w, h, n, extra = CASES[0]
    tmp = str(tmp_path)
    synth_yuv(os.path.join(tmp, "in.yuv"), w, h, n, 8)
    _, _, err = enc("Thorenc_rdocheck", flags, w, h, n, "chk", tmp, extra, {"TB_RDO_VERIFY": "1", "TB_RDO_VERBOSE": "1", "TBR_HOST_WARPS": str(nw)})
    m = re.search(r"verify: (\d+) super blocks compared with the reference's process_block, (\d+) differ", err)
    assert m, err[-1500:]
    assert int(m.group(1)) == ((w + 127) // 128) * ((h + 127) // 128) * n and int(m.group(2)) == 0, err[-3000:]
