"""Link-unchanged test (SURVEY.md §8b): the reference's own host objects (mainenc.o, encode_frame.o, encode_block.o,
transform.o, inter_prediction.o, temporal_interp.o, common_frame.o, ... compiled from /root/reference in place by
oracle/Makefile) linked against libthor_b200.so INSTEAD of enc_kernels{,_hbd}.o / common_kernels{,_hbd}.o must produce the
same .bit stream and reconstruction as the all-reference binary, and Thordec built the same way must decode it bit-exactly.
Every kernel call of the run goes through the drop-in symbols, i.e. through CUDA (one staged launch per call)."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
LDB = ("-HQperiod 12 -mqpP 1.2 -dqpI -2 -lambda_coeffI 0.8 -lambda_coeffP 1.2 -intra_rdo 0 -enable_tb_split 0 -enable_pb_split 0 -early_skip_thr 1.0 "
       "-max_num_ref 2 -use_block_contexts 1 -enable_bipred 0 -encoder_speed 2 -enable_cfl_intra 1 -enable_cfl_inter 0 -cdef 0 -clpf 1").split()
HDB = ("-HQperiod 1 -num_reorder_pics 7 -interp_ref 1 -dqpI -2 -dqpB0 3 -dqpB1 1 -dqpB2 0 -mqpP 1.2 -mqpB 1.2 -mqpB0 1.1 -mqpB1 1.2 -mqpB2 1.3 "
       "-lambda_coeffI 0.8 -lambda_coeffP 1.2 -lambda_coeffB 1.2 -lambda_coeffB0 1.2 -lambda_coeffB1 1.2 -lambda_coeffB2 1.2 -intra_rdo 1 -enable_tb_split 1 "
       "-enable_pb_split 1 -early_skip_thr 0.3 -max_num_ref 4 -use_block_contexts 1 -enable_bipred 1 -encoder_speed 0 -enable_cfl_intra 1 -enable_cfl_inter 0").split()


def synth_yuv(path, w, h, n, bitdepth=8, seed=5):
    rng = np.random.default_rng(seed)
    m = 2 * n + 8
    yy, xx = np.mgrid[0:h + m, 0:w + m]
    base = np.clip(rng.integers(0, 48, ((h + m) // 8 + 1, (w + m) // 8 + 1)).repeat(8, 0).repeat(8, 1)[:h + m, :w + m] + 60 * np.sin(xx / 17.0) + 50 * np.cos(yy / 11.0) + 100, 0, 255)
    with open(path, "wb") as f:
        for k in range(n):
            y = np.clip(base[k:k + h, 2 * k:2 * k + w] + rng.normal(0, 2, (h, w)), 0, 255).astype(np.uint8)
            u = np.clip(128 + 20 * np.sin(xx[:h // 2, :w // 2] / 9.0 + k), 0, 255).astype(np.uint8)
            v = np.clip(128 + 20 * np.cos(yy[:h // 2, :w // 2] / 7.0), 0, 255).astype(np.uint8)
            for p in (y, u, v):
                if bitdepth == 8:
                    f.write(p.tobytes())
                else:
                    f.write(((p.astype(np.uint16) << (bitdepth - 8)) | rng.integers(0, 1 << (bitdepth - 8), p.shape).astype(np.uint16)).astype("<u2").tobytes())


def run(exe, flags, w, h, n, tag, tmp, extra=()):
    bit, rec = os.path.join(tmp, tag + ".bit"), os.path.join(tmp, tag + "_rec.yuv")
    cmd = [os.path.join(REF, exe)] + flags + ["-if", os.path.join(tmp, "in.yuv"), "-of", bit, "-rf", rec, "-width", str(w), "-height", str(h), "-n", str(n),
                                              "-qp", "32", "-f", "30"] + list(extra)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stderr[-2000:]
    return open(bit, "rb").read(), open(rec, "rb").read(), bit


needs = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, "Thorenc_b200")) and os.path.exists(os.path.join(REF, "Thorenc"))),
                           reason="oracle/_ref (reference objects + drop-in link) not built")


@pytest.mark.gpu
@needs
@pytest.mark.parametrize("name,flags,w,h,n,extra", [
    ("ldb_8bit", LDB, 128, 64, 3, ()),
    ("hdb_8bit", HDB + ["-cdef", "0"], 64, 64, 2, ()),          # tiny frames + CDEF corrupt the reference's header (SURVEY.md §8c.3)
    ("ldb_10bit", LDB, 64, 64, 2, ("-bitdepth", "10", "-input_bitdepth", "10")),
    # 8-bit content in 16-bit frames: the encoder's 16-bit kernels predict 0 at one-axis fractions (DESIGN.md §5), the decoder works in 8-bit samples
    ("ldb_8bit_fb16", LDB, 128, 64, 3, ("-frame_bitdepth", "16")),
])
def test_thorenc_thordec_link_unchanged_bit_exact(tmp_path, name, flags, w, h, n, extra):
    tmp = str(tmp_path)
    synth_yuv(os.path.join(tmp, "in.yuv"), w, h, n, 10 if "10bit" in name else 8)
    bit_ref, rec_ref, ref_bitfile = run("Thorenc", flags, w, h, n, "ref", tmp, extra)
    bit_gpu, rec_gpu, bitfile = run("Thorenc_b200", flags, w, h, n, "gpu", tmp, extra)
    assert bit_gpu == bit_ref, "bitstream differs"
    assert rec_gpu == rec_ref, "reconstruction differs"
    out = os.path.join(tmp, "dec.yuv")
    r = subprocess.run(["timeout", "600", os.path.join(REF, "Thordec_b200"), bitfile, out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    if "-frame_bitdepth" in extra:  # the reference's decoder does not reconstruct such an encoder's frames: the drop-in decoder must equal it
        ref_out = os.path.join(tmp, "dec_ref.yuv")
        r = subprocess.run(["timeout", "600", os.path.join(REF, "Thordec"), ref_bitfile, ref_out], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        assert open(out, "rb").read() == open(ref_out, "rb").read(), "decoder output differs from the reference decoder's"
    else:
        assert open(out, "rb").read() == rec_ref, "decoder output differs from the encoder's reconstruction"
