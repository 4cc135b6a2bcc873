"""SURVEY §8f.4: thor_b200/yuvio.py against the reference's own read_yuv_frame / write_yuv_frame (common/common_frame.c:478-654; their results
stored in tests/golden/yuvio_ref.npz, and checked against oracle/_ref/libthorref.so where it is built) and its y4m header rules
(enc/strings.c:376-449).  CPU only."""
import ctypes as C
import importlib.util
import io
import os

import numpy as np
import pytest

from _refstructs import Frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("yuvio", os.path.join(ROOT, "thor_b200", "yuvio.py"))
Y = importlib.util.module_from_spec(spec)
spec.loader.exec_module(Y)
REFSO = os.path.join(ROOT, "oracle", "_ref", "libthorref.so")


def libc_file(path, mode):
    libc = C.CDLL(None)
    libc.fopen.restype = C.c_void_p
    libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
    libc.fclose.argtypes = [C.c_void_p]
    fp = libc.fopen(path.encode(), mode.encode())
    assert fp
    return libc, fp


CASES = [(8, 8), (8, 10), (10, 10), (10, 8), (12, 10)]
GOLDEN = os.path.join(ROOT, "tests", "golden", "yuvio_ref.npz")  # the reference's results on CASES: python tests/test_yuvio.py writes it


def case_input(input_bd, bd):
    rng = np.random.default_rng(3 + input_bd * 16 + bd)
    w, h = 64, 48
    fdt = np.dtype("<u2") if input_bd > 8 else np.dtype("u1")
    return w, h, [rng.integers(0, 1 << input_bd, s).astype(fdt) for s in ((h, w), (h // 2, w // 2), (h // 2, w // 2))]


def reference_io(tmp_path, input_bd, bd):
    """the compiled reference's read_yuv_frame on the case's file, and write_yuv_frame of the frame it read (None where the write is not comparable:
    with a file depth > 8 that differs from the codec's the reference converts into `uint8_t *buf16` (common/common_frame.c:559, 578-581), i.e. stores
    the low BYTE of every sample and writes uninitialised memory behind them)"""
    w, h, src = case_input(input_bd, bd)
    hbd = int(max(input_bd, bd) > 8)
    ref = C.CDLL(REFSO)
    path = os.path.join(str(tmp_path), "in.yuv")
    with open(path, "wb") as f:
        for p in src:
            f.write(p.tobytes())
    fr = Frame(w, h, bd, hbd)
    fr.s.input_bitdepth = input_bd
    libc, fp = libc_file(path, "rb")
    rd = ref.read_yuv_frame_hbd if hbd else ref.read_yuv_frame_lbd
    rd.argtypes = [C.c_void_p, C.c_void_p]
    rd(C.byref(fr.s), fp)
    libc.fclose(fp)
    planes = [fr.plane(p).copy() for p in range(3)]
    if input_bd > 8 and input_bd != bd:
        return planes, None
    out_ref = os.path.join(str(tmp_path), "out_ref.yuv")
    libc, fp = libc_file(out_ref, "wb")
    wr = ref.write_yuv_frame_hbd if hbd else ref.write_yuv_frame_lbd
    wr.argtypes = [C.c_void_p, C.c_void_p]
    wr(C.byref(fr.s), fp)
    libc.fclose(fp)
    return planes, open(out_ref, "rb").read()


def golden_io(input_bd, bd):
    g = np.load(GOLDEN)
    k = "%d_%d" % (input_bd, bd)
    written = g["write_" + k].tobytes() if "write_" + k in g else None
    return [g["read_%s_%d" % (k, p)] for p in range(3)], written


@pytest.mark.parametrize("input_bd,bd", CASES)
def test_read_and_write_match_reference(tmp_path, input_bd, bd):
    w, h, src = case_input(input_bd, bd)
    hbd = int(max(input_bd, bd) > 8)
    want_planes, want_written = golden_io(input_bd, bd)
    if os.path.exists(REFSO):  # the stored results are what the reference computes today
        live_planes, live_written = reference_io(tmp_path, input_bd, bd)
        assert all(np.array_equal(a, b) for a, b in zip(live_planes, want_planes)) and live_written == want_written, "tests/golden/yuvio_ref.npz is stale"
    path = str(tmp_path / "in.yuv")
    with open(path, "wb") as f:
        for p in src:
            f.write(p.tobytes())
    with open(path, "rb") as f:
        got = Y.read_yuv_frame(f, w, h, input_bd, bd)
    for p in range(3):
        assert got[p].dtype == (np.uint16 if hbd else np.uint8)
        assert np.array_equal(got[p], want_planes[p]), "read: plane %d differs" % p
    if want_written is None:
        return
    buf = io.BytesIO()
    Y.write_yuv_frame(buf, got, input_bd, bd)
    assert buf.getvalue() == want_written, "write: bytes differ"


def test_y4m_header_and_reader(tmp_path):
    w, h, n = 32, 16, 3
    rng = np.random.default_rng(9)
    frames = [[rng.integers(0, 1024, s).astype("<u2") for s in ((h, w), (h // 2, w // 2), (h // 2, w // 2))] for _ in range(n)]
    path = str(tmp_path / "clip.y4m")
    with open(path, "wb") as f:
        f.write(b"YUV4MPEG2 W32 H16 F30000:1001 Ip A1:1 C420p10 XYSCSS=420P10\n")
        for fr in frames:
            f.write(b"FRAME\n")
            for p in fr:
                f.write(p.tobytes())
    hdr = Y.parse_y4m_header(open(path, "rb").read(256))
    assert (hdr.width, hdr.height, hdr.subsample, hdr.input_bitdepth, hdr.frame_headerlen) == (32, 16, 420, 10, 6)
    assert abs(hdr.frame_rate - 30000 / 1001) < 1e-9
    r = Y.YuvReader(path, skip=1)
    pinned_like = [np.zeros(p.shape, np.uint16) for p in frames[0]]     # caller-owned staging
    got = r.read(out=pinned_like)
    assert all(np.array_equal(got[p], frames[1][p]) and got[p] is pinned_like[p] for p in range(3))
    got = r.read()
    assert all(np.array_equal(got[p], frames[2][p]) for p in range(3))
    with pytest.raises(EOFError):
        r.read()
    r.close()
    assert Y.parse_y4m_header(b"\x00" * 64) is None
    with pytest.raises(ValueError):
        Y.parse_y4m_header(b"YUV4MPEG2 W32 H16 It C420\nFRAME\n")


if __name__ == "__main__":
    import tempfile
    store = {}
    with tempfile.TemporaryDirectory() as tmp:
        for ibd, bd in CASES:
            planes, written = reference_io(tmp, ibd, bd)
            for p in range(3):
                store["read_%d_%d_%d" % (ibd, bd, p)] = planes[p]
            if written is not None:
                store["write_%d_%d" % (ibd, bd)] = np.frombuffer(written, np.uint8)
    np.savez_compressed(GOLDEN, **store)
