"""Pins the plain-C oracle (oracle/thor_oracle.c) against the compiled, unmodified reference (oracle/_ref,
built from /root/reference by oracle/Makefile).  CPU only.  Skipped when oracle/_ref is absent."""
import ctypes as C
import numpy as np
import pytest
from _libs import oracle, ref, ref_enc, aligned, P, sdt, sfx, rand_plane, full_scale_planes, edge_search, edge_reach
from _refstructs import Frame, random_blkinfo, CdefStrengths, Mv

pytestmark = pytest.mark.skipif(ref() is None, reason="oracle/_ref not built")
O = oracle()
R = ref()
BD = [(0, 8), (1, 10), (1, 12)]
# edge trials per sign whose result lies on a clip_mv limit / is predicted through an active split_mv clamp, at least (the seeded trials reach
# 37..49 / 141..158 of 160 per sign in test_motion_estimate)
ME_EDGE_REACH = np.array([25, 100])
ME_BI_EDGE_REACH = np.array([16, 30])  # of 48 per sign: 24..27 / 43..44


def test_tables():
    g4 = np.ctypeslib.as_array((C.c_int16 * 1024).in_dll(R, "g4mat_hevc")).reshape(32, 32)
    m32 = np.ctypeslib.as_array(C.cast(O.orc_dct_matrix(5), C.POINTER(C.c_int16)), (1024,)).reshape(32, 32)
    assert (g4 == m32).all()
    for l, n in ((2, 4), (3, 8), (4, 16)):
        m = np.ctypeslib.as_array(C.cast(O.orc_dct_matrix(l), C.POINTER(C.c_int16)), (n * n,)).reshape(n, n)
        assert (m == g4[::32 // n, :n]).all()
    for q, name in ((4, "zigzag16"), (8, "zigzag64"), (16, "zigzag256")):
        z = np.ctypeslib.as_array((C.c_int * (q * q)).in_dll(R, name))
        mine = np.ctypeslib.as_array(C.cast(O.orc_zigzag(q), C.POINTER(C.c_int)), (q * q,))
        assert (z == mine).all()
    cq = np.ctypeslib.as_array((C.c_int * 52).in_dll(R, "chroma_qp"))
    assert [O.orc_chroma_qp(i) for i in range(52)] == list(cq)


@pytest.mark.parametrize("hbd,bd", BD)
def test_sad_family(hbd, bd):
    rng = np.random.default_rng(1)
    E = ref_enc(hbd)
    s = sfx(hbd)
    for smooth in (False, True):
        refp = rand_plane(rng, 200, 256, bd, hbd, smooth)
        for (w, h) in [(8, 8), (8, 4), (8, 16), (16, 16), (16, 8), (32, 32), (32, 16), (64, 64), (64, 32), (128, 128), (128, 64), (16, 32), (4, 4), (4, 8)]:
            size = max(w, h)
            org = aligned((size, size), sdt(hbd))
            oy, ox = int(rng.integers(8, 60)), int(rng.integers(8, 100))
            org[...] = refp[oy:oy + size, ox:ox + size] if smooth else rng.integers(0, 1 << bd, (size, size))
            for _ in range(3):
                y, x = int(rng.integers(8, 60)), int(rng.integers(8, 100))
                b = P(refp, y * 256 + x)
                want = getattr(O, "orc_sad_" + s)(P(org), b, size, 256, w, h)
                assert getattr(E, "ref_sad_calc_" + s)(P(org), b, size, 256, w, h) == want
                if w > 4:
                    assert getattr(R, "sad_calc_simd_" + s)(P(org), b, size, 256, w, h) == want
                if w in (4, 8, 16) and h % 4 == 0:  # wider blocks hit a pointer-stepping quirk (common_kernels.c:103-113); only <=16 is used
                    if True:
                        assert getattr(R, "sad_calc_simd_unaligned_" + s)(P(org), b, size, 256, w, h) == want
                if w == h:
                    want = getattr(O, "orc_ssd_" + s)(P(org), P(refp, y * 256 + (x & ~31)), size, 256, w, h)
                    assert getattr(E, "ref_ssd_calc_" + s)(P(org), P(refp, y * 256 + (x & ~31)), size, 256, w, h) == want
                    if w > 4:
                        assert getattr(R, "ssd_calc_simd_" + s)(P(org), P(refp, y * 256 + (x & ~31)), size, 256, w) == want
                xo, xr, xe = C.c_int(9), C.c_int(9), C.c_int(9)
                want = getattr(O, "orc_widesad_" + s)(P(org), b, size, 256, w, h, C.byref(xo))
                assert getattr(E, "ref_widesad_calc_" + s)(P(org), b, size, 256, w, h, C.byref(xe)) == want and xe.value == xo.value
                if w == 16 and h == 16:
                    assert getattr(R, "widesad_calc_simd_" + s)(P(org), b, size, 256, w, h, C.byref(xr)) == want and xr.value == xo.value


@pytest.mark.parametrize("hbd,bd", BD)
def test_fast_subpel_sad(hbd, bd):
    rng = np.random.default_rng(2)
    E = ref_enc(hbd)
    s = sfx(hbd)
    for smooth in (False, True):
        refp = rand_plane(rng, 200, 256, bd, hbd, smooth)
        for (w, h) in [(8, 8), (16, 16), (16, 8), (8, 16), (32, 32), (64, 64), (32, 16), (4, 4)]:
            size = max(w, h)
            org = aligned((size, size), sdt(hbd))
            oy, ox = int(rng.integers(8, 60)), int(rng.integers(8, 100))
            org[...] = refp[oy:oy + size, ox:ox + size]
            for _ in range(3):
                y, x = oy + int(rng.integers(-2, 3)), ox + int(rng.integers(-2, 3))
                b = P(refp, y * 256 + x)
                xs = [C.c_int(0) for _ in range(6)]
                want = getattr(O, "orc_sad_fasthalf_" + s)(P(org), b, size, 256, w, h, C.byref(xs[0]), C.byref(xs[1]))
                got = getattr(E, "ref_sad_calc_fasthalf_" + s)(P(org), b, size, 256, w, h, C.byref(xs[2]), C.byref(xs[3]))
                assert (got, xs[2].value, xs[3].value) == (want, xs[0].value, xs[1].value)
                if w > 4:
                    got = getattr(R, "sad_calc_fasthalf_simd_" + s)(P(org), b, size, 256, w, h, C.byref(xs[4]), C.byref(xs[5]), None)
                    assert (got, xs[4].value, xs[5].value) == (want, xs[0].value, xs[1].value)
                for (fx, fy) in [(0, 0), (2, 0), (0, 2), (-2, 2), (2, 2), (-2, 0), (0, -2)]:
                    xs = [C.c_int(fx if i % 2 == 0 else fy) for i in range(6)]
                    want = getattr(O, "orc_sad_fastquarter_" + s)(P(org), b, size, 256, w, h, C.byref(xs[0]), C.byref(xs[1]))
                    got = getattr(E, "ref_sad_calc_fastquarter_" + s)(P(org), b, size, 256, w, h, C.byref(xs[2]), C.byref(xs[3]))
                    assert (got, xs[2].value, xs[3].value) == (want, xs[0].value, xs[1].value)
                    if w > 4:
                        got = getattr(R, "sad_calc_fastquarter_simd_" + s)(P(org), b, size, 256, w, h, C.byref(xs[4]), C.byref(xs[5]))
                        assert (got, xs[4].value, xs[5].value) == (want, xs[0].value, xs[1].value)


@pytest.mark.parametrize("hbd,bd", BD)
def test_interp(hbd, bd):
    rng = np.random.default_rng(3)
    s = sfx(hbd)
    refp = rand_plane(rng, 200, 256, bd, hbd)
    for (w, h) in [(4, 4), (8, 8), (4, 8), (8, 4), (16, 16), (32, 32), (16, 8), (64, 64), (128, 128)]:
        for bip in (0, 1, 2):
            for xo in range(4):
                for yo in range(4):
                    if xo == 0 and yo == 0:
                        continue
                    y, x = int(rng.integers(8, 40)), int(rng.integers(8, 60))
                    a = aligned((h, w), sdt(hbd)); b = aligned((h, w), sdt(hbd))
                    getattr(O, "orc_interp_luma_" + s)(w, h, xo, yo, P(a), w, P(refp, y * 256 + x), 256, bip, bd)
                    getattr(R, "get_inter_prediction_luma_simd_" + s)(w, h, xo, yo, P(b), w, P(refp, y * 256 + x), 256, bip, bd)
                    assert (a == b).all(), (w, h, bip, xo, yo)
    for (w, h) in [(4, 4), (8, 8), (4, 2), (2, 4), (16, 16), (32, 32), (64, 64), (8, 4)]:
        for xo in range(8):
            for yo in range(8):
                if xo == 0 and yo == 0:
                    continue
                y, x = int(rng.integers(8, 40)), int(rng.integers(8, 60))
                a = aligned((h, w), sdt(hbd)); b = aligned((h, w), sdt(hbd))
                getattr(O, "orc_interp_chroma_" + s)(w, h, xo, yo, P(a), w, P(refp, y * 256 + x), 256, bd)
                if w > 2:
                    getattr(R, "get_inter_prediction_chroma_simd_" + s)(w, h, xo, yo, P(b), w, P(refp, y * 256 + x), 256, bd)
                    assert (a == b).all(), (w, h, xo, yo)
    # full entry incl. MV clamp, against the reference's non-static get_inter_prediction_luma
    f = Frame(128, 96, bd, hbd)
    f.randomize(rng, smooth=False)
    getattr(R, "pad_yuv_frame_" + s)(C.byref(f.s))
    for _ in range(200):
        size = int(rng.choice([8, 16, 32]))
        xpos, ypos = int(rng.integers(0, 128 // size)) * size, int(rng.integers(0, 96 // size)) * size
        mv = Mv(int(rng.integers(-700, 700)), int(rng.integers(-700, 700)))
        sign = int(rng.integers(0, 2))
        getattr(R, "clip_mv_" + s)(C.byref(mv), ypos, xpos, 128, 96, size, size, sign)
        mo = (C.c_int16 * 2)(mv.x, mv.y)
        a = aligned((size, size), sdt(hbd)); b = aligned((size, size), sdt(hbd))
        off = f.origin(0) + ypos * f.sy + xpos
        getattr(R, "get_inter_prediction_luma_" + s)(P(b), P(f.Y, off), size, size, f.sy, size, C.byref(mv), sign, 1, 128, 96, xpos, ypos, bd)
        getattr(O, "orc_get_inter_prediction_luma_" + s)(P(a), P(f.Y, off), size, size, f.sy, size, mo, sign, 1, 128, 96, xpos, ypos, bd)
        assert (a == b).all()


def test_clip_mv_and_bits():
    rng = np.random.default_rng(4)
    E = ref_enc(0)
    for _ in range(3000):
        mv = Mv(int(rng.integers(-9000, 9000)), int(rng.integers(-6000, 6000)))
        mo = (C.c_int16 * 2)(mv.x, mv.y)
        args = (int(rng.integers(0, 1080)), int(rng.integers(0, 1920)), 1920, 1080, int(rng.choice([8, 16, 64])), int(rng.choice([8, 16, 64])), int(rng.integers(0, 2)))
        R.clip_mv_lbd(C.byref(mv), *args)
        O.orc_clip_mv(mo, *args)
        assert (mv.x, mv.y) == (mo[0], mo[1])
        dy, dx = int(rng.integers(-300, 300)), int(rng.integers(-300, 300))
        assert E.ref_quote_mv_bits_lbd(dy, dx) == O.orc_quote_mv_bits(dy, dx)


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_transform_chain(bd):
    rng = np.random.default_rng(5)
    E = ref_enc(0)
    lim = (1 << bd) - 1
    for size in (4, 8, 16, 32, 64, 128):
        for fast in (0, 1):
            for amp in (lim, 20, 3):
                blk = aligned((size, size), np.int16)
                blk[...] = rng.integers(-amp, amp + 1, (size, size))
                c0 = aligned((size, size), np.int16, fill=0); c1 = aligned((size, size), np.int16, fill=0)
                O.orc_transform(P(blk), P(c0), size, fast, bd)
                R.transform_simd(P(blk), P(c1), size, fast, bd)
                q = min(size, 16)
                assert (c0[:q, :q] == c1[:q, :q]).all(), (size, fast, amp)
                for qp in (12, 22, 32, 37, 44, 51):
                    for typ in (0, 1, 2, 3):
                        q0 = aligned((q * q,), np.int16, fill=0); q1 = aligned((q * q,), np.int16, fill=0)
                        cb0 = O.orc_quantize(P(c0), P(q0), qp, size, typ, None)
                        cb1 = E.ref_quantize_lbd(P(c0), P(q1), qp, size, typ, None)
                        assert cb0 == cb1 and (q0 == q1).all()
                    r0 = aligned((size, size), np.int16, fill=0); r1 = aligned((size, size), np.int16, fill=0)
                    O.orc_dequantize(P(q0), P(r0), qp, size, None)
                    R.dequantize_lbd(P(q1), P(r1), qp, size, None)
                    assert (r0 == r1).all()
                    assert O.orc_check_nz_area(P(r0), size) == R.check_nz_area(P(r1), size) if size <= 32 else True
                    b0 = aligned((size, size), np.int16, fill=0); b1 = aligned((size, size), np.int16, fill=0)
                    O.orc_inverse_transform(P(r0), P(b0), size, bd)
                    R.inverse_transform(P(r1), P(b1), size, bd)
                    assert (b0 == b1).all(), (size, qp)
    # sparse coefficient patterns exercise the reference's check_nz_area shortcuts
    for size in (8, 16, 32):
        for pat in range(40):
            r0 = aligned((size, size), np.int16, fill=0)
            k = min(size, [1, 4, 8, 16][pat % 4])
            r0[:k, :k] = rng.integers(-300, 300, (k, k)) * (rng.random((k, k)) < 0.4)
            b0 = aligned((size, size), np.int16); b1 = aligned((size, size), np.int16)
            O.orc_inverse_transform(P(r0), P(b0), size, bd)
            R.inverse_transform_simd(P(r0), P(b1), size, bd)
            assert O.orc_check_nz_area(P(r0), size) == R.check_nz_area(P(r0), size)
            assert (b0 == b1).all()


def box_sum_blocks(rng, size, bd):
    """64x64 and 128x128 residual blocks whose box sums cross +-16384 by small and large amounts at 12 bits: constant blocks at +-(2^bd-1) and
    at +-1025 / -1026 (16 samples sum to 16400 / -16416), checkerboards of 8x8 cells at +-(2^bd-1) and +-2048, sample checkerboards of the same
    amplitudes, cells of random sign near full scale, and uniform noise at full scale"""
    lim = (1 << bd) - 1
    yy, xx = np.mgrid[0:size, 0:size]
    cell = np.where((yy // 8 + xx // 8) % 2, 1, -1)
    dot = np.where((yy + xx) % 2, 1, -1)
    signs = np.kron(rng.choice([-1, 1], (size // 8, size // 8)), np.ones((8, 8), int))
    pats = {"+max": np.full((size, size), lim), "-max": np.full((size, size), -lim), "+1025": np.full((size, size), min(1025, lim)),
            "-1026": np.full((size, size), -min(1026, lim)),
            "cells max": cell * lim, "cells 2048": cell * min(2048, lim), "dots max": dot * lim, "dots 2048": dot * min(2048, lim),
            "cells near max": signs * rng.integers(lim - 200, lim + 1, (size, size)), "noise": rng.integers(-lim, lim + 1, (size, size))}
    for name, v in pats.items():
        blk = aligned((size, size), np.int16)
        blk[...] = v
        yield name, blk


@pytest.mark.parametrize("bd", [10, 12])
@pytest.mark.parametrize("size", [64, 128])
def test_transform_box_sum_against_transform_simd(bd, size):
    """transform_simd's box sum (common/common_kernels.c:1519-1551): 64x64 and 128x128 without fast wrap in int16, with fast they saturate.
    The wrapping sums leave [-16384, 16383] only for 128x128 at 12 bits (16 x 4095 = 65520).  The coefficients are then quantised, dequantised
    and inverse transformed at every qp and coefficient type; 10 bits is the control where no wrapping sum leaves the range"""
    rng = np.random.default_rng(24)
    E = ref_enc(0)
    q = 16
    for fast in (0, 1):
        scale, crossed = size // (32 >> fast), False
        for name, blk in box_sum_blocks(rng, size, bd):
            box = blk.astype(np.int64).reshape(size // scale, scale, size // scale, scale).sum(axis=(1, 3))
            crossed |= bool(((box < -16384) | (box > 16383)).any())
            c0 = aligned((size, size), np.int16, fill=0); c1 = aligned((size, size), np.int16, fill=0)
            O.orc_transform(P(blk), P(c0), size, fast, bd)
            R.transform_simd(P(blk), P(c1), size, fast, bd)
            assert (c0[:q, :q] == c1[:q, :q]).all(), (size, fast, name)
            for qp in range(52):
                for typ in range(4):
                    q0 = aligned((q * q,), np.int16, fill=0); q1 = aligned((q * q,), np.int16, fill=0)
                    cb0 = O.orc_quantize(P(c0), P(q0), qp, size, typ, None)
                    cb1 = E.ref_quantize_lbd(P(c0), P(q1), qp, size, typ, None)
                    assert cb0 == cb1 and (q0 == q1).all(), (size, fast, name, qp, typ)
                r0 = aligned((size, size), np.int16, fill=0); r1 = aligned((size, size), np.int16, fill=0)
                O.orc_dequantize(P(q0), P(r0), qp, size, None)
                R.dequantize_lbd(P(q1), P(r1), qp, size, None)
                assert (r0 == r1).all(), (size, fast, name, qp)
                b0 = aligned((size, size), np.int16, fill=0); b1 = aligned((size, size), np.int16, fill=0)
                O.orc_inverse_transform(P(r0), P(b0), size, bd)
                R.inverse_transform(P(r1), P(b1), size, bd)
                assert (b0 == b1).all(), (size, fast, name, qp)
        # the patterns reach the int16 bound wherever scale^2 full-scale residuals can: 128x128 without fast only at 12 bits
        assert crossed == (scale * scale * ((1 << bd) - 1) > 16383), (size, fast)


def test_calc_cbp():
    rng = np.random.default_rng(6)
    E = ref_enc(0)
    for size in (4, 8, 16):
        for _ in range(300):
            amp = int(rng.choice([2, 6, 40]))
            blk = aligned((size, size), np.int16)
            blk[...] = rng.integers(-amp, amp + 1, (size, size))
            thr = int(rng.integers(1, 60))
            assert O.orc_calc_cbp(P(blk), size, thr) == R.calc_cbp_simd(P(blk), size, thr)
            assert O.orc_calc_cbp_c(P(blk), size, thr) == E.ref_calc_cbp_lbd(P(blk), size, thr)


@pytest.mark.parametrize("hbd,bd", BD)
def test_residual_reconstruct_avg(hbd, bd):
    rng = np.random.default_rng(7)
    s = sfx(hbd)
    E = ref_enc(hbd)
    for size in (4, 8, 16, 32, 64):
        a = rand_plane(rng, size, size, bd, hbd); b = rand_plane(rng, size, size + 16, bd, hbd)
        r0 = aligned((size, size), np.int16); r1 = aligned((size, size), np.int16)
        getattr(O, "orc_residual_" + s)(P(r0), P(a), P(b), size, size, size + 16)
        getattr(E, "ref_get_residual_" + s)(P(r1), P(a), P(b), size, size, size + 16)
        assert (r0 == r1).all()
        r0[...] = rng.integers(-(2 << bd), 2 << bd, (size, size))
        o0 = aligned((size, size + 16), sdt(hbd), fill=0); o1 = aligned((size, size + 16), sdt(hbd), fill=0)
        getattr(O, "orc_reconstruct_" + s)(P(r0), P(a), P(o0), size, size, size + 16, bd)
        getattr(R, "reconstruct_block_" + s)(P(r0), P(a), P(o1), size, size, size + 16, bd)
        assert (o0 == o1).all()
        if size >= 4:
            c = rand_plane(rng, size, size + 16, bd, hbd)
            o0[...] = 0; o1[...] = 0
            getattr(O, "orc_block_avg_" + s)(P(o0), P(b), P(c), size + 16, size + 16, size + 16, size, size)
            getattr(R, "block_avg_simd_" + s)(P(o1), P(b), P(c), size + 16, size + 16, size + 16, size, size)
            assert (o0 == o1).all()


@pytest.mark.parametrize("hbd,bd", BD)
def test_intra(hbd, bd):
    rng = np.random.default_rng(8)
    s = sfx(hbd)
    W, H = 160, 128
    frame = rand_plane(rng, H + 8, W + 8, bd, hbd)
    dt = sdt(hbd)
    for size in (4, 8, 16, 32, 64):
        for trial in range(30):
            cb = size * int(rng.choice([1, 2]))  # coding block = TU or 2x2 TUs
            tb_split = int(cb != size)
            xpos = int(rng.integers(0, (W - cb) // cb + 1)) * cb
            ypos = int(rng.integers(0, (H - cb) // cb + 1)) * cb
            if trial % 5 == 0: xpos = 0
            if trial % 7 == 0: ypos = 0
            i = int(rng.integers(0, 2)) * size if tb_split else 0
            j = int(rng.integers(0, 2)) * size if tb_split else 0
            ur, dl = int(rng.integers(0, 2)), int(rng.integers(0, 2))
            rblock = rand_plane(rng, cb + 2, cb + 2, bd, hbd)
            base = (4 + ypos) * (W + 8) + 4 + xpos
            res = []
            for lib, pre in ((O, "orc_"), (R, "")):
                left = aligned((2 * 128 + 8,), dt, fill=0); top = aligned((2 * 128 + 8,), dt, fill=0); tl = aligned((1,), dt, fill=0)
                name = (pre + "make_top_and_left_" + s)
                getattr(lib, name)(P(left), P(top), P(tl), P(frame, base), W + 8, P(rblock, (1 + i) * (cb + 2) + 1 + j), cb + 2, i, j,
                                   ypos, xpos, size, ur, dl, tb_split, bd)
                preds = []
                for mode in range(10):
                    pb = aligned((size, size), dt, fill=0)
                    fn = getattr(lib, "orc_intra_pred_" + s if lib is O else "get_intra_prediction_" + s)
                    fn(P(left), P(top), int(tl[0]), ypos, xpos, size, P(pb), size, mode, bd)
                    preds.append(pb.copy())
                res.append((left[:2 * size].copy(), top[:2 * size].copy(), int(tl[0]), preds))
            assert (res[0][0] == res[1][0]).all() and (res[0][1] == res[1][1]).all() and res[0][2] == res[1][2]
            for m in range(10):
                assert (res[0][3][m] == res[1][3][m]).all(), (size, m)


@pytest.mark.parametrize("hbd,bd", BD)
def test_intra_full_scale_neighbours(hbd, bd):
    """every intra mode and size with neighbours at 0 and 2^bd-1 (the planar pre-filter's int16 input reaches 8 (2^bd-1), 32760 at 12 bits)"""
    s = sfx(hbd)
    dt = sdt(hbd)
    W, H = 192, 128
    for name, v in full_scale_planes(H + 8, W + 8, (1 << bd) - 1).items():
        frame = aligned((H + 8, W + 8), dt)
        frame[...] = v
        rblock = aligned((130, 130), dt, fill=0)
        for size in (4, 8, 16, 32, 64):
            for xpos, ypos in ((0, 0), (size, 0), (0, size), (size, size), (W - 2 * size, H - 2 * size)):
                base = (4 + ypos) * (W + 8) + 4 + xpos
                ur, dl = int(ypos > 0 and xpos + size < W), int(xpos > 0 and ypos + size < H)
                res = []
                for lib, pre in ((O, "orc_"), (R, "")):
                    left = aligned((2 * 128 + 8,), dt, fill=0); top = aligned((2 * 128 + 8,), dt, fill=0); tl = aligned((1,), dt, fill=0)
                    getattr(lib, pre + "make_top_and_left_" + s)(P(left), P(top), P(tl), P(frame, base), W + 8, P(rblock, 131), 130, 0, 0, ypos, xpos, size, ur, dl, 0, bd)
                    preds = []
                    for mode in range(10):
                        pb = aligned((size, size), dt, fill=0)
                        fn = getattr(lib, "orc_intra_pred_" + s if lib is O else "get_intra_prediction_" + s)
                        fn(P(left), P(top), int(tl[0]), ypos, xpos, size, P(pb), size, mode, bd)
                        preds.append(pb.copy())
                    res.append(preds)
                for m in range(10):
                    assert (res[0][m] == res[1][m]).all(), (name, size, xpos, ypos, m)


@pytest.mark.parametrize("hbd,bd", BD)
def test_cfl(hbd, bd):
    rng = np.random.default_rng(9)
    s = sfx(hbd)
    hit = 0
    # the remap needs a mean squared luma residual above 64 << 2 (bd - 8) (common/common_block.c:361); the noise grows with it above 10 bits
    ns = 1 << max(0, bd - 10)
    for n in (8, 16, 32, 64):
        for trial in range(40):
            y = rand_plane(rng, n, n, bd, hbd, smooth=True)
            ry = aligned((n, n + 8), sdt(hbd))
            ry[...] = np.clip(y.astype(int)[:, :1] * 0 + np.pad(y.astype(int), ((0, 0), (0, 8)), mode="edge") + rng.integers(-40, 41, (n, n + 8)) * (trial % 3) * ns, 0,
                              (1 << bd) - 1)
            k = float(rng.uniform(-1.5, 1.5))
            ys = y.astype(int).reshape(n // 2, 2, n // 2, 2).sum(axis=(1, 3)) // 4
            u0 = aligned((n // 2, n // 2), sdt(hbd)); v0 = aligned((n // 2, n // 2), sdt(hbd))
            u0[...] = np.clip(ys * k + (1 << (bd - 1)) * (1 - k) + rng.integers(-3, 4, ys.shape) * ns, 0, (1 << bd) - 1)
            v0[...] = np.clip(ys * -k + (1 << (bd - 1)) * (1 + k) + rng.integers(-30, 31, ys.shape) * ns, 0, (1 << bd) - 1)
            u1, v1 = u0.copy(), v0.copy()
            u1 = aligned(u0.shape, sdt(hbd), fill=0); u1[...] = u0; v1 = aligned(v0.shape, sdt(hbd), fill=0); v1[...] = v0
            ub = u0.copy()
            getattr(O, "orc_cfl_" + s)(P(y), P(u0), P(v0), P(ry), n, n, n + 8, 1, bd)
            getattr(R, "improve_uv_prediction_" + s)(P(y), P(u1), P(v1), P(ry), n, n, n + 8, 1, bd)
            assert (u0 == u1).all() and (v0 == v1).all()
            hit += int((ub != u0).any())
    assert hit > 10  # the remapping branch was really exercised


@pytest.mark.parametrize("hbd,bd", BD)
@pytest.mark.parametrize("dims", [(192, 136), (320, 192)])
def test_deblock(hbd, bd, dims):
    rng = np.random.default_rng(10)
    s = sfx(hbd)
    w, h = dims
    changed = False
    for qp in (20, 32, 45):
        f = Frame(w, h, bd, hbd, 32, 32)
        f.randomize(rng)
        bi, dd = random_blkinfo(rng, w, h)
        g = f.copy()
        getattr(R, "deblock_frame_y_" + s)(C.byref(g.s), dd, w, h, qp, bd)
        getattr(R, "deblock_frame_uv_" + s)(C.byref(g.s), dd, w, h, O.orc_chroma_qp(qp), bd)
        before = f.y.copy()
        getattr(O, "orc_deblock_y_" + s)(P(f.Y, f.origin(0)), f.sy, P(bi), w, h, qp, bd)
        getattr(O, "orc_deblock_uv_" + s)(P(f.U, f.origin(1)), P(f.V, f.origin(1)), f.sc, P(bi), w, h, 1, O.orc_chroma_qp(qp), bd)
        changed |= bool((before != f.y).any())  # at low qp a noisy frame may pass every edge unfiltered (seen when fuzzing the seeds)
        assert (f.Y == g.Y).all() and (f.U == g.U).all() and (f.V == g.V).all()
    assert changed  # the filter did something at some qp: the comparison above is not vacuous


@pytest.mark.parametrize("hbd,bd", BD)
def test_clpf(hbd, bd):
    rng = np.random.default_rng(11)
    s = sfx(hbd)
    E = ref_enc(hbd)
    w, h = 200, 136
    f = Frame(w, h, bd, hbd, 32, 32)
    f.randomize(rng)
    org = f.copy()
    org.randomize(rng)
    org.y[...] = np.clip(f.y.astype(int) + rng.integers(-6, 7, f.y.shape), 0, (1 << bd) - 1)
    bi, dd = random_blkinfo(rng, w, h)
    # block level, every boundary combination, C and SIMD forms
    for (sx, sy) in [(8, 8), (4, 4), (8, 4), (4, 8)]:
        for bt in range(16):
            for strength in (1, 2, 4):
                x0, y0 = 8 * int(rng.integers(1, 10)), 8 * int(rng.integers(1, 8))
                d0 = aligned((h, w), sdt(hbd), fill=0); d1 = aligned((h, w), sdt(hbd), fill=0); d2 = aligned((h, w), sdt(hbd), fill=0)
                st, dmp = strength << (bd - 8), bd - 4 + 2
                getattr(O, "orc_clpf_block_" + s)(P(f.Y, f.origin(0)), P(d0), f.sy, w, x0, y0, sx, sy, bt, st, dmp)
                getattr(R, "clpf_block_" + s)(P(f.Y, f.origin(0)), P(d1), f.sy, w, x0, y0, sx, sy, bt, st, dmp)
                assert (d0 == d1).all()
                if bt:
                    getattr(R, "clpf_block%d_%s" % (sx, s))(P(f.Y, f.origin(0)), P(d2), f.sy, w, x0, y0, sy, bt, st, dmp)
                else:
                    getattr(R, "clpf_block%d_noclip_%s" % (sx, s))(P(f.Y, f.origin(0)), P(d2), f.sy, w, x0, y0, sy, st, dmp)
                assert (d0 == d2).all(), (sx, sy, bt)
    # detect sums (C semantics; the SIMD detect_clpf adds the same sums twice, enc_kernels.c:259)
    for _ in range(100):
        x0, y0 = 8 * int(rng.integers(0, w // 8)), 8 * int(rng.integers(0, h // 8))
        strength = int(rng.choice([1, 2, 4])) << (bd - 8)
        a = (C.c_int * 2)(5, 7); b = (C.c_int * 2)(5, 7); c = (C.c_int * 2)(0, 0)
        args = (P(f.Y, f.origin(0)), P(org.Y, org.origin(0)), x0, y0, w, h, org.sy, f.sy)
        getattr(O, "orc_detect_clpf_" + s)(*args, C.byref(a, 0), C.byref(a, 4), strength, bd - 8, 8, bd - 4 + 2)
        getattr(R, "detect_clpf_" + s)(*args, C.byref(b, 0), C.byref(b, 4), strength, bd - 8, 8, bd - 4 + 2)
        assert list(a) == list(b)
        getattr(R, "detect_clpf_simd_" + s)(*args, C.byref(c, 0), C.byref(c, 4), strength, bd - 8, 8, bd - 4 + 2)
        assert [c[0], c[1]] == [2 * (a[0] - 5), 2 * (a[1] - 7)]
        m0 = (C.c_int * 4)(1, 2, 3, 4); m1 = (C.c_int * 4)(1, 2, 3, 4); m2 = (C.c_int * 4)(1, 2, 3, 4)
        getattr(O, "orc_detect_multi_clpf_" + s)(*args, m0, bd - 8, 8, bd - 4 + 2)
        getattr(R, "detect_multi_clpf_" + s)(*args, m1, bd - 8, 8, bd - 4 + 2)
        getattr(R, "detect_multi_clpf_simd_" + s)(*args, m2, bd - 8, 8, bd - 4 + 2)
        assert list(m0) == list(m1) == list(m2)
    # whole plane through the reference's cached in-place clpf_frame (no per-block decision)
    for plane in (0, 1, 2):
        for fbl, strength in ((7, 1), (6, 2), (5, 4), (4, 2)):
            if plane and fbl != 4:
                continue
            g = f.copy()
            getattr(R, "clpf_frame_" + s)(C.byref(g.s), C.byref(org.s), dd, None, 0, strength, fbl, bd, plane, 33, None)
            src = f.full(plane)
            dst = src.copy()
            pw, ph = (w, h) if plane == 0 else (w // 2, h // 2)
            getattr(O, "orc_clpf_plane_" + s)(P(src, f.origin(plane)), P(dst, f.origin(plane)), f.stride(plane), pw, ph, P(bi), w // 4, int(plane != 0), None,
                                              fbl, strength, bd, plane, 33)
            o = f.origin(plane); st = f.stride(plane)
            vis = lambda a: a.reshape(-1)[o:o + ph * st].reshape(ph, st)[:, :pw]
            assert (vis(dst) != vis(src)).any()
            assert (vis(dst) == vis(g.full(plane))).all(), (plane, fbl)


@pytest.mark.parametrize("hbd,bd", BD)
def test_cdef(hbd, bd):
    rng = np.random.default_rng(12)
    s = sfx(hbd)
    w, h = 200, 136
    f = Frame(w, h, bd, hbd, 32, 32)
    f.randomize(rng)
    bi, dd = random_blkinfo(rng, w, h)
    for _ in range(200):
        x0, y0 = 8 * int(rng.integers(0, w // 8)), 8 * int(rng.integers(0, h // 8))
        v0, v1, v2 = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        p = P(f.Y, f.origin(0) + y0 * f.sy + x0)
        d0 = getattr(O, "orc_cdef_find_dir_" + s)(p, f.sy, C.byref(v0), bd - 8)
        d1 = getattr(R, "cdef_find_dir_" + s)(p, f.sy, C.byref(v1), bd - 8)
        d2 = getattr(R, "cdef_find_dir_simd_" + s)(p, f.sy, C.byref(v2), bd - 8)
        assert (d0, v0.value) == (d1, v1.value) == (d2, v2.value)
    # block filter: random strengths, all boundary types, both block sizes
    dirs = np.zeros((8, 2), np.int32)
    for d in range(8):
        dx = [[1, 2], [1, 2], [1, 2], [1, 2], [1, 2], [0, 1], [0, 0], [0, -1]][d]
        dy = [[-1, -2], [0, -1], [0, 0], [0, 1], [1, 2], [1, 2], [1, 2], [1, 2]][d]
        dirs[d] = [dy[0] * 32 + dx[0], dy[1] * 32 + dx[1]]
    cs = bd - 8
    for trial in range(300):
        bs = int(rng.choice([4, 8]))
        plane = 0 if bs == 8 else 1
        pw, ph = (w, h) if plane == 0 else (w // 2, h // 2)
        x0, y0 = bs * int(rng.integers(0, pw // bs)), bs * int(rng.integers(0, ph // bs))
        bt = (1 if x0 == 0 else 0) | (4 if y0 == 0 else 0) | (2 if x0 == pw - bs else 0) | (8 if y0 == ph - bs else 0)
        if trial % 3 == 0:
            bt = int(rng.integers(0, 16))
        # tile layout as in the reference (common/common_frame.c:862-865): (0,0) 32-byte aligned, pitch 32
        t0 = aligned((12, 32), np.uint16, fill=0); t1 = aligned((12, 32), np.uint16, fill=0)
        src = f.full(plane)
        getattr(O, "orc_cdef_prepare_input_" + s)(bs, bs, x0, y0, bt, 2, P(t0, 2 * 32 + 16), 32, P(src, f.origin(plane)), f.stride(plane))
        getattr(R, "cdef_prepare_input_" + s)(bs, bs, x0, y0, bt, 2, P(t1, 2 * 32 + 16), 32, P(src, f.origin(plane)), f.stride(plane))
        assert (t0[:bs + 4, 14:14 + bs + 4] == t1[:bs + 4, 14:14 + bs + 4]).all()
        pri = int(rng.integers(0, 16)) << cs; sec = int(rng.choice([0, 1, 2, 4])) << cs
        d = int(rng.integers(0, 8))
        pd = max(int(np.log2(pri >> cs)) if pri >> cs else 0, 5 - plane) + cs; sd = 5 - plane + cs
        o0 = aligned((bs, bs), sdt(hbd), fill=0); o1 = aligned((bs, bs), sdt(hbd), fill=0); o2 = aligned((bs, bs), sdt(hbd), fill=0)
        dptr = lambda o: (P(o), None) if not hbd else (None, P(o))
        O.orc_cdef_filter_block(*dptr(o0), bs, P(t0, 2 * 32 + 16), 32, pri, sec, d, pd, sd, bs, cs)
        R.cdef_filter_block(*dptr(o1), bs, P(t0, 2 * 32 + 16), 32, pri, sec, d, pd, sd, bs, P(dirs), cs)
        R.cdef_filter_block_simd(*dptr(o2), bs, P(t0, 2 * 32 + 16), 32, pri, sec, d, pd, sd, bs, P(dirs), cs)
        assert (o0 == o1).all() and (o0 == o2).all(), (bs, pri, sec, d, bt)
    # whole frame through the reference's cached in-place cdef_frame
    nfb = ((w + 63) // 64) * ((h + 63) // 64)
    cst = (CdefStrengths * nfb)()
    pri = np.zeros((2, nfb), np.int8); sec = np.zeros((2, nfb), np.int8)
    for i in range(nfb):
        for pl in range(2):
            pri[pl, i] = int(rng.integers(0, 16)); sec[pl, i] = int(rng.integers(0, 4))
            cst[i].plane[pl].level = int(pri[pl, i]); cst[i].plane[pl].sec_strength = int(sec[pl, i])
            cst[i].plane[pl].pri_damping = cst[i].plane[pl].sec_damping = 5
    g = f.copy()
    dirs_o = np.zeros((nfb, 64), np.int32); vars_o = np.zeros((nfb, 64), np.int32)
    for plane in (0, 1, 2):
        getattr(R, "cdef_frame_" + s)(cst, C.byref(g.s), None, dd, None, 0, bd, plane)
        src = f.full(plane)
        dst = src.copy()
        getattr(O, "orc_cdef_plane_" + s)(P(src, f.origin(plane)), P(dst, f.origin(plane)), f.stride(plane), w, h, P(bi), w // 4, 1, plane,
                                          P(pri[int(plane != 0)]), P(sec[int(plane != 0)]), 5, 5, P(dirs_o), P(vars_o), bd)
        pw, ph = (w, h) if plane == 0 else (w // 2, h // 2)
        o = f.origin(plane); st = f.stride(plane)
        vis = lambda a: a.reshape(-1)[o:o + ph * st].reshape(ph, st)[:, :pw]
        assert (vis(dst) != vis(src)).any()
        assert (vis(dst) == vis(g.full(plane))).all(), plane


@pytest.mark.parametrize("hbd,bd", BD)
def test_pad_and_scale(hbd, bd):
    rng = np.random.default_rng(13)
    s = sfx(hbd)
    f = Frame(176, 144, bd, hbd)
    f.randomize(rng, smooth=False)
    g = f.copy()
    getattr(R, "pad_yuv_frame_" + s)(C.byref(g.s))
    getattr(O, "orc_pad_plane_" + s)(P(f.Y, f.origin(0)), f.sy, 176, 144, 160, 160)
    getattr(O, "orc_pad_plane_" + s)(P(f.U, f.origin(1)), f.sc, 88, 72, 80, 80)
    getattr(O, "orc_pad_plane_" + s)(P(f.V, f.origin(1)), f.sc, 88, 72, 80, 80)
    H = 144 + 320
    assert (f.Y[:H, :176 + 320] == g.Y[:H, :176 + 320]).all() and (f.U[:72 + 160, :88 + 160] == g.U[:72 + 160, :88 + 160]).all()
    assert (f.V[:72 + 160, :88 + 160] == g.V[:72 + 160, :88 + 160]).all()
    small0 = Frame(88, 72, bd, hbd); small1 = Frame(88, 72, bd, hbd)
    getattr(R, "scale_frame_down2x2_simd_" + s)(C.byref(g.s), C.byref(small1.s))
    getattr(O, "orc_scale_down2x2_" + s)(P(f.Y, f.origin(0)), f.sy, P(small0.Y, small0.origin(0)), small0.sy, 88, 72)
    assert (small0.y == small1.y).all()


@pytest.mark.parametrize("hbd,bd", BD)
def test_motion_estimate(hbd, bd):
    rng = np.random.default_rng(14)
    s = sfx(hbd)
    E = ref_enc(hbd)
    fw, fh = 256, 192
    f = Frame(fw, fh, bd, hbd)
    f.randomize(rng)
    getattr(R, "pad_yuv_frame_" + s)(C.byref(f.s))
    cur = Frame(fw, fh, bd, hbd)
    # current frame = reference shifted by (3,-2) + noise, so the search has a real optimum
    cur.y[...] = np.clip(np.roll(f.y.astype(int), (2, -3), axis=(0, 1)) + rng.integers(-4, 5, f.y.shape), 0, (1 << bd) - 1)
    for trial in range(200):
        size = int(rng.choice([8, 16, 32, 64]))
        part = int(rng.integers(0, 4))  # PART_NONE, HOR, VER, QUAD (incl. the 8x8 quarters of 16x16 blocks: wide-SAD candidates on an 8x8 block)
        width, height = (size, size) if part == 0 else ((size, size // 2) if part == 1 else ((size // 2, size) if part == 2 else (size // 2, size // 2)))
        if min(width, height) < 4: width = height = size
        xpos, ypos = int(rng.integers(0, fw // size)) * size, int(rng.integers(0, fh // size)) * size
        org = aligned((size, size), sdt(hbd))
        org[...] = cur.y[ypos:ypos + size, xpos:xpos + size]
        speed = int(rng.integers(0, 3)); sign = int(rng.integers(0, 2)); bip = int(rng.integers(0, 2))
        lam = float(rng.uniform(2.0, 60.0))
        mvc = (C.c_int16 * 2)(int(rng.integers(-40, 40)), int(rng.integers(-40, 40)))
        mvp = (C.c_int16 * 2)(int(rng.integers(-40, 40)), int(rng.integers(-40, 40)))
        nc = int(rng.integers(0, 7))
        if not (speed == 0 or (size == 16 and bip)):
            nc = max(nc, 1)  # without the telescope stage an empty candidate list leaves mv_opt uninitialised in the reference
        cands = (C.c_int16 * (2 * max(nc, 1)))(*[int(v) for v in rng.integers(-12, 12, 2 * max(nc, 1))])
        m0 = (C.c_int16 * 2)(0, 0); m1 = (C.c_int16 * 2)(0, 0)
        refp = P(f.Y, f.origin(0) + ypos * f.sy + xpos)
        a = getattr(O, "orc_motion_estimate_" + s)(P(org), refp, size, f.sy, width, height, m0, mvc, mvp, C.c_double(lam), speed, bd, sign, fw, fh, xpos, ypos, cands, nc, bip)
        b = getattr(E, "ref_motion_estimate_" + s)(P(org), refp, size, f.sy, width, height, m1, mvc, mvp, C.c_double(lam), speed, bd, sign, fw, fh, xpos, ypos, cands, nc, bip)
        assert (a, m0[0], m0[1]) == (b, m1[0], m1[1]), (trial, size, width, height, speed, sign, bip)
    # edge placement: blocks in the first / last row and column whose best match lies at or past clip_mv's limit, on a picture whose width is
    # a multiple of 16 and on one whose width is not
    reach = np.zeros((2, 2), int)  # [sign][on a clip limit, through an active split_mv clamp]
    for fw, fh in ((256, 192), (200, 136)):
        f = Frame(fw, fh, bd, hbd)
        f.randomize(rng)
        getattr(R, "pad_yuv_frame_" + s)(C.byref(f.s))
        for trial in range(160):
            size = int(rng.choice([8, 16, 32, 64]))
            part = trial % 4
            width, height = (size, size) if part == 0 else ((size, size // 2) if part == 1 else ((size // 2, size) if part == 2 else (size // 2, size // 2)))
            speed, sign, bip = trial // 4 % 3, trial // 12 % 2, trial // 24 % 2
            xpos, ypos, blk, mvc, mvp, near = edge_search(rng, f.Y, fw, fh, size, width, height, sign, bd)
            org = aligned((size, size), sdt(hbd))
            org[...] = blk
            nc = int(rng.integers(0 if speed == 0 or (size == 16 and bip) else 1, 7))
            cl = near(max(nc, 1))
            cands = (C.c_int16 * (2 * len(cl)))(*[v for c in cl for v in c])
            lam = float(rng.uniform(2.0, 60.0))
            m0 = (C.c_int16 * 2)(0, 0); m1 = (C.c_int16 * 2)(0, 0)
            refp = P(f.Y, f.origin(0) + ypos * f.sy + xpos)
            args = (size, f.sy, width, height)
            rest = ((C.c_int16 * 2)(*mvc), (C.c_int16 * 2)(*mvp), C.c_double(lam), speed, bd, sign, fw, fh, xpos, ypos, cands, nc, bip)
            a = getattr(O, "orc_motion_estimate_" + s)(P(org), refp, *args, m0, *rest)
            b = getattr(E, "ref_motion_estimate_" + s)(P(org), refp, *args, m1, *rest)
            assert (a, m0[0], m0[1]) == (b, m1[0], m1[1]), ("edge", fw, trial, xpos, ypos, size, width, height, speed, sign, bip, mvc, mvp, nc)
            reach[sign] += edge_reach(m0[0], m0[1], sign, xpos, ypos, fw, fh, size, width, height)
    assert (reach >= ME_EDGE_REACH).all(), reach


def _ti_pair(rng, w, h, bd, hbd, hard):
    """two padded frames: the second is the first shifted by (1,-2) + noise, with one displaced patch; hard=True adds enough
    noise that the skip test fails almost everywhere and the candidate/cross search runs"""
    a = Frame(w, h, bd, hbd)
    a.randomize(rng)
    b = Frame(w, h, bd, hbd)
    amp = 14 if hard else 3
    for p in range(3):
        sh = (1, -2) if p == 0 else (0, -1)
        b.plane(p)[...] = np.clip(np.roll(a.plane(p).astype(int), sh, axis=(0, 1)) + rng.integers(-amp, amp + 1, a.plane(p).shape), 0, (1 << bd) - 1)
    b.y[h // 4:h // 4 + 40, w // 3:w // 3 + 56] = np.clip(a.y[h // 4 + 6:h // 4 + 46, w // 3 - 9:w // 3 + 47].astype(int) + 20, 0, (1 << bd) - 1)
    return a, b


def ti_levels(w, h):
    import math
    return min(4, int(math.log10(min(w, h)) / math.log10(2.0) - 4.0))  # common/temporal_interp.c:914


@pytest.mark.parametrize("hbd,bd", BD)
def test_interpolate_frames(hbd, bd):
    rng = np.random.default_rng(15)
    s = sfx(hbd)
    for (w, h) in [(128, 72), (192, 136), (320, 192)]:
        for hard in (False, True):
            for ratio, pos in [(2, 1), (4, 1), (4, 3), (8, 5)]:
                a, b = _ti_pair(rng, w, h, bd, hbd, hard)
                getattr(R, "pad_yuv_frame_" + s)(C.byref(a.s)); getattr(R, "pad_yuv_frame_" + s)(C.byref(b.s))
                o1 = Frame(w, h, bd, hbd); o2 = Frame(w, h, bd, hbd)
                getattr(R, "interpolate_frames_" + s)(C.byref(o1.s), C.byref(a.s), C.byref(b.s), ratio, pos)
                getattr(O, "orc_interpolate_frames_" + s)(P(o2.Y, o2.origin(0)), P(o2.U, o2.origin(1)), P(o2.V, o2.origin(1)), o2.sy, o2.sc,
                                                         P(a.Y, a.origin(0)), P(a.U, a.origin(1)), P(a.V, a.origin(1)), P(b.Y, b.origin(0)), P(b.U, b.origin(1)),
                                                         P(b.V, b.origin(1)), a.sy, a.sc, w, h, 160, ratio, pos, ti_levels(w, h))
                for p in range(3):
                    assert (o1.plane(p) == o2.plane(p)).all(), (w, h, hard, ratio, pos, p)
                assert (o1.y != a.y).any()


@pytest.mark.parametrize("hbd,bd", BD)
def test_motion_estimate_bi_and_combine(hbd, bd):
    rng = np.random.default_rng(16)
    s = sfx(hbd)
    E = ref_enc(hbd)
    fw, fh = 192, 128
    f0 = Frame(fw, fh, bd, hbd); f0.randomize(rng)
    f1 = Frame(fw, fh, bd, hbd)
    f1.y[...] = np.clip(np.roll(f0.y.astype(int), (2, 3), axis=(0, 1)) + rng.integers(-4, 5, f0.y.shape), 0, (1 << bd) - 1)
    for f in (f0, f1):
        getattr(R, "pad_yuv_frame_" + s)(C.byref(f.s))
    cur = np.clip((f0.y.astype(int) + np.roll(f0.y.astype(int), (1, 1), axis=(0, 1))) // 2 + rng.integers(-3, 4, f0.y.shape), 0, (1 << bd) - 1)
    for trial in range(40):
        size = int(rng.choice([8, 16, 32, 64]))
        xpos, ypos = int(rng.integers(0, fw // size)) * size, int(rng.integers(0, fh // size)) * size
        org = aligned((size, size), sdt(hbd))
        org[...] = cur[ypos:ypos + size, xpos:xpos + size]
        sign = int(rng.integers(0, 2)); lam = float(rng.uniform(2.0, 40.0))
        mvc = (C.c_int16 * 2)(int(rng.integers(-30, 30)), int(rng.integers(-30, 30)))
        mvp = (C.c_int16 * 2)(int(rng.integers(-30, 30)), int(rng.integers(-30, 30)))
        nc = int(rng.integers(0, 7))
        cands = (C.c_int16 * 16)(*[int(v) for v in rng.integers(-20, 20, 16)])
        m0 = (C.c_int16 * 2)(0, 0); m1 = (C.c_int16 * 2)(0, 0)
        p0 = P(f0.Y, f0.origin(0) + ypos * f0.sy + xpos); p1 = P(f1.Y, f1.origin(0) + ypos * f1.sy + xpos)
        a = getattr(O, "orc_motion_estimate_bi_" + s)(P(org), p0, p1, size, f0.sy, size, size, m0, mvc, mvp, C.c_double(lam), bd, sign, fw, fh, xpos, ypos, cands, nc, 1)
        b = getattr(E, "ref_motion_estimate_bi_" + s)(P(org), p0, p1, size, f0.sy, size, size, m1, mvc, mvp, C.c_double(lam), bd, sign, fw, fh, xpos, ypos, cands, nc, 1)
        assert (a, m0[0], m0[1]) == (b, m1[0], m1[1]), (trial, size, sign, nc)
    # edge placement (see test_motion_estimate); the list entries are quarter-pel vectors, and a vector clipped for one reference is clipped
    # again with the other sign for the second
    reach = np.zeros((2, 2), int)
    for fw, fh in ((256, 192), (200, 136)):
        f0 = Frame(fw, fh, bd, hbd); f0.randomize(rng)
        f1 = Frame(fw, fh, bd, hbd)
        f1.y[...] = np.clip(np.roll(f0.y.astype(int), (2, 3), axis=(0, 1)) + rng.integers(-4, 5, f0.y.shape), 0, (1 << bd) - 1)
        for f in (f0, f1):
            getattr(R, "pad_yuv_frame_" + s)(C.byref(f.s))
        for trial in range(48):
            size = [8, 16, 32, 64][trial % 4]; sign = trial // 4 % 2
            xpos, ypos, blk, mvc, mvp, near = edge_search(rng, f0.Y, fw, fh, size, size, size, sign, bd)
            org = aligned((size, size), sdt(hbd))
            org[...] = blk
            nc = int(rng.integers(0, 5))
            cands = (C.c_int16 * 8)(*[4 * v + int(rng.integers(-3, 4)) for c in near(4) for v in c])
            lam = float(rng.uniform(2.0, 40.0))
            m0 = (C.c_int16 * 2)(0, 0); m1 = (C.c_int16 * 2)(0, 0)
            p0 = P(f0.Y, f0.origin(0) + ypos * f0.sy + xpos); p1 = P(f1.Y, f1.origin(0) + ypos * f1.sy + xpos)
            rest = ((C.c_int16 * 2)(*mvc), (C.c_int16 * 2)(*mvp), C.c_double(lam), bd, sign, fw, fh, xpos, ypos, cands, nc, 1)
            a = getattr(O, "orc_motion_estimate_bi_" + s)(P(org), p0, p1, size, f0.sy, size, size, m0, *rest)
            b = getattr(E, "ref_motion_estimate_bi_" + s)(P(org), p0, p1, size, f0.sy, size, size, m1, *rest)
            assert (a, m0[0], m0[1]) == (b, m1[0], m1[1]), ("edge", fw, trial, xpos, ypos, size, sign, mvc, mvp, nc)
            reach[sign] += np.logical_or(*[edge_reach(m0[0], m0[1], sg, xpos, ypos, fw, fh, size, size, size) for sg in (sign, 1 - sign)])
    assert (reach >= ME_BI_EDGE_REACH).all(), reach
    # element-wise combinations: op 0 against average_blocks_all, op 2 against block_avg_simd, op 1 against its definition
    from _refstructs import Mv
    class BlockPos(C.Structure):
        _fields_ = [("ypos", C.c_uint16), ("xpos", C.c_uint16), ("size", C.c_uint8), ("bwidth", C.c_uint8), ("bheight", C.c_uint8), ("sb_size", C.c_uint8)]
    for size in (8, 16, 64):
        a = rand_plane(rng, size, size, bd, hbd); b = rand_plane(rng, size, size, bd, hbd)
        ac = rand_plane(rng, size // 2, size // 2, bd, hbd); bc = rand_plane(rng, size // 2, size // 2, bd, hbd)
        o0 = aligned((size, size), sdt(hbd), fill=0); o1 = aligned((size, size), sdt(hbd), fill=0)
        u1 = aligned((size // 2, size // 2), sdt(hbd), fill=0); v1 = aligned((size // 2, size // 2), sdt(hbd), fill=0)
        bp = BlockPos(0, 0, size, size, size, 128)
        getattr(R, "average_blocks_all_" + s)(P(o1), P(u1), P(v1), P(a), P(ac), P(ac), P(b), P(bc), P(bc), C.byref(bp), 1)
        getattr(O, "orc_block_combine_" + s)(P(o0), size, P(a), size, P(b), size, size, size, 0, bd)
        assert (o0 == o1).all()
        getattr(O, "orc_block_combine_" + s)(P(o0), size, P(a), size, P(b), size, size, size, 1, bd)
        assert (o0 == np.clip(2 * a.astype(int) - b.astype(int), 0, (1 << bd) - 1)).all()
        getattr(O, "orc_block_combine_" + s)(P(o0), size, P(a), size, P(b), size, size, size, 2, bd)
        getattr(R, "block_avg_simd_" + s)(P(o1), P(a), P(b), size, size, size, size, size)
        assert (o0 == o1).all()


@pytest.mark.parametrize("hbd,bd", BD)
def test_cdef_search(hbd, bd):
    """encoder-side CDEF strength search: oracle distortion table + greedy selection against the reference's cdef_search()"""
    from _libs import ref_frame
    F = ref_frame(hbd)
    rng = np.random.default_rng(17)
    s = sfx(hbd)
    # dist_8x8 (double arithmetic)
    for _ in range(300):
        a = rand_plane(rng, 8, 24, bd, hbd, smooth=bool(rng.integers(0, 2))); b = aligned((8, 8), sdt(hbd))
        b[...] = np.clip(a[:, :8].astype(int) + rng.integers(-9, 10, (8, 8)), 0, (1 << bd) - 1)
        assert getattr(O, "orc_dist_8x8_" + s)(P(b), 8, P(a), 24, bd - 8) == getattr(F, "ref_dist_8x8_" + s)(P(b), 8, P(a), 24, bd - 8)
    for (w, h), speed, cbits, qp in [((192, 136), 1, 3, 30), ((320, 192), 1, 1, 40), ((200, 136), 0, 2, 34), ((192, 128), 2, 3, 36)]:
        f = Frame(w, h, bd, hbd, 32, 32)
        f.randomize(rng)
        org = f.copy()
        for p in range(3):
            org.plane(p)[...] = np.clip(f.plane(p).astype(int) + rng.integers(-7, 8, f.plane(p).shape), 0, (1 << bd) - 1)
        bi, dd = random_blkinfo(rng, w, h, p_skip=0.25)
        nfb = ((w + 63) // 64) * ((h + 63) // 64)
        lam = 60.0
        st = (C.c_int * 8)(*[127] * 8); ust = (C.c_int * 8)(*[127] * 8)
        level = (C.c_int * (2 * nfb))(); sec = (C.c_int * (2 * nfb))(); dirs = (C.c_int * (64 * nfb))(); vars_ = (C.c_int * (64 * nfb))(); sbits = C.c_int(0)
        bits = getattr(F, "ref_cdef_search_" + s)(C.byref(f.s), C.byref(org.s), dd, w, h, bd, qp, C.c_double(lam), cbits, speed, st, ust, level, sec, dirs, vars_, C.byref(sbits))
        # oracle: distortion table, then selection
        mse = np.zeros((2, nfb, 64), np.uint64); od = np.zeros((nfb, 64), np.int32); ov = np.zeros((nfb, 64), np.int32); ask = np.zeros(nfb, np.uint8)
        getattr(O, "orc_cdef_search_mse_" + s)(P(f.Y, f.origin(0)), P(f.U, f.origin(1)), P(f.V, f.origin(1)), P(org.Y, org.origin(0)), P(org.U, org.origin(1)),
                                                P(org.V, org.origin(1)), f.sy, f.sc, w, h, P(bi), speed, 5, bd, P(mse), P(od), P(ov), P(ask))
        live = np.flatnonzero(ask == 0)
        m0 = np.ascontiguousarray(mse[0][live]); m1 = np.ascontiguousarray(mse[1][live])
        ost = (C.c_int * 16)(); oust = (C.c_int * 16)(); sel = (C.c_int * max(1, len(live)))()
        obits = O.orc_cdef_select(P(m0), P(m1), len(live), speed, cbits, C.c_double(lam), ost, oust, sel)
        assert obits == bits
        assert list(ost)[:1 << bits] == list(st)[:1 << bits] and list(oust)[:1 << bits] == list(ust)[:1 << bits]
        for k, fb in enumerate(live):
            assert level[2 * fb] == ost[sel[k]] >> 2 and sec[2 * fb] == ost[sel[k]] & 3, (fb, k)
            assert level[2 * fb + 1] == oust[sel[k]] >> 2 and sec[2 * fb + 1] == oust[sel[k]] & 3
            # directions / variances of the blocks inside the frame
            for m in range(8):
                for n in range(8):
                    if (fb % ((w + 63) // 64)) * 64 + n * 8 < w and (fb // ((w + 63) // 64)) * 64 + m * 8 < h:
                        assert od[fb, m * 8 + n] == dirs[fb * 64 + m * 8 + n] and ov[fb, m * 8 + n] == vars_[fb * 64 + m * 8 + n]
        assert sbits.value == bits * len(live)


def test_coeff_bits():
    """SURVEY 8f.2: bits emitted by write_coeff (enc/write_bits.c:145) — oracle length count against the reference's bit writer"""
    R = ref()
    class Stream(C.Structure):
        _fields_ = [("bytesize", C.c_uint32), ("bytepos", C.c_uint32), ("bitstream", C.c_void_p), ("bitbuf", C.c_uint32), ("bitrest", C.c_uint32)]
    buf = (C.c_uint8 * 8192)()
    rng = np.random.default_rng(23)
    # put_vlc code lengths
    st = Stream(8192, 0, C.addressof(buf), 0, 32)
    R.put_vlc.restype = C.c_uint; R.put_vlc.argtypes = [C.c_int, C.c_uint, C.c_void_p]
    for n in (0, 1, 6, 10):
        for cn in list(range(0, 80)) + [127, 128, 255, 1000, 4097, 32768, 65535]:
            assert O.orc_vlc_len(n, cn) == R.put_vlc(n, cn, C.byref(st)), (n, cn)
            st.bytepos = 0
    R.write_coeff.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]; R.write_coeff.restype = None
    R.get_bit_pos.argtypes = [C.c_void_p]
    n = 0
    for size in (4, 8, 16, 32, 64):
        q = min(size, 16)
        for typ in range(4):
            for trial in range(120):
                dens = [0.02, 0.1, 0.3, 0.7, 1.0][trial % 5]
                amp = [1, 2, 5, 40, 3000][(trial // 5) % 5]
                c = aligned((q, q), np.int16)
                c[...] = rng.integers(-amp, amp + 1, (q, q)) * (rng.random((q, q)) < dens)
                if trial % 7 == 0:
                    c[...] = 0; c[0, 0] = rng.choice([-1, 1, 2, -3])
                if trial % 11 == 0:
                    c[q - 1, q - 1] = 1
                if not c.any():
                    assert O.orc_coeff_bits(P(c), size, typ) == 0
                    continue
                st = Stream(8192, 0, C.addressof(buf), 0, 32)
                R.write_coeff(C.byref(st), P(c), size, typ)
                assert O.orc_coeff_bits(P(c), size, typ) == R.get_bit_pos(C.byref(st)), (size, typ, trial)
                n += 1
    assert n > 1500


@pytest.mark.parametrize("hbd,bd", BD)
def test_motion_estimate_sync(hbd, bd):
    """a5 gap of round 1: motion_estimate_sync (enc/encode_block.c:713-796, -sync 1) restated in the oracle and pinned against the reference's file-static function
    through the trampoline.  (No CUDA form yet: the RD-loop binding leaves -sync 1 to the reference's own loop.)"""
    rng = np.random.default_rng(21)
    s = sfx(hbd)
    E = ref_enc(hbd)
    fw, fh = 192, 128
    f0 = Frame(fw, fh, bd, hbd); f0.randomize(rng)
    getattr(R, "pad_yuv_frame_" + s)(C.byref(f0.s))
    cur = np.clip(np.roll(f0.y.astype(int), (1, -2), axis=(0, 1)) + rng.integers(-3, 4, f0.y.shape), 0, (1 << bd) - 1)
    for trial in range(40):
        size = int(rng.choice([8, 16, 32, 64]))
        w, h = size, size
        if trial % 3 == 1: h = size // 2      # PART_HOR
        if trial % 3 == 2: w = size // 2      # PART_VER
        xpos, ypos = int(rng.integers(0, fw // size)) * size, int(rng.integers(0, fh // size)) * size
        org = aligned((size, size), sdt(hbd))
        org[...] = cur[ypos:ypos + size, xpos:xpos + size]
        sign = int(rng.integers(0, 2)); lam = float(rng.uniform(2.0, 40.0)); bip = int(rng.integers(0, 2))
        mvc = (C.c_int16 * 2)(int(rng.integers(-30, 30)), int(rng.integers(-30, 30)))
        mvp = (C.c_int16 * 2)(int(rng.integers(-30, 30)), int(rng.integers(-30, 30)))
        base = [int(v) for v in rng.integers(-40, 40, 16)]
        ca = (C.c_int16 * 16)(*base); cb = (C.c_int16 * 16)(*base)   # both sides scribble on entries 4 and 5
        m0 = (C.c_int16 * 2)(0, 0); m1 = (C.c_int16 * 2)(0, 0)
        p0 = P(f0.Y, f0.origin(0) + ypos * f0.sy + xpos)
        a = getattr(O, "orc_motion_estimate_sync_" + s)(P(org), p0, size, f0.sy, w, h, m0, mvc, mvp, C.c_double(lam), bd, sign, fw, fh, xpos, ypos, ca, bip)
        b = getattr(E, "ref_motion_estimate_sync_" + s)(P(org), p0, size, f0.sy, w, h, m1, mvc, mvp, C.c_double(lam), bd, sign, fw, fh, xpos, ypos, cb, bip)
        assert (a, m0[0], m0[1]) == (b, m1[0], m1[1]), (trial, size, w, h, sign)
        assert list(ca) == list(cb)
