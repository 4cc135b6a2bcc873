"""The frame-level in-loop filters and temporal interpolation across qp, frame geometry, CLPF filter-block flags and real block state.

One table of frame geometries (GEOMS) drives every test here.  The entry points under test are tb_deblock_frame, tb_cdef_frame,
tb_cdef_search_mse, tb_clpf_frame, tb_clpf_detect_frame and tb_interpolate_frames (with the pyramid it builds and caches between calls).

  expected  the compiled reference in oracle/_ref (deblock_frame_y/uv, cdef_frame, clpf_frame with its per-filter-block decision callback,
            detect_multi_clpf, interpolate_frames, cdef_search) when it is present, the plain-C oracle otherwise;
  CPU       the oracle against the reference on every case of the table, so the fallback is pinned where it is used;
  GPU       the device against the expected value, bit-exact on every plane; then the whole filter chain on the reference encoder's own pre-filter
            reconstruction and block state (the committed golden RD-loop jobs, and two captured cases of tests/test_rdo_matrix.py).

The geometries reach what 64-multiple widths do not: partial 64x64 CDEF and CLPF filter blocks in both directions, chroma planes 4 samples wider
than a multiple of 8, a 1-level and a 4-level interpolation pyramid with odd-sized levels, and the only large 10-bit case."""
import ctypes as C
import math

import numpy as np
import pytest

from _libs import oracle, ref, ref_frame, P, sfx
from _refstructs import BLKINFO, CdefStrengths, Frame, deblock_data, random_blkinfo

O = oracle()
R = ref()
HAVE_REF = R is not None and ref_frame(0) is not None and ref_frame(1) is not None
EXPECT = "ref" if HAVE_REF else "oracle"
needs_ref = pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref not built")

GEOMS = [
    # w     h     bit depths  why
    (64,   64,   (8, 10)),   # one CDEF block, one CLPF block at 64 and 128; a 2-level pyramid
    (200,  136,  (8, 10)),   # partial filter blocks in both directions; chroma width 100 (4 mod 8, 4 mod 16)
    (136,  200,  (8, 10)),   # the same, in portrait
    (240,  120,  (8, 10)),   # partial in width, luma width a multiple of 16 (no CDEF-search chroma quirk); a 2-level pyramid
    (424,  264,  (8, 10)),   # a 4-level pyramid whose deepest level is 53x33
    (1920, 1080, (10,)),     # the only large high-bit-depth case
]
CASES = [(w, h, bd) for w, h, bds in GEOMS for bd in bds]
CASE_IDS = ["%dx%d_%dbit" % c for c in CASES]
QPS = (8, 20, 36, 51)                    # every qp >> 4 step of the CLPF damping
DEBLOCK_QPS = (0, 15, 16, 29, 30, 37, 51)
DAMPINGS = ((3, 6), (4, 3), (5, 5), (6, 4))   # (primary, secondary): 3..6 each, as the 2-bit field of the stream allows
DECISION = C.CFUNCTYPE(C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_uint, C.c_uint,
                       C.c_uint, C.c_uint, C.c_int)   # clpf_frame's decision callback (common/common_frame.h:50)


def hbd_of(bd):
    return int(bd > 8)


def nfb64(w, h):
    return ((w + 63) >> 6) * ((h + 63) >> 6)


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# content and block state
# ---------------------------------------------------------------------------------------------------------------------------------------------------
def content(seed, w, h, bd, noisy):
    """(reconstruction, original): the seeded Frame.randomize content; noisy=True adds noise of a third of the range, clipped to 0 and 2^bd-1, and a
    checkerboard of 8x8 blocks at 0 and 2^bd-1 (the idea of test_rdo_matrix.hard_yuv)"""
    rng = np.random.default_rng(seed)
    maxv = (1 << bd) - 1
    f = Frame(w, h, bd, hbd_of(bd), 32, 32)
    f.randomize(rng)
    if noisy:
        for p in range(3):
            a = f.plane(p)
            a[...] = np.clip(a.astype(int) + rng.integers(-(maxv // 3), maxv // 3 + 1, a.shape), 0, maxv)
        yy, xx = np.mgrid[0:24, 0:24]
        f.y[8:32, 8:32] = ((yy // 8 + xx // 8) % 2) * maxv
    org = f.copy()
    for p in range(3):
        org.plane(p)[...] = np.clip(f.plane(p).astype(int) + rng.integers(-7, 8, f.plane(p).shape), 0, maxv)
    return f, org


def blkinfo(seed, w, h, variant=None):
    """random_blkinfo with 128x128 roots and motion vectors within +-40.  With a variant, the first 64x64 filter block is one skipped block and the
    last has no skipped block (a frame of one filter block gets the first when variant is even, the second when it is odd)."""
    bi, dd = random_blkinfo(np.random.default_rng(seed), w, h, root=128, mv_range=40)
    if variant is None:
        return bi, dd
    nh = (w + 63) >> 6
    last = nfb64(w, h) - 1
    if last > 0 or variant % 2 == 0:
        cell = np.zeros((), BLKINFO)
        cell["size"] = 64
        bi[:16, :16] = cell
    if last > 0 or variant % 2 == 1:
        y0, x0 = (last // nh) * 16, (last % nh) * 16
        blk = bi[y0:y0 + 16, x0:x0 + 16]
        skip = blk["mode"] == 0
        blk["mode"][skip] = 2
        blk["cbp_y"][skip] = 1
    return bi, deblock_data(bi)


def allskip_of(bi, pw, ph, sub, fbl):
    """per filter block of side 2^fbl of a plane: every coded block skipped (common/common_frame.c:1042-1053, plane width as the grid pitch)"""
    bs, fb = (4 if sub else 8), 1 << fbl
    nh, nv = (pw + fb - 1) >> fbl, (ph + fb - 1) >> fbl
    flat = bi.reshape(-1)["mode"]
    out = np.ones(nh * nv, bool)
    for k in range(nv):
        for l in range(nh):
            for y in range(k * fb, min(ph, (k + 1) * fb), bs):
                for x in range(l * fb, min(pw, (l + 1) * fb), bs):
                    if flat[((y << sub) // 4) * (pw // 4) + ((x << sub) // 4)] != 0:
                        out[k * nh + l] = False
    return out


def fb_patterns(n, seed):
    """per-filter-block flags: all on, all off, a checkerboard, a seeded pattern"""
    rng = np.random.default_rng(seed)
    return {"on": np.ones(n, np.uint8), "off": np.zeros(n, np.uint8), "checker": (np.arange(n) % 2).astype(np.uint8),
            "seeded": rng.integers(0, 2, n).astype(np.uint8)}


def planes(f):
    return [f.plane(p).copy() for p in range(3)]


def assert_planes(got, want, what):
    for p in range(3):
        assert np.array_equal(got[p], want[p]), (what, "plane", p, int((got[p] != want[p]).sum()))


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# the expected values: impl "ref" (oracle/_ref) or "oracle"
# ---------------------------------------------------------------------------------------------------------------------------------------------------
def deblock_host(f, bi, dd, qp, impl):
    g = f.copy()
    s, w, h, bd = sfx(f.hbd), f.width, f.height, f.bitdepth
    if impl == "ref":
        getattr(R, "deblock_frame_y_" + s)(C.byref(g.s), dd, w, h, qp, bd)
        getattr(R, "deblock_frame_uv_" + s)(C.byref(g.s), dd, w, h, O.orc_chroma_qp(qp), bd)
    else:
        getattr(O, "orc_deblock_y_" + s)(P(g.Y, g.origin(0)), g.sy, P(bi), w, h, qp, bd)
        getattr(O, "orc_deblock_uv_" + s)(P(g.U, g.origin(1)), P(g.V, g.origin(1)), g.sc, P(bi), w, h, 1, O.orc_chroma_qp(qp), bd)
    return g


def cdef_host(f, bi, dd, pri, sec, pd, sd, impl):
    """all three planes in the encoder's order; pri/sec: int8 [2, nfb] (luma, chroma) level and sec_strength"""
    g = f.copy()
    s, w, h, bd = sfx(f.hbd), f.width, f.height, f.bitdepth
    nfb = nfb64(w, h)
    if impl == "ref":
        cst = (CdefStrengths * nfb)()
        for i in range(nfb):
            for c in range(2):
                st = cst[i].plane[c]
                st.level, st.sec_strength, st.pri_damping, st.sec_damping = int(pri[c, i]), int(sec[c, i]), pd, sd
        for plane in range(3):
            getattr(R, "cdef_frame_" + s)(cst, C.byref(g.s), None, dd, None, 0, bd, plane)
    else:
        dirs = np.zeros((nfb, 64), np.int32); vars_ = np.zeros((nfb, 64), np.int32)
        for plane in range(3):
            src = g.full(plane)
            dst = src.copy()
            c = int(plane > 0)
            getattr(O, "orc_cdef_plane_" + s)(P(src, g.origin(plane)), P(dst, g.origin(plane)), g.stride(plane), w, h, P(bi), w // 4, 1, plane, P(pri[c]), P(sec[c]),
                                              pd, sd, P(dirs), P(vars_), bd)
            src[...] = dst
    return g


def clpf_host(f, org, bi, dd, plane, fbl, strength, qp, fb_on, impl, asked=None):
    """one plane; fb_on: the luma filter-block flags or None.  asked collects the (k, l) the reference's decision callback was called for."""
    g = f.copy()
    s, w, h, bd = sfx(f.hbd), f.width, f.height, f.bitdepth
    flags = fb_on if plane == 0 else None
    if impl == "ref":
        if flags is not None:
            nh = (w + (1 << fbl) - 1) >> fbl

            def decide(k, l, *_):
                if asked is not None:
                    asked.append((k, l))
                return int(flags[k * nh + l])
            cb = DECISION(decide)
            getattr(R, "clpf_frame_" + s)(C.byref(g.s), C.byref(org.s), dd, None, 1, strength, fbl, bd, plane, qp, cb)
        else:
            getattr(R, "clpf_frame_" + s)(C.byref(g.s), C.byref(org.s), dd, None, 0, strength, fbl, bd, plane, qp, None)
    else:
        src = g.full(plane)
        dst = src.copy()
        pw, ph = (w, h) if plane == 0 else (w // 2, h // 2)
        getattr(O, "orc_clpf_plane_" + s)(P(src, g.origin(plane)), P(dst, g.origin(plane)), g.stride(plane), pw, ph, P(bi), w // 4, int(plane != 0),
                                          None if flags is None else P(flags), fbl, strength, bd, plane, qp)
        src[...] = dst
    return g


def detect_host(rec, org, bi, plane, qp, impl):
    """per 8x8 block of the plane, detect_multi_clpf's four sums with clpf_rdo's skip lookup (enc/encode_frame.c:563-576: luma width as the pitch)"""
    s, w, h, bd = sfx(rec.hbd), rec.width, rec.height, rec.bitdepth
    sub = int(plane != 0)
    pw, ph = w >> sub, h >> sub
    fn = getattr(R, "detect_multi_clpf_simd_" + s) if impl == "ref" else getattr(O, "orc_detect_multi_clpf_" + s)
    damping = bd - 4 - sub + (qp >> 4)
    flat = bi.reshape(-1)["mode"]
    nbx, nby = pw >> 3, ph >> 3
    out = np.zeros((nbx * nby, 4), np.int32)
    a, b = P(rec.full(plane), rec.origin(plane)), P(org.full(plane), org.origin(plane))
    for k in range(nbx * nby):
        x0, y0 = (k % nbx) * 8, (k // nbx) * 8
        if flat[((y0 << sub) // 4) * (w // 4) + ((x0 << sub) // 4)] != 0:
            m = (C.c_int * 4)(0, 0, 0, 0)
            fn(a, b, x0, y0, pw, ph, org.stride(plane), rec.stride(plane), m, bd - 8, 8, damping)
            out[k] = list(m)
    return out


def search_table(rec, org, bi, speed):
    """the oracle's cdef_search distortion table: (mse [2, nfb, 64], dirs, vars, allskip)"""
    s, w, h, bd = sfx(rec.hbd), rec.width, rec.height, rec.bitdepth
    nfb = nfb64(w, h)
    mse = np.zeros((2, nfb, 64), np.uint64); od = np.zeros((nfb, 64), np.int32); ov = np.zeros((nfb, 64), np.int32); ask = np.zeros(nfb, np.uint8)
    getattr(O, "orc_cdef_search_mse_" + s)(P(rec.Y, rec.origin(0)), P(rec.U, rec.origin(1)), P(rec.V, rec.origin(1)), P(org.Y, org.origin(0)), P(org.U, org.origin(1)),
                                            P(org.V, org.origin(1)), rec.sy, rec.sc, w, h, P(bi), speed, 5, bd, P(mse), P(od), P(ov), P(ask))
    return mse, od, ov, ask


SEARCH_LAMBDA, SEARCH_QP = 60.0, 34


def cdef_bits_of(speed):
    return 3 - speed if speed < 2 else 2


def select(mse, ask, speed):
    """orc_cdef_select on the filter blocks that are not all skip: (nb_strength_bits, level [2, nfb], sec [2, nfb]) with -1 for all-skip blocks"""
    live = np.flatnonzero(ask == 0)
    m0 = np.ascontiguousarray(mse[0][live]); m1 = np.ascontiguousarray(mse[1][live])
    st = (C.c_int * 16)(); ust = (C.c_int * 16)(); sel = (C.c_int * max(1, len(live)))()
    bits = O.orc_cdef_select(P(m0), P(m1), len(live), speed, cdef_bits_of(speed), C.c_double(SEARCH_LAMBDA), st, ust, sel)
    level = np.full((2, ask.size), -1); sec = np.full((2, ask.size), -1)
    for k, fb in enumerate(live):
        level[0, fb], sec[0, fb] = st[sel[k]] >> 2, st[sel[k]] & 3
        level[1, fb], sec[1, fb] = ust[sel[k]] >> 2, ust[sel[k]] & 3
    return bits, level, sec


def search_ref(rec, org, dd, speed):
    """the reference's cdef_search: (nb_strength_bits, level [2, nfb], sec [2, nfb]) with -1 for all-skip blocks, dirs, vars"""
    s, w, h, bd = sfx(rec.hbd), rec.width, rec.height, rec.bitdepth
    nfb = nfb64(w, h)
    st = (C.c_int * 8)(*[127] * 8); ust = (C.c_int * 8)(*[127] * 8)
    level = (C.c_int * (2 * nfb))(); sec = (C.c_int * (2 * nfb))(); dirs = (C.c_int * (64 * nfb))(); vars_ = (C.c_int * (64 * nfb))(); sbits = C.c_int(0)
    bits = getattr(ref_frame(rec.hbd), "ref_cdef_search_" + s)(C.byref(rec.s), C.byref(org.s), dd, w, h, bd, SEARCH_QP, C.c_double(SEARCH_LAMBDA),
                                                               cdef_bits_of(speed), speed, st, ust, level, sec, dirs, vars_, C.byref(sbits))
    return bits, np.array(level).reshape(nfb, 2).T.copy(), np.array(sec).reshape(nfb, 2).T.copy(), np.array(dirs).reshape(nfb, 64), np.array(vars_).reshape(nfb, 64)


def inside(w, h):
    """[nfb, 64] mask of the 8x8 luma blocks of each filter block that lie inside the frame"""
    nh, nv = (w + 63) >> 6, (h + 63) >> 6
    m = np.zeros((nh * nv, 64), bool)
    for fb in range(nh * nv):
        for k in range(64):
            m[fb, k] = (fb % nh) * 64 + (k % 8) * 8 < w and (fb // nh) * 64 + (k // 8) * 8 < h
    return m


def search_selection_want(rec, org, dd, mse, ask, speed, impl):
    """what cdef_search chooses: the reference's choice, or the oracle's table (mse, ask: search_table) through orc_cdef_select"""
    if impl == "ref":
        bits, level, sec, _, _ = search_ref(rec, org, dd, speed)
        level[:, ask != 0] = -1; sec[:, ask != 0] = -1
        return bits, level, sec
    return select(mse, ask, speed)


# ---- temporal interpolation
TI_ALL_PAIRS = [(r, p) for r in range(2, 17) for p in range(1, r)]
TI_ENC_PAIRS = sorted({(2, 1)} | {(r, 1) for r in range(2, 16)} | {(g, g - 1) for g in (4, 8, 16)})
TI_GEOMS = [(w, h, bds, TI_ALL_PAIRS if (w, h) in ((64, 64), (200, 136)) else TI_ENC_PAIRS) for w, h, bds in GEOMS] + [(128, 40, (8, 10), TI_ENC_PAIRS)]


def ti_levels(w, h):
    return min(4, int(math.log10(min(w, h)) / math.log10(2.0) - 4.0))  # common/temporal_interp.c:914


def ti_pair(seed, w, h, bd, hard):
    """two padded frames: the second is the first shifted by (1,-2) plus noise, with one displaced patch (the content of test_gpu_parity._ti_case,
    with the patch sized to the frame); hard=True adds enough noise that the skip test fails almost everywhere"""
    rng = np.random.default_rng(seed)
    hbd, maxv = hbd_of(bd), (1 << bd) - 1
    a = Frame(w, h, bd, hbd); a.randomize(rng)
    b = Frame(w, h, bd, hbd)
    amp = 14 if hard else 3
    for p in range(3):
        sh = (1, -2) if p == 0 else (0, -1)
        b.plane(p)[...] = np.clip(np.roll(a.plane(p).astype(int), sh, axis=(0, 1)) + rng.integers(-amp, amp + 1, a.plane(p).shape), 0, maxv)
    ph, pw = min(40, h // 2 - 8), min(56, w // 2 - 10)
    y0, x0 = h // 4, w // 3
    b.y[y0:y0 + ph, x0:x0 + pw] = np.clip(a.y[y0 + 6:y0 + 6 + ph, x0 - 9:x0 - 9 + pw].astype(int) + 20, 0, maxv)
    s = sfx(hbd)
    for f in (a, b):
        for p, (pw_, ph_, pad) in enumerate(((w, h, 160), (w // 2, h // 2, 80), (w // 2, h // 2, 80))):
            getattr(O, "orc_pad_plane_" + s)(P(f.full(p), f.origin(p)), f.stride(p), pw_, ph_, pad, pad)
    return a, b


def ti_host(a, b, ratio, pos, impl):
    w, h, bd, hbd = a.width, a.height, a.bitdepth, a.hbd
    s = sfx(hbd)
    o = Frame(w, h, bd, hbd)
    if impl == "ref":
        getattr(R, "interpolate_frames_" + s)(C.byref(o.s), C.byref(a.s), C.byref(b.s), ratio, pos)
    else:
        getattr(O, "orc_interpolate_frames_" + s)(P(o.Y, o.origin(0)), P(o.U, o.origin(1)), P(o.V, o.origin(1)), o.sy, o.sc, P(a.Y, a.origin(0)), P(a.U, a.origin(1)),
                                                 P(a.V, a.origin(1)), P(b.Y, b.origin(0)), P(b.U, b.origin(1)), P(b.V, b.origin(1)), a.sy, a.sc, w, h, 160, ratio, pos,
                                                 ti_levels(w, h))
    return planes(o)


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# the sub-cases of each stage, shared by the CPU pin and the GPU check
# ---------------------------------------------------------------------------------------------------------------------------------------------------
def deblock_cases(w, h, bd):
    qps = range(52) if (w, h) == (200, 136) else DEBLOCK_QPS
    for noisy in (False, True):
        f, _ = content(1000 + w + h + bd + noisy, w, h, bd, noisy)
        bi, dd = blkinfo(2000 + w + h + bd + noisy, w, h)
        for qp in qps:
            yield (noisy, qp), f, bi, dd, qp


def cdef_cases(w, h, bd):
    """per filter block (pri, sec) walks pri 0..15 and sec 0..3 over the four damping pairs"""
    nfb = nfb64(w, h)
    for noisy in (False, True):
        f, _ = content(3000 + w + h + bd + noisy, w, h, bd, noisy)
        bi, dd = blkinfo(4000 + w + h + bd + noisy, w, h, noisy)
        for r, (pd, sd) in enumerate(DAMPINGS):
            idx = r * nfb + np.arange(nfb) + 5 * noisy
            pri = np.stack([(idx * 7) % 16, (idx * 5 + 3) % 16]).astype(np.int8)
            sec = np.stack([idx % 4, (idx + 1) % 4]).astype(np.int8)
            yield (noisy, pd, sd), f, bi, dd, pri, sec, pd, sd


def clpf_cases(w, h, bd):
    """(label, plane, fbl, strength, qp, fb_on or None): without flags at every qp step; luma at every filter-block size with each flag pattern;
    chroma at 16 (flags passed, and ignored)"""
    i = 0
    for qp in QPS:
        for plane in range(3):
            yield ("noflags", plane, qp), plane, 6 if plane == 0 else 4, (1, 2, 4)[i % 3], qp, None
            i += 1
    for fbl in range(4, 8):
        n = ((w + (1 << fbl) - 1) >> fbl) * ((h + (1 << fbl) - 1) >> fbl)
        for name, flags in fb_patterns(n, 5000 + fbl + w).items():
            yield ("flags", fbl, name), 0, fbl, (1, 2, 4)[i % 3], QPS[i % 4], flags
            i += 1
    n16 = ((w + 15) >> 4) * ((h + 15) >> 4)
    for plane in (1, 2):
        yield ("chroma_flags", plane), plane, 4, (1, 2, 4)[i % 3], QPS[i % 4], fb_patterns(n16, 6000)["off"]
        i += 1


def clpf_frames(w, h, bd, variants=(False, True)):
    for noisy in variants:
        f, org = content(7000 + w + h + bd + noisy, w, h, bd, noisy)
        bi, dd = blkinfo(8000 + w + h + bd + noisy, w, h, noisy)
        yield noisy, f, org, bi, dd


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# CPU: the oracle against the reference on every case of the table
# ---------------------------------------------------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_oracle_equals_reference_deblock(case):
    changed = False
    for label, f, bi, dd, qp in deblock_cases(*case):
        a, b = deblock_host(f, bi, dd, qp, "oracle"), deblock_host(f, bi, dd, qp, "ref")
        assert_planes(planes(a), planes(b), label)
        changed |= any((a.plane(p) != f.plane(p)).any() for p in range(3))
    assert changed


@needs_ref
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_oracle_equals_reference_cdef(case):
    changed = False
    for label, f, bi, dd, pri, sec, pd, sd in cdef_cases(*case):
        a, b = cdef_host(f, bi, dd, pri, sec, pd, sd, "oracle"), cdef_host(f, bi, dd, pri, sec, pd, sd, "ref")
        assert_planes(planes(a), planes(b), label)
        changed |= (a.y != f.y).any()
    assert changed


@needs_ref
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_oracle_equals_reference_clpf(case):
    w, h, bd = case
    matters = 0
    for noisy, f, org, bi, dd in clpf_frames(w, h, bd):
        for label, plane, fbl, strength, qp, flags in clpf_cases(w, h, bd):
            asked = []
            a = clpf_host(f, org, bi, dd, plane, fbl, strength, qp, flags, "oracle")
            b = clpf_host(f, org, bi, dd, plane, fbl, strength, qp, flags, "ref", asked)
            assert np.array_equal(a.plane(plane), b.plane(plane)), (noisy, label)
            if plane == 0 and flags is not None:
                # the reference asks for exactly the filter blocks that are not all skip
                live = ~allskip_of(bi, w, h, 0, fbl)
                nh = (w + (1 << fbl) - 1) >> fbl
                assert sorted(k * nh + l for k, l in asked) == list(np.flatnonzero(live)), label
                matters += int((live & (flags == 0)).any())
    assert matters  # a filter block signalled off was not all skip: the flags changed what was filtered


@needs_ref
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_oracle_equals_reference_clpf_detect(case):
    w, h, bd = case
    nonzero = set()
    for noisy, f, org, bi, dd in clpf_frames(w, h, bd):
        for plane in range(3):
            for qp in QPS:
                a, b = detect_host(f, org, bi, plane, qp, "oracle"), detect_host(f, org, bi, plane, qp, "ref")
                assert np.array_equal(a, b), (noisy, plane, qp)
                if a.any():
                    nonzero.add(plane)
    assert nonzero == {0, 1, 2}


@needs_ref
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_oracle_equals_reference_cdef_search(case):
    """the oracle's table through orc_cdef_select chooses what the reference's cdef_search chooses, and finds the same directions and variances"""
    w, h, bd = case
    for noisy, f, org, bi, dd in clpf_frames(w, h, bd):
        for speed in range(3):
            bits, level, sec, rdirs, rvars = search_ref(f, org, dd, speed)
            mse, od, ov, ask = search_table(f, org, bi, speed)
            obits, olevel, osec = select(mse, ask, speed)
            live = ask == 0
            assert obits == bits, (noisy, speed)
            assert np.array_equal(olevel[:, live], level[:, live]) and np.array_equal(osec[:, live], sec[:, live]), (noisy, speed)
            m = inside(w, h) & live[:, None]
            assert np.array_equal(od[m], rdirs[m]) and np.array_equal(ov[m], rvars[m])


@needs_ref
@pytest.mark.parametrize("geom", TI_GEOMS, ids=["%dx%d" % g[:2] for g in TI_GEOMS])
def test_oracle_equals_reference_interpolation(geom):
    w, h, bds, pairs = geom
    for bd in bds:
        for hard in (False, True):
            a, b = ti_pair(9000 + w + h + bd + hard, w, h, bd, hard)
            for ratio, pos in pairs:
                assert_planes(ti_host(a, b, ratio, pos, "oracle"), ti_host(a, b, ratio, pos, "ref"), (bd, hard, ratio, pos))


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: the device against the expected value
# ---------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tb():
    import thor_b200 as t
    t.init(0)
    return t


def dev_frame(tb, f, pad=32):
    d = tb.Frame(f.width, f.height, 2 if f.hbd else 1, pad)
    d.upload(f.y, f.u, f.v)
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_deblock_matrix(tb, case):
    changed = False
    for label, f, bi, dd, qp in deblock_cases(*case):
        d, dbi = dev_frame(tb, f), tb.DevBuf.from_array(bi)
        tb.check(tb.lib.tb_deblock_frame(d.h, dbi.ptr, qp, case[2]))
        want = planes(deblock_host(f, bi, dd, qp, EXPECT))
        assert_planes(d.download(), want, label)
        changed |= any((want[p] != f.plane(p)).any() for p in range(3))
    assert changed


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_cdef_matrix(tb, case):
    w, h, bd = case
    nfb = nfb64(w, h)
    ddv = tb.DevBuf(nfb * 2 * 64 * 4)
    for label, f, bi, dd, pri, sec, pd, sd in cdef_cases(w, h, bd):
        d, scr, dbi = dev_frame(tb, f), tb.Frame(w, h, 2 if f.hbd else 1, 32), tb.DevBuf.from_array(bi)
        dpri = [tb.DevBuf.from_array(pri[c]) for c in range(2)]; dsec = [tb.DevBuf.from_array(sec[c]) for c in range(2)]
        for plane in range(3):
            c = int(plane > 0)
            tb.check(tb.lib.tb_cdef_frame(d.h, scr.h, dbi.ptr, dpri[c].ptr, dsec[c].ptr, pd, sd, ddv.ptr, bd, plane))
        assert_planes(d.download(), planes(cdef_host(f, bi, dd, pri, sec, pd, sd, EXPECT)), label)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_clpf_matrix(tb, case):
    w, h, bd = case
    esz = 2 if bd > 8 else 1
    for noisy, f, org, bi, dd in clpf_frames(w, h, bd):
        dbi = tb.DevBuf.from_array(bi)
        scr = tb.Frame(w, h, esz, 32)
        for label, plane, fbl, strength, qp, flags in clpf_cases(w, h, bd):
            d = dev_frame(tb, f)
            dfl = None if flags is None else tb.DevBuf.from_array(flags)
            tb.check(tb.lib.tb_clpf_frame(d.h, scr.h, dbi.ptr, None if dfl is None else dfl.ptr, fbl, strength, bd, plane, qp))
            want = clpf_host(f, org, bi, dd, plane, fbl, strength, qp, flags, EXPECT)
            assert_planes(d.download(), planes(want), (noisy, label))
        # all three planes in one call: luma at the given size with the flags, chroma at 16 without them
        for fbl in range(4, 8):
            n = ((w + (1 << fbl) - 1) >> fbl) * ((h + (1 << fbl) - 1) >> fbl)
            flags = fb_patterns(n, 5100 + fbl)["seeded"]
            strength, qp = (1, 2, 4)[fbl % 3], QPS[fbl % 4]
            d, dfl = dev_frame(tb, f), tb.DevBuf.from_array(flags)
            tb.check(tb.lib.tb_clpf_frame(d.h, scr.h, dbi.ptr, dfl.ptr, fbl, strength, bd, -1, qp))
            g = f
            for plane in range(3):
                g = clpf_host(g, org, bi, dd, plane, fbl if plane == 0 else 4, strength, qp, flags, EXPECT)
            assert_planes(d.download(), planes(g), (noisy, "plane -1", fbl))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_clpf_detect_matrix(tb, case):
    w, h, bd = case
    for noisy, f, org, bi, dd in clpf_frames(w, h, bd):
        d, dorg, dbi = dev_frame(tb, f), dev_frame(tb, org), tb.DevBuf.from_array(bi)
        for plane in range(3):
            sub = int(plane != 0)
            nb = ((w >> sub) >> 3) * ((h >> sub) >> 3)
            dsum = tb.DevBuf(16 * nb)
            for qp in QPS:
                tb.check(tb.lib.tb_clpf_detect_frame(d.h, dorg.h, dbi.ptr, plane, bd, qp, dsum.ptr))
                want = detect_host(f, org, bi, plane, qp, EXPECT)
                got = dsum.download(np.int32, (nb, 4))
                assert np.array_equal(got, want), (noisy, plane, qp, int((got != want).any(axis=1).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_cdef_search_matrix(tb, case):
    w, h, bd = case
    nfb = nfb64(w, h)
    m_in = inside(w, h)
    # at 1080p the expected tables take most of the time (on the host): the smooth content only
    for noisy, f, org, bi, dd in clpf_frames(w, h, bd, (False,) if w * h > 1 << 20 else (False, True)):
        d, dorg, dbi = dev_frame(tb, f), dev_frame(tb, org), tb.DevBuf.from_array(bi)
        ddv = tb.DevBuf(nfb * 2 * 64 * 4); dsk = tb.DevBuf(max(nfb, 16)); dmse = tb.DevBuf(2 * nfb * 64 * 8)
        for speed in range(3):
            check_search(tb, d, dorg, dbi, ddv, dsk, dmse, f, org, bi, dd, speed, m_in, (noisy, speed))


def check_search(tb, d, dorg, dbi, ddv, dsk, dmse, f, org, bi, dd, speed, m_in, label):
    """tb_cdef_search_mse against the oracle's table (the chroma entries of the documented quirk masked where luma width = 8 mod 16, see
    test_gpu_parity.test_cdef_search_mse); where it does not apply, the device's table through orc_cdef_select must choose what cdef_search chooses"""
    w, h, bd = f.width, f.height, f.bitdepth
    nfb = nfb64(w, h)
    tb.check(tb.lib.tb_cdef_search_mse(d.h, dorg.h, dbi.ptr, speed, 5, bd, ddv.ptr, dsk.ptr, dmse.ptr))
    got = dmse.download(np.uint64, (2, nfb, 64)); gsk = dsk.download(np.uint8, (max(nfb, 16),))[:nfb]
    dv = ddv.download(np.int32, (nfb, 2, 64))
    mse, od, ov, ask = search_table(f, org, bi, speed)
    assert np.array_equal(gsk, ask), label
    live = ask == 0
    m = m_in & live[:, None]
    assert np.array_equal(dv[:, 0][m], od[m]) and np.array_equal(dv[:, 1][m], ov[m]), label
    if (w >> 1) & 7:
        nh = (w + 63) // 64
        got[1, nh - 1::nh] = 0; mse[1, nh - 1::nh] = 0
    assert np.array_equal(got, mse), (label, int((got != mse).sum()))
    if live.any():
        assert mse.any()
    if not (w >> 1) & 7:
        bits, level, sec = select(got, gsk, speed)
        wbits, wlevel, wsec = search_selection_want(f, org, dd, mse, ask, speed, EXPECT)
        assert (bits, level.tolist(), sec.tolist()) == (wbits, wlevel.tolist(), wsec.tolist()), label


def ti_schedule():
    """every (geometry, bit depth, hard, ratio, pos) of TI_GEOMS in chunks of 8 calls, visited round robin over (geometry, bit depth): consecutive
    chunks differ in geometry or sample size, so the device rebuilds its cached pyramid and vector fields between chunks and reuses them within one"""
    queues = []
    for w, h, bds, pairs in TI_GEOMS:
        for bd in bds:
            items = [(hard, r, p) for hard in (False, True) for r, p in pairs]
            queues.append(((w, h, bd), [items[i:i + 8] for i in range(0, len(items), 8)]))
    order = []
    for c in range(max(len(q) for _, q in queues)):
        for key, chunks in queues:
            if c < len(chunks):
                order.append((key, chunks[c]))
    return order


@pytest.mark.gpu
def test_interpolation_interleaved(tb):
    sched = ti_schedule()
    assert all(a[0] != b[0] for a, b in zip(sched, sched[1:]))
    assert ti_levels(128, 40) == 1 and ti_levels(424, 264) == 4
    frames, n = {}, 0
    for (w, h, bd), chunk in sched:
        esz = 2 if bd > 8 else 1
        for hard, ratio, pos in chunk:
            key = (w, h, bd, hard)
            if key not in frames:
                a, b = ti_pair(9000 + w + h + bd + hard, w, h, bd, hard)
                dev = []
                for f in (a, b):
                    t = tb.Frame(w, h, esz); t.upload(f.y, f.u, f.v)
                    r = tb.Frame(w, h, esz)
                    tb.check(tb.lib.tb_create_reference_frame(r.h, t.h))
                    dev.append(r)
                frames[key] = (a, b, dev, tb.Frame(w, h, esz))
            a, b, dev, out = frames[key]
            tb.check(tb.lib.tb_interpolate_frames(out.h, dev[0].h, dev[1].h, ratio, pos))
            assert_planes(out.download(), ti_host(a, b, ratio, pos, EXPECT), (w, h, bd, hard, ratio, pos))
            n += 1
    assert n == sum(len(bds) * 2 * len(pairs) for _, _, bds, pairs in TI_GEOMS)


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: the filter chain on the reference encoder's own pre-filter reconstruction and block state
# ---------------------------------------------------------------------------------------------------------------------------------------------------
def rdo_blkinfo(job):
    """the RD-loop job's per-4x4 block state (RDO_BLK) as tb_blkinfo_t and DeblockData: mode; cbp_y != 0; size, tb_split and pb_part; mv0 and mv1"""
    w, h = job.hdr.width, job.hdr.height
    blk = job.blk
    bi = np.zeros(blk.size, BLKINFO)
    for name in ("mode", "size", "tb_split", "pb_part", "mv0x", "mv0y", "mv1x", "mv1y"):
        bi[name] = blk[name]
    bi["cbp_y"] = blk["cbp_y"] != 0
    bi = bi.reshape(h // 4, w // 4)
    return bi, deblock_data(bi)


def job_frames(job):
    """(pre-filter reconstruction, original) of one job as padded host frames"""
    w, h, bd = job.hdr.width, job.hdr.height, job.hdr.bitdepth
    rec, org = Frame(w, h, bd, hbd_of(bd), 32, 32), Frame(w, h, bd, hbd_of(bd), 32, 32)
    for p in range(3):
        rec.plane(p)[...] = job.rec[p]
        org.plane(p)[...] = job.orig[p]
    return rec, org


def run_chain(tb, jobs, seed):
    """every frame at its own qp, in the encoder's order: deblocking; the CDEF search table and selection on the deblocked frame; CDEF with seeded
    strengths; the CLPF detection sums on the CDEF output; CLPF on all planes with seeded luma flags.  Each stage's output is compared."""
    rng = np.random.default_rng(seed)
    stages = {"deblock": 0, "cdef": 0, "clpf": 0}
    for job in jobs:
        w, h, bd, qp = job.hdr.width, job.hdr.height, job.hdr.bitdepth, job.hdr.qp
        esz, nfb = 2 if bd > 8 else 1, nfb64(w, h)
        label = (w, h, bd, job.frame_num, qp)
        bi, dd = rdo_blkinfo(job)
        f, org = job_frames(job)
        d, dorg, scr, dbi = dev_frame(tb, f), dev_frame(tb, org), tb.Frame(w, h, esz, 32), tb.DevBuf.from_array(bi)
        # 1. deblocking
        tb.check(tb.lib.tb_deblock_frame(d.h, dbi.ptr, qp, bd))
        g = deblock_host(f, bi, dd, qp, EXPECT)
        assert_planes(d.download(), planes(g), ("deblock",) + label)
        stages["deblock"] += any((g.plane(p) != f.plane(p)).any() for p in range(3))
        # 5. the CDEF search on the deblocked frame
        ddv = tb.DevBuf(nfb * 2 * 64 * 4); dsk = tb.DevBuf(max(nfb, 16)); dmse = tb.DevBuf(2 * nfb * 64 * 8)
        check_search(tb, d, dorg, dbi, ddv, dsk, dmse, g, org, bi, dd, int(rng.integers(0, 3)), inside(w, h), ("cdef search",) + label)
        # 2. CDEF with seeded strengths
        pri = rng.integers(0, 16, (2, nfb)).astype(np.int8); sec = rng.integers(0, 4, (2, nfb)).astype(np.int8)
        dpri = [tb.DevBuf.from_array(pri[c]) for c in range(2)]; dsec = [tb.DevBuf.from_array(sec[c]) for c in range(2)]
        for plane in range(3):
            c = int(plane > 0)
            tb.check(tb.lib.tb_cdef_frame(d.h, scr.h, dbi.ptr, dpri[c].ptr, dsec[c].ptr, 5, 5, ddv.ptr, bd, plane))
        g2 = cdef_host(g, bi, dd, pri, sec, 5, 5, EXPECT)
        assert_planes(d.download(), planes(g2), ("cdef",) + label)
        stages["cdef"] += (g2.y != g.y).any()
        # 4. detection sums on the CDEF output
        for plane in range(3):
            sub = int(plane != 0)
            nb = ((w >> sub) >> 3) * ((h >> sub) >> 3)
            dsum = tb.DevBuf(16 * nb)
            tb.check(tb.lib.tb_clpf_detect_frame(d.h, dorg.h, dbi.ptr, plane, bd, qp, dsum.ptr))
            assert np.array_equal(dsum.download(np.int32, (nb, 4)), detect_host(g2, org, bi, plane, qp, EXPECT)), ("detect", plane) + label
        # 3. CLPF with seeded luma flags
        fbl = int(rng.integers(4, 8)); strength = int(rng.choice([1, 2, 4]))
        n = ((w + (1 << fbl) - 1) >> fbl) * ((h + (1 << fbl) - 1) >> fbl)
        flags = rng.integers(0, 2, n).astype(np.uint8)
        dfl = tb.DevBuf.from_array(flags)
        tb.check(tb.lib.tb_clpf_frame(d.h, scr.h, dbi.ptr, dfl.ptr, fbl, strength, bd, -1, qp))
        g3 = g2
        for plane in range(3):
            g3 = clpf_host(g3, org, bi, dd, plane, fbl if plane == 0 else 4, strength, qp, flags, EXPECT)
        assert_planes(d.download(), planes(g3), ("clpf", fbl, strength) + label)
        stages["clpf"] += (g3.y != g2.y).any()
    if all(j.hdr.qp < 16 for j in jobs):
        del stages["deblock"]   # beta is 0 below qp 16: deblocking may leave every frame unchanged
    assert all(stages.values()), stages   # every stage changed some frame: the comparisons are not vacuous


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["hdb_128x136", "hdb_hard_q4_10bit"])
def test_filter_chain_on_golden_rdo_jobs(tb, tmp_path, case):
    from test_rdo_jobs import golden_jobs
    from thor_b200 import rdo_jobs as RJ
    golden_jobs(str(tmp_path), case)
    run_chain(tb, RJ.load_jobs(str(tmp_path)), 11)


@pytest.mark.gpu
@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref not built")
@pytest.mark.parametrize("name", ["speed1_hard_rect", "ldb_q45_hard"])
def test_filter_chain_on_captured_matrix_cases(tb, tmp_path, name):
    """real block state at widths that are not multiples of 64 (200x72, 256x136 with 128x128 super blocks)"""
    from test_rdo_jobs import capture
    from test_rdo_matrix import BY_NAME, CONTENT
    from thor_b200 import rdo_jobs as RJ
    _, flags, w, h, n, qp, bd, content_ = BY_NAME[name]
    run_chain(tb, RJ.load_jobs(capture(str(tmp_path), flags, w, h, n, bd, qp, CONTENT[content_])), 12)
