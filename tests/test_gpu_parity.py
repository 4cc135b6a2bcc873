"""GPU parity: every CUDA path of libthor_b200.so, called through its C ABI, against the plain-C oracle on the same
seeded inputs (bit-exact).  Where oracle/_ref travelled to the box, the compiled reference is checked too."""
import ctypes as C
import numpy as np
import pytest

from _libs import oracle, ref, aligned, P, sdt, sfx, rand_plane, full_scale_planes, edge_search, edge_reach
from _refstructs import Frame as HFrame, random_blkinfo

pytestmark = pytest.mark.gpu
O = oracle()
BD = [(0, 8), (1, 8), (1, 10), (1, 12)]  # (1, 8): 8-bit content in 16-bit frames (-frame_bitdepth 16)


@pytest.fixture(scope="module")
def tb():
    import thor_b200 as t
    t.init(0)
    return t


def dptr(a):
    return C.c_void_p(a.ctypes.data)


# ------------------------------------------------------------------------------------------------------------------
# (A) drop-in symbols
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hbd,bd", BD)
def test_dropin_sad_family(tb, hbd, bd):
    rng = np.random.default_rng(101)
    s = sfx(hbd)
    L = tb.lib
    for smooth in (False, True):
        refp = rand_plane(rng, 200, 256, bd, hbd, smooth)
        for (w, h) in [(8, 8), (8, 4), (16, 16), (16, 8), (32, 32), (64, 64), (128, 128), (64, 32), (16, 32)]:
            size = max(w, h)
            org = aligned((size, size), sdt(hbd))
            oy, ox = int(rng.integers(8, 60)), int(rng.integers(8, 100))
            org[...] = refp[oy:oy + size, ox:ox + size] if smooth else rng.integers(0, 1 << bd, (size, size))
            for _ in range(2):
                y, x = oy + int(rng.integers(-3, 4)), ox + int(rng.integers(-3, 4))
                b = P(refp, y * 256 + x)
                assert getattr(L, "sad_calc_simd_" + s)(P(org), b, size, 256, w, h) == getattr(O, "orc_sad_" + s)(P(org), b, size, 256, w, h)
                assert getattr(L, "sad_calc_simd_unaligned_" + s)(P(refp, (y + 1) * 256 + x + 1), b, 256, 256, w, h) == \
                    getattr(O, "orc_sad_" + s)(P(refp, (y + 1) * 256 + x + 1), b, 256, 256, w, h)
                if w == h:
                    assert getattr(L, "ssd_calc_simd_" + s)(P(org), b, size, 256, w) == getattr(O, "orc_ssd_" + s)(P(org), b, size, 256, w, h)
                x0, x1 = C.c_int(9), C.c_int(9)
                assert getattr(L, "widesad_calc_simd_" + s)(P(org), b, size, 256, w, h, C.byref(x0)) == \
                    getattr(O, "orc_widesad_" + s)(P(org), b, size, 256, w, h, C.byref(x1))
                assert x0.value == x1.value
                xs = [C.c_int(0) for _ in range(4)]
                got = getattr(L, "sad_calc_fasthalf_simd_" + s)(P(org), b, size, 256, w, h, C.byref(xs[0]), C.byref(xs[1]))
                want = getattr(O, "orc_sad_fasthalf_" + s)(P(org), b, size, 256, w, h, C.byref(xs[2]), C.byref(xs[3]))
                assert (got, xs[0].value, xs[1].value) == (want, xs[2].value, xs[3].value)
                for (fx, fy) in [(0, 0), (2, 0), (0, -2), (-2, 2)]:
                    xs = [C.c_int(fx if i % 2 == 0 else fy) for i in range(4)]
                    got = getattr(L, "sad_calc_fastquarter_simd_" + s)(P(org), b, size, 256, w, h, C.byref(xs[0]), C.byref(xs[1]))
                    want = getattr(O, "orc_sad_fastquarter_" + s)(P(org), b, size, 256, w, h, C.byref(xs[2]), C.byref(xs[3]))
                    assert (got, xs[0].value, xs[1].value) == (want, xs[2].value, xs[3].value)


@pytest.mark.parametrize("hbd,bd", BD)
def test_dropin_interp_avg(tb, hbd, bd):
    rng = np.random.default_rng(102)
    s = sfx(hbd)
    L = tb.lib
    refp = rand_plane(rng, 200, 256, bd, hbd)
    for (w, h) in [(4, 4), (8, 8), (4, 8), (16, 16), (32, 32), (64, 64), (128, 128), (16, 8)]:
        for bip in (0, 1, 2):
            for (xo, yo) in [(1, 0), (0, 3), (2, 2), (1, 3), (3, 1), (2, 0), (2, 1)]:
                y, x = int(rng.integers(8, 40)), int(rng.integers(8, 60))
                a = aligned((h, w + 8), sdt(hbd), fill=7); b = aligned((h, w + 8), sdt(hbd), fill=7)
                getattr(O, "orc_interp_luma_" + s)(w, h, xo, yo, P(a), w + 8, P(refp, y * 256 + x), 256, bip, bd)
                getattr(L, "get_inter_prediction_luma_simd_" + s)(w, h, xo, yo, P(b), w + 8, P(refp, y * 256 + x), 256, bip, bd)
                assert (a == b).all(), (w, h, bip, xo, yo)
    for (w, h) in [(4, 4), (8, 8), (2, 2), (16, 16), (64, 64), (8, 4)]:
        for (xo, yo) in [(1, 0), (0, 5), (4, 4), (7, 3), (2, 6)]:
            y, x = int(rng.integers(8, 40)), int(rng.integers(8, 60))
            a = aligned((h, w), sdt(hbd)); b = aligned((h, w), sdt(hbd))
            getattr(O, "orc_interp_chroma_" + s)(w, h, xo, yo, P(a), w, P(refp, y * 256 + x), 256, bd)
            getattr(L, "get_inter_prediction_chroma_simd_" + s)(w, h, xo, yo, P(b), w, P(refp, y * 256 + x), 256, bd)
            assert (a == b).all()
    for size in (4, 8, 16, 64):
        p0 = rand_plane(rng, size, size + 16, bd, hbd); p1 = rand_plane(rng, size, size + 16, bd, hbd)
        o0 = aligned((size, size + 16), sdt(hbd), fill=0); o1 = aligned((size, size + 16), sdt(hbd), fill=0)
        getattr(O, "orc_block_avg_" + s)(P(o0), P(p0), P(p1), size + 16, size + 16, size + 16, size, size)
        getattr(L, "block_avg_simd_" + s)(P(o1), P(p0), P(p1), size + 16, size + 16, size + 16, size, size)
        assert (o0 == o1).all()


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_dropin_transform_quant(tb, bd):
    rng = np.random.default_rng(103)
    L = tb.lib
    lim = (1 << bd) - 1
    for size in (4, 8, 16, 32, 64, 128):
        q = min(size, 16)
        coefs = []
        for fast in (0, 1):
            for amp in (lim, 25, 3):
                blk = aligned((size, size), np.int16)
                blk[...] = rng.integers(-amp, amp + 1, (size, size))
                c0 = aligned((size, size), np.int16, fill=0); c1 = aligned((size, size), np.int16, fill=0)
                O.orc_transform(P(blk), P(c0), size, fast, bd)
                L.transform_simd(P(blk), P(c1), size, fast, bd)
                assert (c0[:q, :q] == c1[:q, :q]).all(), (size, fast, amp)
                coefs.append((c0, (fast, amp)))
        # coefficients of magnitude 32768 (and 32767): the bound the quantiser's and dequantiser's 32-bit arithmetic relies on
        edge = aligned((size, size), np.int16, fill=0)
        edge[:q, :q] = rng.choice(np.array([-32768, 32767], np.int16), (q, q))
        coefs.append((edge, "edge"))
        for c0, what in coefs:
            for qp in range(52):
                for typ in range(4):
                    q0 = aligned((q * q,), np.int16, fill=0); q1 = aligned((q * q,), np.int16, fill=0)
                    cb0 = O.orc_quantize(P(c0), P(q0), qp, size, typ, None)
                    cb1 = L.tb_quantize(P(c0), P(q1), qp, size, typ)
                    assert cb0 == cb1 and (q0 == q1).all(), (size, qp, typ, what)
                r0 = aligned((size, size), np.int16, fill=0); r1 = aligned((size, size), np.int16, fill=0)
                O.orc_dequantize(P(q0), P(r0), qp, size, None)
                L.tb_dequantize(P(q1), P(r1), qp, size)
                assert (r0 == r1).all(), (size, qp, what)
                if size <= 32:
                    assert O.orc_check_nz_area(P(r0), size) == L.check_nz_area(P(r0), size)
                b0 = aligned((size, size), np.int16, fill=0); b1 = aligned((size, size), np.int16, fill=0)
                O.orc_inverse_transform(P(r0), P(b0), size, bd)
                if size < 64:  # the reference routes 64/128 through inverse_transform() in transform.c (32x32 kernel + replication)
                    L.inverse_transform_simd(P(r0), P(b1), size, bd)
                    assert (b0 == b1).all(), (size, qp, what)
        # the edge block itself as levels: the dequantiser's largest products and shifts
        lv = np.ascontiguousarray(edge[:q, :q]).reshape(-1)
        for qp in range(52):
            r0 = aligned((size, size), np.int16, fill=0); r1 = aligned((size, size), np.int16, fill=0)
            O.orc_dequantize(P(lv), P(r0), qp, size, None)
            L.tb_dequantize(P(lv), P(r1), qp, size)
            assert (r0 == r1).all(), (size, qp, "edge levels")
        assert L.tb_quantize(P(edge), P(q1), 52, size, 0) == tb.TB_ERR_ARG
    for size in (4, 8, 16):
        for _ in range(60):
            blk = aligned((size, size), np.int16)
            blk[...] = rng.integers(-int(rng.choice([2, 6, 40])), 41, (size, size))
            thr = int(rng.integers(1, 60))
            assert O.orc_calc_cbp(P(blk), size, thr) == L.calc_cbp_simd(P(blk), size, thr)


@pytest.mark.parametrize("hbd,bd", BD)
def test_dropin_filters(tb, hbd, bd):
    rng = np.random.default_rng(104)
    s = sfx(hbd)
    L = tb.lib
    w, h = 200, 136
    f = HFrame(w, h, bd, hbd, 32, 32)
    f.randomize(rng)
    org = f.copy()
    org.y[...] = np.clip(f.y.astype(int) + rng.integers(-6, 7, f.y.shape), 0, (1 << bd) - 1)
    for (sx, sy) in [(8, 8), (4, 4), (8, 4)]:
        for bt in (0, 1, 2, 4, 8, 5, 10, 15):
            x0, y0 = 8 * int(rng.integers(1, 10)), 8 * int(rng.integers(1, 8))
            d0 = aligned((h, w), sdt(hbd), fill=0); d1 = aligned((h, w), sdt(hbd), fill=0)
            st, dmp = 2 << (bd - 8), bd - 4 + 2
            getattr(O, "orc_clpf_block_" + s)(P(f.Y, f.origin(0)), P(d0), f.sy, w, x0, y0, sx, sy, bt, st, dmp)
            if bt:
                getattr(L, "clpf_block%d_%s" % (sx, s))(P(f.Y, f.origin(0)), P(d1), f.sy, w, x0, y0, sy, bt, st, dmp)
            else:
                getattr(L, "clpf_block%d_noclip_%s" % (sx, s))(P(f.Y, f.origin(0)), P(d1), f.sy, w, x0, y0, sy, st, dmp)
            assert (d0 == d1).all(), (sx, sy, bt)
    for _ in range(25):
        x0, y0 = 8 * int(rng.integers(0, w // 8)), 8 * int(rng.integers(0, h // 8))
        strength = int(rng.choice([1, 2, 4])) << (bd - 8)
        a = (C.c_int * 2)(0, 0); c = (C.c_int * 2)(3, 4)
        args = (P(f.Y, f.origin(0)), P(org.Y, org.origin(0)), x0, y0, w, h, org.sy, f.sy)
        getattr(O, "orc_detect_clpf_" + s)(*args, C.byref(a, 0), C.byref(a, 4), strength, bd - 8, 8, bd - 4 + 2)
        getattr(L, "detect_clpf_simd_" + s)(*args, C.byref(c, 0), C.byref(c, 4), strength, bd - 8, 8, bd - 4 + 2)
        assert [c[0], c[1]] == [3 + 2 * a[0], 4 + 2 * a[1]]
        m0 = (C.c_int * 4)(1, 2, 3, 4); m1 = (C.c_int * 4)(1, 2, 3, 4)
        getattr(O, "orc_detect_multi_clpf_" + s)(*args, m0, bd - 8, 8, bd - 4 + 2)
        getattr(L, "detect_multi_clpf_simd_" + s)(*args, m1, bd - 8, 8, bd - 4 + 2)
        assert list(m0) == list(m1)
        v0, v1 = C.c_int32(0), C.c_int32(0)
        p = P(f.Y, f.origin(0) + y0 * f.sy + x0)
        assert getattr(O, "orc_cdef_find_dir_" + s)(p, f.sy, C.byref(v0), bd - 8) == getattr(L, "cdef_find_dir_simd_" + s)(p, f.sy, C.byref(v1), bd - 8)
        assert v0.value == v1.value
    cs = bd - 8
    dirs = np.zeros((8, 2), np.int32)
    for trial in range(40):
        bs = int(rng.choice([4, 8]))
        plane = 0 if bs == 8 else 1
        pw, ph = (w, h) if plane == 0 else (w // 2, h // 2)
        x0, y0 = bs * int(rng.integers(0, pw // bs)), bs * int(rng.integers(0, ph // bs))
        bt = (1 if x0 == 0 else 0) | (4 if y0 == 0 else 0) | (2 if x0 == pw - bs else 0) | (8 if y0 == ph - bs else 0)
        t0 = aligned((12, 32), np.uint16, fill=0)
        getattr(O, "orc_cdef_prepare_input_" + s)(bs, bs, x0, y0, bt, 2, P(t0, 2 * 32 + 16), 32, P(f.full(plane), f.origin(plane)), f.stride(plane))
        pri = int(rng.integers(0, 16)) << cs; sec = int(rng.choice([0, 1, 2, 4])) << cs
        d = int(rng.integers(0, 8))
        pd = max(int(np.log2(pri >> cs)) if pri >> cs else 0, 5 - plane) + cs; sd = 5 - plane + cs
        o0 = aligned((bs, bs), sdt(hbd), fill=0); o1 = aligned((bs, bs), sdt(hbd), fill=0)
        dp = lambda o: (P(o), None) if not hbd else (None, P(o))
        O.orc_cdef_filter_block(*dp(o0), bs, P(t0, 2 * 32 + 16), 32, pri, sec, d, pd, sd, bs, cs)
        L.cdef_filter_block_simd(*dp(o1), bs, P(t0, 2 * 32 + 16), 32, pri, sec, d, pd, sd, bs, P(dirs), cs)
        assert (o0 == o1).all(), (bs, pri, sec, d, bt)


@pytest.mark.parametrize("hbd,bd", BD)
def test_cfl(tb, hbd, bd):
    rng = np.random.default_rng(105)
    s = sfx(hbd)
    hit = 0
    ns = 1 << max(0, bd - 10)  # noise grows with the remap threshold above 10 bits (tests/test_oracle_vs_ref.py::test_cfl)
    for n in (8, 16, 32, 64):
        for trial in range(12):
            y = rand_plane(rng, n, n, bd, hbd, smooth=True)
            ry = aligned((n, n + 8), sdt(hbd))
            ry[...] = np.clip(np.pad(y.astype(int), ((0, 0), (0, 8)), mode="edge") + rng.integers(-40, 41, (n, n + 8)) * (trial % 3) * ns, 0, (1 << bd) - 1)
            k = float(rng.uniform(-1.5, 1.5))
            ys = y.astype(int).reshape(n // 2, 2, n // 2, 2).sum(axis=(1, 3)) // 4
            u0 = aligned((n // 2, n // 2), sdt(hbd)); v0 = aligned((n // 2, n // 2), sdt(hbd))
            u0[...] = np.clip(ys * k + (1 << (bd - 1)) * (1 - k) + rng.integers(-3, 4, ys.shape) * ns, 0, (1 << bd) - 1)
            v0[...] = np.clip(ys * -k + (1 << (bd - 1)) * (1 + k) + rng.integers(-30, 31, ys.shape) * ns, 0, (1 << bd) - 1)
            u1 = aligned(u0.shape, sdt(hbd)); u1[...] = u0; v1 = aligned(v0.shape, sdt(hbd)); v1[...] = v0
            ub = u0.copy()
            getattr(O, "orc_cfl_" + s)(P(y), P(u0), P(v0), P(ry), n, n, n + 8, 1, bd)
            tb.lib.tb_improve_uv_prediction(2 if hbd else 1, P(y), P(u1), P(v1), P(ry), n, n, n + 8, 1, bd)
            assert (u0 == u1).all() and (v0 == v1).all()
            hit += int((ub != u0).any())
    assert hit > 5


# ------------------------------------------------------------------------------------------------------------------
# (B) batched entry points on resident frames
# ------------------------------------------------------------------------------------------------------------------
def make_frames(tb, rng, w, h, bd, hbd, shift=(2, -3)):
    """host reference frame (padded by the oracle) + current frame, and their device twins (reference padded on the GPU)"""
    s = sfx(hbd)
    href = HFrame(w, h, bd, hbd)
    href.randomize(rng)
    cur = HFrame(w, h, bd, hbd)
    cur.y[...] = np.clip(np.roll(href.y.astype(int), shift, axis=(0, 1)) + rng.integers(-4, 5, href.y.shape), 0, (1 << bd) - 1)
    cur.u[...] = href.u; cur.v[...] = href.v
    esz = 2 if hbd else 1
    drec = tb.Frame(w, h, esz); dref = tb.Frame(w, h, esz); dcur = tb.Frame(w, h, esz)
    drec.upload(href.y, href.u, href.v)
    tb.check(tb.lib.tb_create_reference_frame(dref.h, drec.h))
    dcur.upload(cur.y, cur.u, cur.v)
    for p, (pw, ph, padh) in enumerate(((w, h, 160), (w // 2, h // 2, 80), (w // 2, h // 2, 80))):
        getattr(O, "orc_pad_plane_" + s)(P(href.full(p), href.origin(p)), href.stride(p), pw, ph, padh, padh)
    return href, cur, dref, dcur, drec


@pytest.mark.parametrize("hbd,bd", BD)
def test_reference_frame_and_pad(tb, hbd, bd):
    rng = np.random.default_rng(106)
    w, h = 192, 136
    href, cur, dref, dcur, drec = make_frames(tb, rng, w, h, bd, hbd)
    esz = 2 if hbd else 1
    # read back the whole padded luma/chroma planes of the GPU reference frame and compare with the oracle's padding
    for p in range(3):
        ptr, st = dref.plane(p)
        pw, ph, pad = (w, h, 160) if p == 0 else (w // 2, h // 2, 80)
        assert st == href.stride(p)
        nbytes = (ph + 2 * pad) * st * esz
        raw = np.empty(nbytes, np.uint8)
        tb.check(tb.lib.tb_memcpy_d2h(raw.ctypes.data, ptr - (pad * st + pad) * esz, nbytes))
        got = raw.view(sdt(hbd)).reshape(ph + 2 * pad, st)[:, :pw + 2 * pad]
        want = href.full(p)[:ph + 2 * pad, :pw + 2 * pad]
        assert (got == want).all(), p
    # pad in place == idempotent second application
    tb.check(tb.lib.tb_pad_frame(dref.h))
    ptr, st = dref.plane(0)
    raw = np.empty((h + 320) * st * esz, np.uint8)
    tb.check(tb.lib.tb_memcpy_d2h(raw.ctypes.data, ptr - (160 * st + 160) * esz, raw.nbytes))
    assert (raw.view(sdt(hbd)).reshape(h + 320, st)[:, :w + 320] == href.Y[:h + 320, :w + 320]).all()
    # 2x2 down-scaling
    small = tb.Frame(w // 2, h // 2, esz)
    tb.check(tb.lib.tb_scale_down2x2(dref.h, small.h))
    y, _, _ = small.download()
    want = aligned((h // 2, w // 2), sdt(hbd))
    getattr(O, "orc_scale_down2x2_" + sfx(hbd))(P(href.Y, href.origin(0)), href.sy, P(want), w // 2, w // 2, h // 2)
    assert (y == want).all()


@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_sad(tb, hbd, bd):
    rng = np.random.default_rng(107)
    s = sfx(hbd)
    w, h = 256, 192
    href, cur, dref, dcur, _ = make_frames(tb, rng, w, h, bd, hbd)
    esz = 2 if hbd else 1
    rptr, rst = dref.plane(0); optr, ost = dcur.plane(0)
    n = 600
    items = np.zeros(n, tb.SAD_ITEM)
    want = np.zeros(n, np.uint32); wantx = np.zeros(n, np.int32); want64 = np.zeros(n, np.uint64)
    shapes = [(4, 4), (4, 8), (8, 4), (8, 8), (16, 8), (8, 16), (16, 16), (32, 32), (64, 64), (128, 128), (64, 32)]
    meta = []
    for i in range(n):
        bw, bh = shapes[i % len(shapes)]
        x = 4 * int(rng.integers(0, (w - bw) // 4 + 1)); y = 4 * int(rng.integers(0, (h - bh) // 4 + 1))
        dx, dy = int(rng.integers(-150, 150)), int(rng.integers(-150, 150))
        dx = int(np.clip(x + dx, -140, w + 140 - bw)) - x; dy = int(np.clip(y + dy, -140, h + 140 - bh)) - y
        items[i] = (optr + (y * ost + x) * esz, rptr + ((y + dy) * rst + x + dx) * esz, ost, rst, bw, bh, 0)
        meta.append((x, y, dx, dy, bw, bh))
    d_items = tb.DevBuf.from_array(items)
    d_out = tb.DevBuf(4 * n); d_out2 = tb.DevBuf(4 * n); d_out64 = tb.DevBuf(8 * n)
    for kind in (0, 1, 2):
        tb.check(tb.lib.tb_sad_batch(d_items.ptr, n, esz, kind, d_out.ptr, d_out2.ptr, d_out64.ptr))
        got = d_out.download(np.uint32, n); got2 = d_out2.download(np.int32, n); got64 = d_out64.download(np.uint64, n)
        for i, (x, y, dx, dy, bw, bh) in enumerate(meta):
            a = P(cur.Y, cur.origin(0) + y * cur.sy + x); b = P(href.Y, href.origin(0) + (y + dy) * href.sy + x + dx)
            if kind == 0:
                assert got[i] == getattr(O, "orc_sad_" + s)(a, b, cur.sy, href.sy, bw, bh), i
            elif kind == 1:
                xo = C.c_int(0)
                assert got[i] == getattr(O, "orc_widesad_" + s)(a, b, cur.sy, href.sy, bw, bh, C.byref(xo)) and got2[i] == xo.value, i
            else:
                assert got64[i] == getattr(O, "orc_ssd_" + s)(a, b, cur.sy, href.sy, bw, bh), i


def me_batch(tb, rng, hbd, bd, w, h, n, edge, sizes, speed, bip):
    """n searches on a w x h frame pair in one tb_motion_estimate_batch, the last `edge` of them placed at the picture's edges (edge_search,
    signs alternating; their blocks come from a buffer of their own), each against the oracle.  Returns (differences, reach):
    reach[sign] counts the edge results on a clip_mv limit / through an active split_mv clamp (edge_reach)."""
    s = sfx(hbd)
    esz = 2 if hbd else 1
    href, cur, dref, dcur, _ = make_frames(tb, rng, w, h, bd, hbd)
    rptr, rst = dref.plane(0); optr, ost = dcur.plane(0)
    dorg = tb.DevBuf(max(edge, 1) * 128 * 128 * esz)
    items = np.zeros(n, tb.ME_ITEM)
    orgs = np.zeros((max(edge, 1), 128 * 128), sdt(hbd))
    cands, meta = [], []
    for i in range(n):
        e = i - (n - edge)
        size = int(rng.choice(sizes))
        part = int(rng.integers(0, 4))
        bw, bh, ox, oy = size, size, 0, 0
        if part == 1: bh = size // 2; oy = int(rng.integers(0, 2)) * bh
        if part == 2: bw = size // 2; ox = int(rng.integers(0, 2)) * bw
        if part == 3: bw = bh = size // 2; ox = int(rng.integers(0, 2)) * bw; oy = int(rng.integers(0, 2)) * bh
        nc = int(rng.integers(0, 9))
        if speed != 0 and nc == 0:
            nc = 1
        lam = float(rng.uniform(2.0, 60.0))
        if e < 0:
            xpos = int(rng.integers(0, w // size)) * size; ypos = int(rng.integers(0, h // size)) * size
            sign = int(rng.integers(0, 2))
            cc = rng.integers(-12, 12, (nc, 2)).astype(np.int16)
            mvc = rng.integers(-40, 40, 2); mvp = rng.integers(-40, 40, 2)
            org = cur.y[ypos:ypos + size, xpos:xpos + size]
            po, so = optr + ((ypos + oy) * ost + xpos + ox) * esz, ost
        else:
            sign = e % 2
            xpos, ypos, org, mvc, mvp, near = edge_search(rng, href.Y, w, h, size, bw, bh, sign, bd)
            cc = np.array(near(nc), np.int16).reshape(nc, 2)
            orgs[e, :size * size] = org.reshape(-1)
            po, so = dorg.ptr + (e * 128 * 128 + oy * size + ox) * esz, size
        items[i] = (po, rptr + ((ypos + oy) * rst + xpos + ox) * esz, so, rst, xpos, ypos, size, bw, bh, sign,
                    mvc[0], mvc[1], mvp[0], mvp[1], sum(len(c) for c in cands), nc, lam)
        cands.append(cc)
        meta.append((np.array(org), e >= 0, size, bw, bh, ox, oy, xpos, ypos, sign, cc, mvc, mvp, lam))
    dorg.upload(orgs)
    call = np.concatenate(cands + [np.zeros((1, 2), np.int16)]).astype(np.int16)
    d_items = tb.DevBuf.from_array(items); d_c = tb.DevBuf.from_array(call); d_out = tb.DevBuf(8 * n)
    tb.check(tb.lib.tb_motion_estimate_batch(d_items.ptr, n, d_c.ptr, esz, bd, speed, bip, w, h, d_out.ptr))
    got = d_out.download(tb.ME_RESULT, n)
    bad, reach = [], np.zeros((2, 2), int)
    for i, (blk, is_edge, size, bw, bh, ox, oy, xpos, ypos, sign, cc, mvc, mvp, lam) in enumerate(meta):
        org = aligned((size, size), sdt(hbd))
        org[...] = blk
        m0 = (C.c_int16 * 2)(0, 0)
        cands = (C.c_int16 * (2 * max(len(cc), 1)))(*[int(v) for v in cc.reshape(-1)] or [0, 0])
        cost = getattr(O, "orc_motion_estimate_" + s)(P(org, oy * size + ox), P(href.Y, href.origin(0) + (ypos + oy) * href.sy + xpos + ox), size, href.sy, bw, bh, m0,
                                                       (C.c_int16 * 2)(int(mvc[0]), int(mvc[1])), (C.c_int16 * 2)(int(mvp[0]), int(mvp[1])), C.c_double(lam), speed, bd,
                                                       sign, w, h, xpos, ypos, cands, len(cc), bip)
        res = (int(got[i]["cost"]), int(got[i]["mvx"]), int(got[i]["mvy"]))
        if res != (cost & 0xffffffff, m0[0], m0[1]):
            bad.append((w, h, i, is_edge, size, bw, bh, xpos, ypos, sign, len(cc), res, (cost, m0[0], m0[1])))
        if is_edge:
            reach[sign] += edge_reach(res[1], res[2], sign, xpos, ypos, w, h, size, bw, bh)
    return bad, reach


def me_batches(tb, hbd, bd, seed, dims, n, edge, sizes, speed, bip):
    """me_batch on each frame size of dims; the differences and reach of all of them"""
    rng = np.random.default_rng(seed)
    bad, reach = [], np.zeros((2, 2), int)
    for w, h in dims:
        b, r = me_batch(tb, rng, hbd, bd, w, h, n, edge, sizes, speed, bip)
        bad += b; reach += r
    return bad, reach


# the edge searches' results per sign on a clip_mv limit / through an active split_mv clamp, at least, as fractions of the edge items of one
# sign (the oracle's results for the same seeded items reach 0.22..0.39 / 0.89..0.98, and 0.47..0.53 / 0.75..0.87 in the bi-directional search)
ME_EDGE_REACH = np.array([0.15, 0.75])
ME_BI_EDGE_REACH = np.array([0.3, 0.55])
EDGE_DIMS = ((256, 192), (200, 136))


@pytest.mark.parametrize("hbd,bd", BD)
@pytest.mark.parametrize("speed,bip", [(0, 1), (0, 0), (1, 0), (2, 0), (1, 1)])
def test_batch_motion_estimate(tb, hbd, bd, speed, bip):
    """8x8 .. 64x64 coding blocks and their partitions at random positions and at the picture's edges; same results as the oracle"""
    bad, reach = me_batches(tb, hbd, bd, 108 + speed * 7 + bip, EDGE_DIMS, 160, 64, (8, 16, 32, 64), speed, bip)
    assert not bad, (len(bad), bad[:8])
    assert (reach >= ME_EDGE_REACH * 64).all(), reach


@pytest.mark.parametrize("hbd,bd", BD)
@pytest.mark.parametrize("sizes,n,bip", [((8,), 160, 1), ((8, 16), 480, 1), ((8,), 96, 0)])
def test_motion_estimate_small_blocks(tb, hbd, bd, sizes, n, bip):
    """blocks of <= 64 samples, incl. the wide-SAD candidates of 8x8 partitions of 16x16 coding blocks; same results as the oracle"""
    bad, reach = me_batches(tb, hbd, bd, 137 + n, EDGE_DIMS, n, n // 2, sizes, 0, bip)
    assert not bad, (len(bad), bad[:6])
    assert (reach >= ME_EDGE_REACH * (n // 2)).all(), reach


@pytest.mark.parametrize("hbd,bd", BD)
def test_motion_estimate_large_blocks(tb, hbd, bd):
    """64x64 and 128x128 coding blocks and their partitions (32x32 .. 128x128 prediction blocks); same results as the oracle"""
    bad, reach = me_batches(tb, hbd, bd, 131, ((384, 256), (200, 136)), 36, 18, (64, 128), 0, 1)
    assert not bad, (len(bad), bad[:6])
    assert (reach >= ME_EDGE_REACH * 18).all(), reach


@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_interp(tb, hbd, bd):
    rng = np.random.default_rng(109)
    s = sfx(hbd)
    w, h = 256, 192
    esz = 2 if hbd else 1
    href, cur, dref, dcur, _ = make_frames(tb, rng, w, h, bd, hbd)
    # the last `edge` items sit at the picture's edges with vectors at or past clip_mv's limit (edge_search), then clipped; 128-wide and
    # 128-tall luma blocks go through warp_interp_strips_u8 on 8-bit frames, as in the RD loop
    n, edge = 600, 200
    items = np.zeros(n, tb.INTERP_ITEM)
    out = tb.DevBuf(n * 128 * 128 * esz)
    meta = []
    clamped = 0
    for i in range(n):
        chroma = int(i % 3 == 2)
        size = int(rng.choice([4, 8, 16, 32, 64, 128] if not chroma else [4, 8, 16, 32]))
        bw, bh = size, size
        if i % 5 == 1: bw //= 2
        if i % 5 == 2: bh //= 2
        bw, bh = max(bw, 4 if not chroma else 2), max(bh, 4 if not chroma else 2)
        pw, ph = (w, h) if not chroma else (w // 2, h // 2)
        xpos = int(rng.integers(0, pw // size)) * size; ypos = int(rng.integers(0, ph // size)) * size
        sign = int(rng.integers(0, 2))
        # luma-resolution MV, clipped like the callers do (common/inter_prediction.c:209)
        mv = (C.c_int16 * 2)(int(rng.integers(-600, 600)), int(rng.integers(-600, 600)))
        if i >= n - edge:
            lx, ly, _, emv, _, _ = edge_search(rng, href.Y, w, h, size << chroma, bw << chroma, bh << chroma, sign, bd)
            xpos, ypos = lx >> chroma, ly >> chroma
            mv[0], mv[1] = emv
        lx, ly = (xpos, ypos) if not chroma else (xpos * 2, ypos * 2)
        O.orc_clip_mv(mv, ly, lx, w, h, bw << chroma, bh << chroma, sign)
        clamped += i >= n - edge and not chroma and edge_reach(mv[0], mv[1], sign, xpos, ypos, w, h, size, bw, bh)[1]
        ptr, st = dref.plane(1 if chroma else 0)
        items[i] = (ptr + (ypos * st + xpos) * esz, out.ptr + i * 128 * 128 * esz, st, bw, xpos, ypos, mv[0], mv[1], bw, bh, sign, chroma, pw, ph, 0)
        meta.append((chroma, bw, bh, xpos, ypos, sign, mv[0], mv[1], pw, ph))
    assert clamped >= 100, clamped  # luma edge items predicted through an active split_mv clamp (130 of 133 with this seed)
    d_items = tb.DevBuf.from_array(items)
    for bip in (0, 1):
        tb.check(tb.lib.tb_interp_batch(d_items.ptr, n, esz, bd, bip))
        got = out.download(sdt(hbd), (n, 128 * 128))
        for i, (chroma, bw, bh, xpos, ypos, sign, mvx, mvy, pw, ph) in enumerate(meta):
            want = aligned((bh, bw), sdt(hbd))
            mv = (C.c_int16 * 2)(mvx, mvy)
            pl = 1 if chroma else 0
            src = P(href.full(pl), href.origin(pl) + ypos * href.stride(pl) + xpos)
            if chroma:
                getattr(O, "orc_get_inter_prediction_chroma_" + s)(P(want), src, bw, bh, href.stride(pl), bw, mv, sign, pw, ph, xpos, ypos, bd)
            else:
                getattr(O, "orc_get_inter_prediction_luma_" + s)(P(want), src, bw, bh, href.stride(pl), bw, mv, sign, bip, pw, ph, xpos, ypos, bd)
            assert (got[i, :bw * bh].reshape(bh, bw) == want).all(), (i, meta[i])


def txfm_chain_in_runs(tb, items, esz, bd, hbd, recbuf, cqbuf, res, rec, cq):
    """the batch again, its items ordered by size and `fast` flag so that the chain forms take runs of consecutive items together (up to
    12 of 4x4/8x8, four of a larger size), every third one without coeffq: each item's result, reconstruction and levels must be those
    of the first launch, and an item without coeffq writes no levels"""
    n = len(items)
    order = np.lexsort((items["fast"] & tb.TXFM_FAST, items["size"]))
    runs = items[order].copy()
    noq = np.arange(n) % 3 == 2
    runs["coeffq"][noq] = 0
    recbuf.upload(np.zeros(len(rec), sdt(hbd))); cqbuf.upload(np.zeros((n, 256), np.int16))
    d_items = tb.DevBuf.from_array(runs); d_out = tb.DevBuf(16 * n)
    tb.check(tb.lib.tb_txfm_chain_batch(d_items.ptr, n, esz, bd, d_out.ptr))
    assert (d_out.download(tb.TXFM_RESULT, n) == res[order]).all()
    assert (recbuf.download(sdt(hbd), (len(rec),)) == rec).all()
    cq2 = cqbuf.download(np.int16, (n, 256))
    nq = np.arange(256) < np.minimum(items["size"].astype(int), 16)[:, None] ** 2  # the levels an item writes
    assert (cq2 == np.where(nq, cq, 0))[order[~noq]].all() and not cq2[order[noq]].any()


@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_txfm_chain(tb, hbd, bd):
    rng = np.random.default_rng(110)
    s = sfx(hbd)
    w, h = 256, 256
    esz = 2 if hbd else 1
    href, cur, dref, dcur, drec = make_frames(tb, rng, w, h, bd, hbd)
    n = 300
    items = np.zeros(n, tb.TXFM_ITEM)
    optr, ost = dcur.plane(0); pptr, pst = dref.plane(0)
    recbuf = tb.DevBuf(n * 128 * 128 * esz if n * 128 * 128 * esz < (1 << 28) else 1 << 28)
    cqbuf = tb.DevBuf(n * 256 * 2)
    meta = []
    sizes = [4, 8, 16, 32, 64, 128]
    recofs = 0
    for i in range(n):
        size = sizes[i % 6] if i % 12 < 11 else 4
        x = 4 * int(rng.integers(0, (w - size) // 4 + 1)); y = 4 * int(rng.integers(0, (h - size) // 4 + 1))
        px, py = x + int(rng.integers(-4, 5)), y + int(rng.integers(-4, 5))
        qp = int(rng.integers(0, 52)); typ = int(rng.integers(0, 4)); fast = int(rng.integers(0, 2))
        bits_flag = tb.TXFM_BITS if i % 5 else 0  # most items also ask for the write_coeff bit count (SURVEY 8f.2)
        items[i] = (optr + (y * ost + x) * esz, pptr + (py * pst + px) * esz, recbuf.ptr + recofs * esz, cqbuf.ptr + i * 512, ost, pst, size, size, qp, typ, fast | bits_flag)
        meta.append((size, x, y, px, py, qp, typ, fast, recofs))
        recofs += size * size
    d_items = tb.DevBuf.from_array(items); d_out = tb.DevBuf(16 * n)
    tb.check(tb.lib.tb_txfm_chain_batch(d_items.ptr, n, esz, bd, d_out.ptr))
    res = d_out.download(tb.TXFM_RESULT, n)
    rec = recbuf.download(sdt(hbd), (recofs,))
    cq = cqbuf.download(np.int16, (n, 256))
    ncbp = 0
    for i, (size, x, y, px, py, qp, typ, fast, ro) in enumerate(meta):
        q = min(size, 16)
        org = P(cur.Y, cur.origin(0) + y * cur.sy + x); prd = P(href.Y, href.origin(0) + py * href.sy + px)
        blk = aligned((size, size), np.int16); cf = aligned((size, size), np.int16, fill=0); cq0 = aligned((q * q,), np.int16, fill=0)
        getattr(O, "orc_residual_" + s)(P(blk), prd, org, size, href.sy, cur.sy)
        O.orc_transform(P(blk), P(cf), size, fast, bd)
        cbp = O.orc_quantize(P(cf), P(cq0), qp, size, typ, None)
        want = aligned((size, size), sdt(hbd))
        if cbp:
            rc = aligned((size, size), np.int16, fill=0); rb = aligned((size, size), np.int16)
            O.orc_dequantize(P(cq0), P(rc), qp, size, None)
            O.orc_inverse_transform(P(rc), P(rb), size, bd)
            getattr(O, "orc_reconstruct_" + s)(P(rb), prd, P(want), size, href.sy, size, bd)
        else:
            want[...] = href.Y[160 + py:160 + py + size, 160 + px:160 + px + size]
        ssd = getattr(O, "orc_ssd_" + s)(org, P(want), cur.sy, size, size, size)
        assert int(res[i]["cbp"]) == cbp, (i, size, qp)
        assert (cq[i, :q * q] == cq0).all(), (i, size, qp, typ)
        assert (rec[ro:ro + size * size].reshape(size, size) == want).all(), (i, size, qp)
        assert int(res[i]["ssd"]) == ssd, (i, size)
        want_bits = O.orc_coeff_bits(P(cq0), size, typ) if (i % 5 and cbp) else 0
        assert int(res[i]["bits"]) == want_bits, (i, size, qp, typ, int(res[i]["bits"]), want_bits)
        ncbp += cbp
    assert 0 < ncbp < n
    txfm_chain_in_runs(tb, items, esz, bd, hbd, recbuf, cqbuf, res, rec, cq)


def full_scale_blocks(bd, hbd, n=128):
    """(name, orig, pred) n x n pairs whose residual is +-(2^bd-1): constant of either sign, 8x8 cells and single samples of alternating sign"""
    maxv = (1 << bd) - 1
    yy, xx = np.mgrid[0:n, 0:n]
    out = []
    for name, o in (("max - 0", np.ones((n, n), int)), ("0 - max", np.zeros((n, n), int)), ("cells", (yy // 8 + xx // 8) % 2), ("dots", (yy + xx) % 2)):
        org = aligned((n, n), sdt(hbd)); prd = aligned((n, n), sdt(hbd))
        org[...] = o * maxv; prd[...] = (1 - o) * maxv
        out.append((name, org, prd))
    return out


@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_txfm_chain_full_scale(tb, hbd, bd):
    """the chain on residuals of +-(2^bd-1) at every size, qp and fast flag, where the int16 intermediates have the least headroom: at 12 bits
    the box sums of 128x128 without fast wrap in int16 and those with fast saturate (common/common_kernels.c:1519-1551)"""
    s = sfx(hbd)
    esz = 2 if hbd else 1
    pats = full_scale_blocks(bd, hbd)
    d_org = [tb.DevBuf.from_array(o) for _, o, _ in pats]; d_prd = [tb.DevBuf.from_array(p) for _, _, p in pats]
    meta = []
    for k in range(len(pats)):
        for size in (4, 8, 16, 32, 64, 128):
            for qp in range(52):
                for fast in (0, 1):
                    meta.append((k, size, qp, (qp + size + k) % 4, fast))
    n = len(meta)
    recofs = np.cumsum([0] + [m[1] * m[1] for m in meta])
    recbuf = tb.DevBuf(int(recofs[-1]) * esz); cqbuf = tb.DevBuf(n * 512)
    items = np.zeros(n, tb.TXFM_ITEM)
    for i, (k, size, qp, typ, fast) in enumerate(meta):
        items[i] = (d_org[k].ptr, d_prd[k].ptr, recbuf.ptr + int(recofs[i]) * esz, cqbuf.ptr + i * 512, 128, 128, size, size, qp, typ, fast | tb.TXFM_BITS)
    d_items = tb.DevBuf.from_array(items); d_out = tb.DevBuf(16 * n)
    tb.check(tb.lib.tb_txfm_chain_batch(d_items.ptr, n, esz, bd, d_out.ptr))
    res = d_out.download(tb.TXFM_RESULT, n)
    rec = recbuf.download(sdt(hbd), (int(recofs[-1]),))
    cq = cqbuf.download(np.int16, (n, 256))
    bad = []
    for i, (k, size, qp, typ, fast) in enumerate(meta):
        name, org, prd = pats[k]
        q = min(size, 16)
        blk = aligned((size, size), np.int16); cf = aligned((size, size), np.int16, fill=0); cq0 = aligned((q * q,), np.int16, fill=0)
        getattr(O, "orc_residual_" + s)(P(blk), P(prd), P(org), size, 128, 128)
        O.orc_transform(P(blk), P(cf), size, fast, bd)
        cbp = O.orc_quantize(P(cf), P(cq0), qp, size, typ, None)
        want = aligned((size, size), sdt(hbd))
        if cbp:
            rc = aligned((size, size), np.int16, fill=0); rb = aligned((size, size), np.int16)
            O.orc_dequantize(P(cq0), P(rc), qp, size, None)
            O.orc_inverse_transform(P(rc), P(rb), size, bd)
            getattr(O, "orc_reconstruct_" + s)(P(rb), P(prd), P(want), size, 128, size, bd)
        else:
            want[...] = prd[:size, :size]
        ssd = getattr(O, "orc_ssd_" + s)(P(org), P(want), 128, size, size, size)
        bits = O.orc_coeff_bits(P(cq0), size, typ) if cbp else 0
        got = rec[recofs[i]:recofs[i] + size * size].reshape(size, size)
        if not (int(res[i]["cbp"]) == cbp and (cq[i, :q * q] == cq0).all() and (got == want).all() and int(res[i]["ssd"]) == ssd and int(res[i]["bits"]) == bits):
            bad.append((name, size, qp, typ, fast))
    assert not bad, (len(bad), bad[:8])
    txfm_chain_in_runs(tb, items, esz, bd, hbd, recbuf, cqbuf, res, rec, cq)


@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_intra(tb, hbd, bd):
    rng = np.random.default_rng(111)
    s = sfx(hbd)
    w, h = 256, 192
    esz = 2 if hbd else 1
    href, cur, dref, dcur, drec = make_frames(tb, rng, w, h, bd, hbd)
    ptr, st = drec.plane(0)
    n = 500
    items = np.zeros(n, tb.INTRA_ITEM)
    out = tb.DevBuf(n * 64 * 64 * esz)
    meta = []
    for i in range(n):
        size = int(rng.choice([4, 8, 16, 32, 64]))
        xpos = int(rng.integers(0, w // size)) * size; ypos = int(rng.integers(0, h // size)) * size
        if i % 7 == 0: xpos = 0
        if i % 11 == 0: ypos = 0
        mode = i % 10
        ur = int(rng.integers(0, 2)) if (ypos > 0 and xpos + size < w) else 0
        dl = int(rng.integers(0, 2)) if (xpos > 0 and ypos + size < h) else 0
        items[i] = (ptr + (ypos * st + xpos) * esz, out.ptr + i * 64 * 64 * esz, st, xpos, ypos, size, mode, ur, dl)
        meta.append((size, xpos, ypos, mode, ur, dl))
    d_items = tb.DevBuf.from_array(items)
    tb.check(tb.lib.tb_intra_batch(d_items.ptr, n, esz, bd))
    got = out.download(sdt(hbd), (n, 64 * 64))
    for i, (size, xpos, ypos, mode, ur, dl) in enumerate(meta):
        left = aligned((264,), sdt(hbd), fill=0); top = aligned((264,), sdt(hbd), fill=0); tl = aligned((1,), sdt(hbd), fill=0)
        getattr(O, "orc_make_top_and_left_" + s)(P(left), P(top), P(tl), P(href.Y, href.origin(0) + ypos * href.sy + xpos), href.sy, None, 0, 0, 0, ypos, xpos, size, ur,
                                                  dl, 0, bd)
        want = aligned((size, size), sdt(hbd))
        getattr(O, "orc_intra_pred_" + s)(P(left), P(top), int(tl[0]), ypos, xpos, size, P(want), size, mode, bd)
        assert (got[i, :size * size].reshape(size, size) == want).all(), (i, meta[i])


@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_intra_full_scale_neighbours(tb, hbd, bd):
    """every intra mode and size with neighbours at 0 and 2^bd-1, at the frame's edges and inside it, with and without the up-right and
    down-left neighbours"""
    s = sfx(hbd)
    w, h = 192, 128
    esz = 2 if hbd else 1
    for name, v in full_scale_planes(h, w, (1 << bd) - 1).items():
        f = HFrame(w, h, bd, hbd)
        f.y[...] = v
        drec = tb.Frame(w, h, esz)
        drec.upload(f.y, f.u, f.v)
        ptr, st = drec.plane(0)
        meta = []
        for size in (4, 8, 16, 32, 64):
            for xpos, ypos in ((0, 0), (size, 0), (0, size), (size, size), (w - 2 * size, h - 2 * size)):
                for mode in range(10):
                    ur = int(ypos > 0 and xpos + size < w)
                    dl = int(xpos > 0 and ypos + size < h and mode % 2 == 0)
                    meta.append((size, xpos, ypos, mode, ur, dl))
        n = len(meta)
        items = np.zeros(n, tb.INTRA_ITEM)
        out = tb.DevBuf(n * 64 * 64 * esz)
        for i, (size, xpos, ypos, mode, ur, dl) in enumerate(meta):
            items[i] = (ptr + (ypos * st + xpos) * esz, out.ptr + i * 64 * 64 * esz, st, xpos, ypos, size, mode, ur, dl)
        d_items = tb.DevBuf.from_array(items)
        tb.check(tb.lib.tb_intra_batch(d_items.ptr, n, esz, bd))
        got = out.download(sdt(hbd), (n, 64 * 64))
        for i, (size, xpos, ypos, mode, ur, dl) in enumerate(meta):
            left = aligned((264,), sdt(hbd), fill=0); top = aligned((264,), sdt(hbd), fill=0); tl = aligned((1,), sdt(hbd), fill=0)
            getattr(O, "orc_make_top_and_left_" + s)(P(left), P(top), P(tl), P(f.Y, f.origin(0) + ypos * f.sy + xpos), f.sy, None, 0, 0, 0, ypos, xpos, size, ur, dl, 0, bd)
            want = aligned((size, size), sdt(hbd))
            getattr(O, "orc_intra_pred_" + s)(P(left), P(top), int(tl[0]), ypos, xpos, size, P(want), size, mode, bd)
            assert (got[i, :size * size].reshape(size, size) == want).all(), (name, meta[i])


def run_filters(tb, rng, w, h, bd, hbd, qp=33):
    """deblock -> CDEF (3 planes) -> CLPF (3 planes) on the GPU and in the oracle; returns (gpu planes, oracle frame)"""
    s = sfx(hbd)
    esz = 2 if hbd else 1
    f = HFrame(w, h, bd, hbd, 32, 32)
    f.randomize(rng)
    org = f.copy()
    for p in range(3):
        org.plane(p)[...] = np.clip(f.plane(p).astype(int) + rng.integers(-5, 6, f.plane(p).shape), 0, (1 << bd) - 1)
    bi, _ = random_blkinfo(rng, w, h)
    drec = tb.Frame(w, h, esz, 32); dscr = tb.Frame(w, h, esz, 32); dorg = tb.Frame(w, h, esz, 32)
    drec.upload(f.y, f.u, f.v); dorg.upload(org.y, org.u, org.v)
    dbi = tb.DevBuf.from_array(bi)
    stages = {}
    # --- deblock
    tb.check(tb.lib.tb_deblock_frame(drec.h, dbi.ptr, qp, bd))
    getattr(O, "orc_deblock_y_" + s)(P(f.Y, f.origin(0)), f.sy, P(bi), w, h, qp, bd)
    getattr(O, "orc_deblock_uv_" + s)(P(f.U, f.origin(1)), P(f.V, f.origin(1)), f.sc, P(bi), w, h, 1, O.orc_chroma_qp(qp), bd)
    stages["deblock"] = (drec.download(), [f.plane(p).copy() for p in range(3)])
    # --- CLPF detect sums on the deblocked frame
    nb = (w // 8) * (h // 8)
    dsum = tb.DevBuf(16 * nb)
    tb.check(tb.lib.tb_clpf_detect_frame(drec.h, dorg.h, dbi.ptr, 0, bd, qp, dsum.ptr))
    gs = dsum.download(np.int32, (nb, 4))
    ws = np.zeros((nb, 4), np.int32)
    for b in range(nb):
        x0, y0 = (b % (w // 8)) * 8, (b // (w // 8)) * 8
        if bi[y0 // 4, x0 // 4]["mode"] != 0:
            m = (C.c_int * 4)(0, 0, 0, 0)
            getattr(O, "orc_detect_multi_clpf_" + s)(P(f.Y, f.origin(0)), P(org.Y, org.origin(0)), x0, y0, w, h, org.sy, f.sy, m, bd - 8, 8, bd - 4 + (qp >> 4))
            ws[b] = list(m)
    stages["detect"] = (gs, ws)
    # --- CDEF
    nfb = ((w + 63) // 64) * ((h + 63) // 64)
    pri = rng.integers(0, 16, (2, nfb)).astype(np.int8); sec = rng.integers(0, 4, (2, nfb)).astype(np.int8)
    dpri = [tb.DevBuf.from_array(pri[k]) for k in range(2)]; dsec = [tb.DevBuf.from_array(sec[k]) for k in range(2)]
    ddv = tb.DevBuf(nfb * 2 * 64 * 4)
    dirs = np.zeros((nfb, 64), np.int32); vars_ = np.zeros((nfb, 64), np.int32)
    for plane in range(3):
        tb.check(tb.lib.tb_cdef_frame(drec.h, dscr.h, dbi.ptr, dpri[int(plane > 0)].ptr, dsec[int(plane > 0)].ptr, 5, 5, ddv.ptr, bd, plane))
        src = f.full(plane)
        dst = src.copy()
        getattr(O, "orc_cdef_plane_" + s)(P(src, f.origin(plane)), P(dst, f.origin(plane)), f.stride(plane), w, h, P(bi), w // 4, 1, plane, P(pri[int(plane > 0)]),
                                          P(sec[int(plane > 0)]), 5, 5, P(dirs), P(vars_), bd)
        src[...] = dst
    stages["cdef"] = (drec.download(), [f.plane(p).copy() for p in range(3)])
    # --- CLPF
    for plane, (fbl, strength) in enumerate(((6, 2), (4, 1), (4, 4))):
        tb.check(tb.lib.tb_clpf_frame(drec.h, dscr.h, dbi.ptr, None, fbl, strength, bd, plane, qp))
        src = f.full(plane)
        dst = src.copy()
        pw, ph = (w, h) if plane == 0 else (w // 2, h // 2)
        getattr(O, "orc_clpf_plane_" + s)(P(src, f.origin(plane)), P(dst, f.origin(plane)), f.stride(plane), pw, ph, P(bi), w // 4, int(plane != 0), None, fbl, strength,
                                          bd, plane, qp)
        src[...] = dst
    stages["clpf"] = (drec.download(), [f.plane(p).copy() for p in range(3)])
    return stages


@pytest.mark.parametrize("hbd,bd", BD)
@pytest.mark.parametrize("dims", [(192, 136), (320, 192)])
def test_frame_filters(tb, hbd, bd, dims):
    rng = np.random.default_rng(112)
    stages = run_filters(tb, rng, dims[0], dims[1], bd, hbd)
    for name in ("deblock", "cdef", "clpf"):
        got, want = stages[name]
        for p in range(3):
            assert (got[p] == want[p]).all(), (name, p, int((got[p] != want[p]).sum()))
    gs, ws = stages["detect"]
    assert (gs == ws).all()


def test_frame_filters_1080p(tb):
    """BASELINE size: the whole in-loop filter chain on a 1920x1080 frame, bit-exact against the oracle."""
    rng = np.random.default_rng(113)
    stages = run_filters(tb, rng, 1920, 1080, 8, 0, qp=35)
    for name in ("deblock", "cdef", "clpf"):
        got, want = stages[name]
        for p in range(3):
            assert (got[p] == want[p]).all(), (name, p)
    assert (stages["detect"][0] == stages["detect"][1]).all()


def test_me_1080p_properties(tb):
    """Full-size, size-independent properties of the motion search on a 1920x1080 frame pair: (i) a pure global
    translation of the reference, offered as a candidate, is kept through all refinement stages with zero SAD, (ii) results do not depend on batch order."""
    rng = np.random.default_rng(114)
    w, h, bd, hbd, esz = 1920, 1080, 8, 0, 1
    href = HFrame(w, h, bd, hbd)
    href.randomize(rng, smooth=False)
    getattr(O, "orc_pad_plane_lbd")(P(href.Y, href.origin(0)), href.sy, w, h, 160, 160)
    cur = HFrame(w, h, bd, hbd)
    # cur(y,x) = ref(y+2, x-3)  <=>  MV = (-3*4, +2*4) quarter-pels
    cur.y[...] = href.Y[160 + 2:160 + 2 + h, 160 - 3:160 - 3 + w]
    drec = tb.Frame(w, h, esz); dref = tb.Frame(w, h, esz); dcur = tb.Frame(w, h, esz)
    drec.upload(href.y, href.u, href.v); dcur.upload(cur.y, cur.u, cur.v)
    tb.check(tb.lib.tb_create_reference_frame(dref.h, drec.h))
    rptr, rst = dref.plane(0); optr, ost = dcur.plane(0)
    blocks = [(x, y) for y in range(0, h - 15, 16) for x in range(0, w, 16)]
    n = len(blocks)
    items = np.zeros(n, tb.ME_ITEM)
    for i, (x, y) in enumerate(blocks):
        items[i] = (optr + (y * ost + x) * esz, rptr + (y * rst + x) * esz, ost, rst, x, y, 16, 16, 16, 0, 0, 0, 0, 0, 0, 1, 4.0)
    # white-noise content has no gradient for the telescope search to follow, so the true displacement is offered as
    # the (single) candidate vector, like a neighbour's MV would be in the encoder
    cands = tb.DevBuf.from_array(np.array([[-3, 2]], np.int16))
    d_items = tb.DevBuf.from_array(items); d_out = tb.DevBuf(8 * n)
    tb.check(tb.lib.tb_motion_estimate_batch(d_items.ptr, n, cands.ptr, esz, bd, 0, 1, w, h, d_out.ptr))
    r1 = d_out.download(tb.ME_RESULT, n)
    assert (r1["mvx"] == -12).all() and (r1["mvy"] == 8).all()
    bits_cost = O.orc_quote_mv_bits(8, -12)
    assert (r1["cost"] == int(4.0 * bits_cost + 0.5)).all()
    perm = rng.permutation(n)
    d_items.upload(items[perm])
    tb.check(tb.lib.tb_motion_estimate_batch(d_items.ptr, n, cands.ptr, esz, bd, 0, 1, w, h, d_out.ptr))
    r2 = d_out.download(tb.ME_RESULT, n)
    assert (r2 == r1[perm]).all()


def _ti_case(tb, rng, w, h, bd, hbd, hard, ratio, pos):
    import math
    s = sfx(hbd)
    esz = 2 if hbd else 1
    a = HFrame(w, h, bd, hbd); a.randomize(rng)
    b = HFrame(w, h, bd, hbd)
    amp = 14 if hard else 3
    for p in range(3):
        sh = (1, -2) if p == 0 else (0, -1)
        b.plane(p)[...] = np.clip(np.roll(a.plane(p).astype(int), sh, axis=(0, 1)) + rng.integers(-amp, amp + 1, a.plane(p).shape), 0, (1 << bd) - 1)
    b.y[h // 4:h // 4 + 40, w // 3:w // 3 + 56] = np.clip(a.y[h // 4 + 6:h // 4 + 46, w // 3 - 9:w // 3 + 47].astype(int) + 20, 0, (1 << bd) - 1)
    dev = []
    for f in (a, b):
        t = tb.Frame(w, h, esz); t.upload(f.y, f.u, f.v)
        r = tb.Frame(w, h, esz)
        tb.check(tb.lib.tb_create_reference_frame(r.h, t.h))
        dev.append(r)
        for p, (pw, ph, pad) in enumerate(((w, h, 160), (w // 2, h // 2, 80), (w // 2, h // 2, 80))):
            getattr(O, "orc_pad_plane_" + s)(P(f.full(p), f.origin(p)), f.stride(p), pw, ph, pad, pad)
    out = tb.Frame(w, h, esz)
    tb.check(tb.lib.tb_interpolate_frames(out.h, dev[0].h, dev[1].h, ratio, pos))
    got = out.download()
    o2 = HFrame(w, h, bd, hbd)
    levels = min(4, int(math.log10(min(w, h)) / math.log10(2.0) - 4.0))
    getattr(O, "orc_interpolate_frames_" + s)(P(o2.Y, o2.origin(0)), P(o2.U, o2.origin(1)), P(o2.V, o2.origin(1)), o2.sy, o2.sc, P(a.Y, a.origin(0)), P(a.U, a.origin(1)),
                                             P(a.V, a.origin(1)), P(b.Y, b.origin(0)), P(b.U, b.origin(1)), P(b.V, b.origin(1)), a.sy, a.sc, w, h, 160, ratio, pos, levels)
    return got, [o2.plane(p).copy() for p in range(3)], a


@pytest.mark.parametrize("hbd,bd", BD)
def test_interpolate_frames(tb, hbd, bd):
    rng = np.random.default_rng(115)
    for (w, h) in [(128, 72), (192, 136), (320, 192)]:
        for hard in (False, True):
            for ratio, pos in [(2, 1), (4, 3), (8, 5)]:
                got, want, a = _ti_case(tb, rng, w, h, bd, hbd, hard, ratio, pos)
                for p in range(3):
                    assert (got[p] == want[p]).all(), (w, h, hard, ratio, pos, p, int((got[p] != want[p]).sum()))
                assert (got[0] != a.y).any()


def test_interpolate_frames_1080p(tb):
    rng = np.random.default_rng(116)
    for hard in (False, True):
        got, want, _ = _ti_case(tb, rng, 1920, 1080, 8, 0, hard, 2, 1)
        for p in range(3):
            assert (got[p] == want[p]).all(), (hard, p, int((got[p] != want[p]).sum()))


@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_motion_estimate_bi_and_combine(tb, hbd, bd):
    """the bi-directional search at random positions and, for the last 40 items of a batch, at the picture's edges (edge_search; the list
    entries are quarter-pel vectors, clipped again with the other sign for the second reference); then the element-wise combinations"""
    rng = np.random.default_rng(117)
    s = sfx(hbd)
    esz = 2 if hbd else 1
    n, edge = 100, 40
    reach = np.zeros((2, 2), int)
    for w, h in ((192, 128),) + EDGE_DIMS:
        href, cur, dref, dcur, _ = make_frames(tb, rng, w, h, bd, hbd)
        href2, _, dref2, _, _ = make_frames(tb, rng, w, h, bd, hbd, shift=(-1, 2))
        r0, rst = dref.plane(0); r1, _ = dref2.plane(0); optr, ost = dcur.plane(0)
        items = np.zeros(n, tb.ME_BI_ITEM)
        cands = rng.integers(-20, 20, (n, 4, 2)).astype(np.int16)
        dorg = tb.DevBuf(edge * 64 * 64 * esz)
        orgs = np.zeros((edge, 64 * 64), sdt(hbd))
        meta = []
        for i in range(n):
            size = int(rng.choice([8, 16, 32, 64]))
            nc = int(rng.integers(0, 5)); lam = float(rng.uniform(2.0, 40.0))
            e = i - (n - edge)
            if e < 0:
                xpos = int(rng.integers(0, w // size)) * size; ypos = int(rng.integers(0, h // size)) * size
                sign = int(rng.integers(0, 2))
                mvc = rng.integers(-30, 30, 2); mvp = rng.integers(-30, 30, 2)
                org = cur.y[ypos:ypos + size, xpos:xpos + size]
                po, so = optr + (ypos * ost + xpos) * esz, ost
            else:
                sign = e % 2
                xpos, ypos, org, mvc, mvp, near = edge_search(rng, href.Y, w, h, size, size, size, sign, bd)
                cands[i] = [[4 * v + int(rng.integers(-3, 4)) for v in c] for c in near(4)]
                orgs[e, :size * size] = org.reshape(-1)
                po, so = dorg.ptr + e * 64 * 64 * esz, size
            items[i] = (po, r0 + (ypos * rst + xpos) * esz, r1 + (ypos * rst + xpos) * esz, so, rst, xpos, ypos, size, sign, 0, 0,
                        mvc[0], mvc[1], mvp[0], mvp[1], 4 * i, nc, lam)
            meta.append((np.array(org), e >= 0, size, xpos, ypos, sign, nc, lam, mvc, mvp))
        dorg.upload(orgs)
        d_items = tb.DevBuf.from_array(items); d_c = tb.DevBuf.from_array(cands); d_out = tb.DevBuf(8 * n)
        tb.check(tb.lib.tb_motion_estimate_bi_batch(d_items.ptr, n, d_c.ptr, esz, bd, 1, w, h, d_out.ptr))
        got = d_out.download(tb.ME_RESULT, n)
        for i, (blk, is_edge, size, xpos, ypos, sign, nc, lam, mvc, mvp) in enumerate(meta):
            org = aligned((size, size), sdt(hbd))
            org[...] = blk
            m0 = (C.c_int16 * 2)(0, 0)
            cc = (C.c_int16 * 8)(*[int(v) for v in cands[i].reshape(-1)])
            cost = getattr(O, "orc_motion_estimate_bi_" + s)(P(org), P(href.Y, href.origin(0) + ypos * href.sy + xpos), P(href2.Y, href2.origin(0) + ypos * href2.sy + xpos), size,
                                                              href.sy, size, size, m0, (C.c_int16 * 2)(int(mvc[0]), int(mvc[1])), (C.c_int16 * 2)(int(mvp[0]), int(mvp[1])),
                                                              C.c_double(lam), bd, sign, w, h, xpos, ypos, cc, nc, 1)
            res = (int(got[i]["cost"]), int(got[i]["mvx"]), int(got[i]["mvy"]))
            assert res == (cost, m0[0], m0[1]), (w, h, i, is_edge, size, xpos, ypos, sign, nc)
            if is_edge:
                reach[sign] += np.logical_or(*[edge_reach(res[1], res[2], sg, xpos, ypos, w, h, size, size, size) for sg in (sign, 1 - sign)])
        if (w, h) == (192, 128):
            first = w, h, href, cur, dref, dcur
    assert (reach >= ME_BI_EDGE_REACH * 3 * edge // 2).all(), reach
    w, h, href, cur, dref, dcur = first
    r0, rst = dref.plane(0); optr, ost = dcur.plane(0)
    # element-wise combinations on resident frames
    m = 90
    citems = np.zeros(m, tb.COMBINE_ITEM)
    out = tb.DevBuf(m * 64 * 64 * esz)
    cm = []
    for i in range(m):
        bw, bh = int(rng.choice([4, 8, 16, 32, 64])), int(rng.choice([4, 8, 16, 32, 64]))
        x, y = int(rng.integers(0, w - bw)), int(rng.integers(0, h - bh))
        citems[i] = (optr + (y * ost + x) * esz, r0 + (y * rst + x) * esz, out.ptr + i * 64 * 64 * esz, ost, rst, bw, bw, bh)
        cm.append((bw, bh, x, y))
    d_ci = tb.DevBuf.from_array(citems)
    for op in (0, 1, 2):
        tb.check(tb.lib.tb_block_combine_batch(d_ci.ptr, m, esz, op, bd))
        res = out.download(sdt(hbd), (m, 64 * 64))
        for i, (bw, bh, x, y) in enumerate(cm):
            want = aligned((bh, bw), sdt(hbd))
            getattr(O, "orc_block_combine_" + s)(P(want), bw, P(cur.Y, cur.origin(0) + y * cur.sy + x), cur.sy, P(href.Y, href.origin(0) + y * href.sy + x), href.sy, bw, bh, op, bd)
            assert (res[i, :bw * bh].reshape(bh, bw) == want).all(), (op, i)


@pytest.mark.parametrize("hbd,bd", BD)
def test_cdef_search_mse(tb, hbd, bd):
    """encoder-side CDEF strength search: the device distortion table must equal the oracle's (which is pinned against the reference's
    cdef_search through the greedy selection, tests/test_oracle_vs_ref.py::test_cdef_search)"""
    rng = np.random.default_rng(118)
    s = sfx(hbd)
    esz = 2 if hbd else 1
    for (w, h), speed in [((192, 136), 1), ((320, 192), 0), ((200, 136), 2)]:
        f = HFrame(w, h, bd, hbd, 32, 32); f.randomize(rng)
        org = f.copy()
        for p in range(3):
            org.plane(p)[...] = np.clip(f.plane(p).astype(int) + rng.integers(-7, 8, f.plane(p).shape), 0, (1 << bd) - 1)
        bi, _ = random_blkinfo(rng, w, h, p_skip=0.25)
        nfb = ((w + 63) // 64) * ((h + 63) // 64)
        drec = tb.Frame(w, h, esz, 32); dorg = tb.Frame(w, h, esz, 32)
        drec.upload(f.y, f.u, f.v); dorg.upload(org.y, org.u, org.v)
        dbi = tb.DevBuf.from_array(bi); ddv = tb.DevBuf(nfb * 2 * 64 * 4); dsk = tb.DevBuf(max(nfb, 16)); dmse = tb.DevBuf(2 * nfb * 64 * 8)
        tb.check(tb.lib.tb_cdef_search_mse(drec.h, dorg.h, dbi.ptr, speed, 5, bd, ddv.ptr, dsk.ptr, dmse.ptr))
        got = dmse.download(np.uint64, (2, nfb, 64)); gsk = dsk.download(np.uint8, (max(nfb, 16),))[:nfb]
        mse = np.zeros((2, nfb, 64), np.uint64); od = np.zeros((nfb, 64), np.int32); ov = np.zeros((nfb, 64), np.int32); ask = np.zeros(nfb, np.uint8)
        getattr(O, "orc_cdef_search_mse_" + s)(P(f.Y, f.origin(0)), P(f.U, f.origin(1)), P(f.V, f.origin(1)), P(org.Y, org.origin(0)), P(org.U, org.origin(1)),
                                                P(org.V, org.origin(1)), f.sy, f.sc, w, h, P(bi), speed, 5, bd, P(mse), P(od), P(ov), P(ask))
        assert (gsk == ask).all()
        if (w >> 1) & 7:
            # chroma blocks 4 wide and 8 tall: the reference filters sizex x sizex samples and then sums sizey rows of its scratch
            # block, i.e. rows left over from the previous call (enc/encode_frame.c:358-372); the device sums the filtered rows it has.
            nh = (w + 63) // 64
            got[1, nh - 1::nh] = 0; mse[1, nh - 1::nh] = 0
        assert (got == mse).all(), (w, h, speed, int((got != mse).sum()))
        assert mse.any()
