"""SAD, wide SAD, SSD and inter prediction at the rectangular blocks the bottom edges of 1080p and 2160p frames leave.  1080 = 8 * 128 + 56 and
2160 = 16 * 128 + 112, so the last super-block row is 56 or 112 rows tall, and in inter frames the RD loop decides the blocks that cross the
picture's bottom edge as rectangular skips (encode_rect): luma blocks 128, 64, 32 and 16 wide and 56, 24, 8 (1080p) or 112, 48, 16 (2160p) tall,
chroma blocks half of each (28, 12, 4 and 56, 24, 8 rows), all of them on the picture's last rows.  Widths stay powers of two.

GPU: tb_sad_batch (all three kinds) and tb_interp_batch (bi-prediction filters off and on) against the plain-C oracle, at every bit-depth mode.
CPU: the oracle against the compiled reference at the same shapes (SAD kernels, and the whole luma and chroma prediction of a rectangular block,
get_inter_prediction_yuv with clip_mv and split_mv's clamps), so that the oracle the GPU side is compared with is pinned there too."""
import ctypes as C

import numpy as np
import pytest

from _libs import P, aligned, oracle, ref, ref_enc, sdt, sfx
from _refstructs import Frame as HFrame, Mv

O = oracle()
BD = [(0, 8), (1, 8), (1, 10), (1, 12)]  # (1, 8): 8-bit content in 16-bit frames (-frame_bitdepth 16)
W = 256
# frame height: the heights inside the picture of the blocks that cross its bottom edge
EDGES = {184: (56, 24, 8), 240: (112, 48, 16)}   # the bottom rows of 1080 and 2160
WIDTHS = (128, 64, 32, 16)


def edge_blocks(rng, h, n_per_shape):
    """(chroma, x, y, width, height, plane width, plane height) of luma and chroma blocks ending on the picture's last row, in every column: every
    width with every edge height up to the width (a block is never taller than its size: (128, 56), (64, 56), (32, 24) and (16, 8) at 1080,
    (128, 112), (64, 48) and (32, 16) at 2160, and the other pairs at the same heights)"""
    out = []
    for bh in EDGES[h]:
        for bw in WIDTHS:
            if bh > bw:
                continue
            for k in range(n_per_shape):
                col = (W // bw - 1) if k == 0 else int(rng.integers(0, W // bw))
                for chroma in (0, 1):
                    s = 1 + chroma
                    out.append((chroma, col * bw // s, (h - bh) // s, bw // s, bh // s, W // s, h // s))
    return out


def random_mv(rng, x, y, bw, bh, pw, ph, chroma, sign):
    """a quarter-pel vector clipped as the RD loop clips it (clip_mv on the luma block): often far below the picture, where split_mv's
    pic_height - ypos clamp takes over, and at every fraction"""
    s = 1 + chroma
    mv = (C.c_int16 * 2)(int(rng.integers(-700, 700)), int(rng.integers(-300, 700)) * (1 if rng.integers(0, 3) else -1))
    O.orc_clip_mv(mv, y * s, x * s, pw * s, ph * s, bw * s, bh * s, sign)
    return mv


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: the batched kernels against the oracle
# ---------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tb():
    import thor_b200 as t
    t.init(0)
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("h", sorted(EDGES))
@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_sad_at_bottom_edge_blocks(tb, hbd, bd, h):
    from test_gpu_parity import make_frames
    rng = np.random.default_rng(171 + h)
    s = sfx(hbd)
    esz = 2 if hbd else 1
    href, cur, dref, dcur, _ = make_frames(tb, rng, W, h, bd, hbd)
    blocks = edge_blocks(rng, h, 3)
    items = np.zeros(len(blocks), tb.SAD_ITEM)
    meta = []
    for i, (chroma, x, y, bw, bh, pw, ph) in enumerate(blocks):
        pl = 1 if chroma else 0
        rptr, rst = dref.plane(pl); optr, ost = dcur.plane(pl)
        # the reference block anywhere within the padding the motion search reaches, below the picture included
        lim = 140 >> chroma
        dx = int(np.clip(x + rng.integers(-lim, lim), -lim, pw + lim - bw)) - x
        dy = int(np.clip(y + rng.integers(-lim, lim), -lim, ph + lim - bh)) - y
        items[i] = (optr + (y * ost + x) * esz, rptr + ((y + dy) * rst + x + dx) * esz, ost, rst, bw, bh, 0)
        meta.append((pl, x, y, dx, dy, bw, bh))
    d_items = tb.DevBuf.from_array(items)
    n = len(blocks)
    d_out = tb.DevBuf(4 * n); d_out2 = tb.DevBuf(4 * n); d_out64 = tb.DevBuf(8 * n)
    for kind in (0, 1, 2):
        tb.check(tb.lib.tb_sad_batch(d_items.ptr, n, esz, kind, d_out.ptr, d_out2.ptr, d_out64.ptr))
        got = d_out.download(np.uint32, n); got2 = d_out2.download(np.int32, n); got64 = d_out64.download(np.uint64, n)
        bad = []
        for i, (pl, x, y, dx, dy, bw, bh) in enumerate(meta):
            a = P(cur.full(pl), cur.origin(pl) + y * cur.stride(pl) + x)
            b = P(href.full(pl), href.origin(pl) + (y + dy) * href.stride(pl) + x + dx)
            if kind == 0:
                ok = got[i] == getattr(O, "orc_sad_" + s)(a, b, cur.stride(pl), href.stride(pl), bw, bh)
            elif kind == 1:
                xo = C.c_int(0)
                ok = got[i] == getattr(O, "orc_widesad_" + s)(a, b, cur.stride(pl), href.stride(pl), bw, bh, C.byref(xo)) and got2[i] == xo.value
            else:
                ok = got64[i] == getattr(O, "orc_ssd_" + s)(a, b, cur.stride(pl), href.stride(pl), bw, bh)
            if not ok:
                bad.append((kind, meta[i]))
        assert not bad, (len(bad), bad[:6])


@pytest.mark.gpu
@pytest.mark.parametrize("h", sorted(EDGES))
@pytest.mark.parametrize("hbd,bd", BD)
def test_batch_interp_at_bottom_edge_blocks(tb, hbd, bd, h):
    from test_gpu_parity import make_frames
    rng = np.random.default_rng(173 + h)
    s = sfx(hbd)
    esz = 2 if hbd else 1
    href, cur, dref, dcur, _ = make_frames(tb, rng, W, h, bd, hbd)
    blocks = edge_blocks(rng, h, 4)
    n = len(blocks)
    items = np.zeros(n, tb.INTERP_ITEM)
    out = tb.DevBuf(n * 128 * 128 * esz)
    meta = []
    below = 0
    for i, (chroma, x, y, bw, bh, pw, ph) in enumerate(blocks):
        sign = int(rng.integers(0, 2))
        mv = random_mv(rng, x, y, bw, bh, pw, ph, chroma, sign)
        below += ((-mv[1] if sign else mv[1]) >> (2 + chroma)) > ph - y   # predicted through split_mv's clamp at the bottom edge
        ptr, st = dref.plane(chroma)
        items[i] = (ptr + (y * st + x) * esz, out.ptr + i * 128 * 128 * esz, st, bw, x, y, mv[0], mv[1], bw, bh, sign, chroma, pw, ph, 0)
        meta.append((chroma, bw, bh, x, y, sign, mv[0], mv[1], pw, ph))
    assert below >= n // 8, below
    d_items = tb.DevBuf.from_array(items)
    for bip in (0, 1):
        tb.check(tb.lib.tb_interp_batch(d_items.ptr, n, esz, bd, bip))
        got = out.download(sdt(hbd), (n, 128 * 128))
        bad = []
        for i, (chroma, bw, bh, x, y, sign, mvx, mvy, pw, ph) in enumerate(meta):
            want = aligned((bh, bw), sdt(hbd))
            mv = (C.c_int16 * 2)(mvx, mvy)
            src = P(href.full(chroma), href.origin(chroma) + y * href.stride(chroma) + x)
            if chroma:
                getattr(O, "orc_get_inter_prediction_chroma_" + s)(P(want), src, bw, bh, href.stride(1), bw, mv, sign, pw, ph, x, y, bd)
            else:
                getattr(O, "orc_get_inter_prediction_luma_" + s)(P(want), src, bw, bh, href.stride(0), bw, mv, sign, bip, pw, ph, x, y, bd)
            if not (got[i, :bw * bh].reshape(bh, bw) == want).all():
                bad.append((bip, meta[i]))
        assert not bad, (len(bad), bad[:6])


# ---------------------------------------------------------------------------------------------------------------------------------------------------
# CPU: the oracle against the compiled reference at the same shapes
# ---------------------------------------------------------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(ref() is None, reason="oracle/_ref not built")


class BlockPos(C.Structure):
    """block_pos_t (common/types.h)"""
    _fields_ = [("ypos", C.c_uint16), ("xpos", C.c_uint16), ("size", C.c_uint8), ("bwidth", C.c_uint8), ("bheight", C.c_uint8), ("sb_size", C.c_uint8)]


@needs_ref
@pytest.mark.parametrize("h", sorted(EDGES))
@pytest.mark.parametrize("hbd,bd", BD)
def test_oracle_sad_at_bottom_edge_blocks_equals_reference(hbd, bd, h):
    rng = np.random.default_rng(175 + h)
    E, R = ref_enc(hbd), ref()
    s = sfx(hbd)
    f = HFrame(W, h, bd, hbd)
    f.randomize(rng, smooth=False)
    bad = []
    for chroma, x, y, bw, bh, pw, ph in edge_blocks(rng, h, 2):
        pl = 1 if chroma else 0
        org = aligned((bh, bw), sdt(hbd))
        org[...] = rng.integers(0, 1 << bd, (bh, bw))
        b = P(f.full(pl), f.origin(pl) + y * f.stride(pl) + x)
        st = f.stride(pl)
        want = getattr(O, "orc_sad_" + s)(P(org), b, bw, st, bw, bh)
        got = [getattr(E, "ref_sad_calc_" + s)(P(org), b, bw, st, bw, bh)] + ([getattr(R, "sad_calc_simd_" + s)(P(org), b, bw, st, bw, bh)] if bw > 4 else [])
        xo, xe = C.c_int(9), C.c_int(9)
        wide = (getattr(O, "orc_widesad_" + s)(P(org), b, bw, st, bw, bh, C.byref(xo)), xo.value)
        got_wide = (getattr(E, "ref_widesad_calc_" + s)(P(org), b, bw, st, bw, bh, C.byref(xe)), xe.value)
        ssd = getattr(O, "orc_ssd_" + s)(P(org), b, bw, st, bw, bh)
        got_ssd = getattr(E, "ref_ssd_calc_" + s)(P(org), b, bw, st, bw, bh)
        if any(g != want for g in got) or wide != got_wide or ssd != got_ssd:
            bad.append((chroma, x, y, bw, bh))
    assert not bad, (len(bad), bad[:6])


@needs_ref
@pytest.mark.parametrize("h", sorted(EDGES))
@pytest.mark.parametrize("hbd,bd", BD)
def test_oracle_prediction_of_bottom_edge_blocks_equals_reference(hbd, bd, h):
    """the reference's get_inter_prediction_yuv on a rectangular block (block_pos bwidth x bheight inside a size x size block, as encode_rect
    predicts it) against the oracle's luma and chroma predictions of the same block"""
    rng = np.random.default_rng(177 + h)
    R = ref()
    s = sfx(hbd)
    f = HFrame(W, h, bd, hbd)
    f.randomize(rng, smooth=False)
    getattr(R, "pad_yuv_frame_" + s)(C.byref(f.s))
    bad, below = [], 0
    luma = [b for b in edge_blocks(rng, h, 3) if not b[0]]
    for _, x, y, bw, bh, _, _ in luma:
        size = bw
        for bip in (0, 1):
            sign = int(rng.integers(0, 2))
            mv = random_mv(rng, x, y, bw, bh, W, h, 0, sign)
            below += ((-mv[1] if sign else mv[1]) >> 2) > h - y
            mvs = (Mv * 4)(*[Mv(mv[0], mv[1])] * 4)
            bp = BlockPos(y, x, size, bw, bh, 128)
            ry, ru, rv = aligned((size, size), sdt(hbd)), aligned((size // 2, size // 2), sdt(hbd)), aligned((size // 2, size // 2), sdt(hbd))
            getattr(R, "get_inter_prediction_yuv_" + s)(C.byref(f.s), P(ry), P(ru), P(rv), C.byref(bp), mvs, sign, W, h, bip, 0, bd)
            oy = aligned((bh, bw), sdt(hbd))
            getattr(O, "orc_get_inter_prediction_luma_" + s)(P(oy), P(f.Y, f.origin(0) + y * f.sy + x), bw, bh, f.sy, bw, mv, sign, bip, W, h, x, y, bd)
            ok = (ry[:bh, :bw] == oy).all()
            for p, rp in ((1, ru), (2, rv)):
                oc = aligned((bh // 2, bw // 2), sdt(hbd))
                getattr(O, "orc_get_inter_prediction_chroma_" + s)(P(oc), P(f.full(p), f.origin(p) + y // 2 * f.sc + x // 2), bw // 2, bh // 2, f.sc, bw // 2, mv, sign,
                                                                   W // 2, h // 2, x // 2, y // 2, bd)
                ok = ok and (rp[:bh // 2, :bw // 2] == oc).all()
            if not ok:
                bad.append((bip, x, y, bw, bh, sign, mv[0], mv[1]))
    assert below >= len(luma) // 4, below
    assert not bad, (len(bad), bad[:6])
