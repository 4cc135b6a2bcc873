"""ctypes mirrors of the reference structs the frame-level functions take (test infrastructure only).
Layouts follow /root/reference/common/types.h:58-80 (yuv_frame_t), :132-187 (mv_t, inter_pred_t, cbp_t,
cdef_strength(s), deblock_data_t)."""
import ctypes as C
import numpy as np
from _libs import aligned, sdt


class YuvFrame(C.Structure):
    _fields_ = [("y", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p)] + [
        (n, C.c_int) for n in ("width", "height", "stride_y", "stride_c", "offset_y", "offset_c", "pad_hor_y", "pad_hor_c",
                               "pad_ver_y", "pad_ver_c", "area_y", "area_c", "sub", "subsample", "frame_num", "bitdepth",
                               "input_bitdepth")]


class Mv(C.Structure):
    _fields_ = [("x", C.c_int16), ("y", C.c_int16)]


class InterPred(C.Structure):
    _fields_ = [("mv0", Mv), ("mv1", Mv), ("ref_idx0", C.c_uint32), ("ref_idx1", C.c_uint32), ("bipred_flag", C.c_uint32)]


class Cbp(C.Structure):
    _fields_ = [("y", C.c_int), ("u", C.c_int), ("v", C.c_int)]


class DeblockData(C.Structure):
    _fields_ = [("mode", C.c_int), ("cbp", Cbp), ("size", C.c_uint8), ("tb_split", C.c_uint8), ("pb_part", C.c_int),
                ("inter_pred", InterPred), ("inter_pred_arr", InterPred * 16)]


class CdefStrength(C.Structure):
    _fields_ = [("level", C.c_int), ("sec_strength", C.c_int), ("pri_damping", C.c_int), ("sec_damping", C.c_int)]


class CdefStrengths(C.Structure):
    _fields_ = [("dir", C.c_int * 64), ("var", C.c_int * 64), ("plane", CdefStrength * 2)]


assert C.sizeof(DeblockData) == 364

BLKINFO = np.dtype([("mode", "u1"), ("cbp_y", "u1"), ("size", "u1"), ("tb_split", "u1"), ("pb_part", "u1"), ("pad", "u1", 3),
                    ("mv0x", "i2"), ("mv0y", "i2"), ("mv1x", "i2"), ("mv1y", "i2")])
assert BLKINFO.itemsize == 16


class Frame:
    """A padded 4:2:0 frame with the reference's geometry (common/common_frame.c:435-469)."""

    def __init__(self, width, height, bitdepth=8, hbd=0, pad_hor=160, pad_ver=160):
        self.width, self.height, self.bitdepth, self.hbd = width, height, bitdepth, hbd
        self.ph, self.pv = pad_hor, pad_ver
        self.phc, self.pvc = pad_hor >> 1, pad_ver >> 1
        self.sy = (width + 2 * pad_hor + 15) & ~15
        self.sc = ((width >> 1) + 2 * self.phc + 15) & ~15
        dt = sdt(hbd)
        self.Y = aligned((height + 2 * pad_ver + 1, self.sy), dt)
        self.U = aligned(((height >> 1) + 2 * self.pvc + 1, self.sc), dt)
        self.V = aligned(((height >> 1) + 2 * self.pvc + 1, self.sc), dt)
        self.s = YuvFrame()
        isz = np.dtype(dt).itemsize
        self.s.y = self.Y.ctypes.data + (pad_ver * self.sy + pad_hor) * isz
        self.s.u = self.U.ctypes.data + (self.pvc * self.sc + self.phc) * isz
        self.s.v = self.V.ctypes.data + (self.pvc * self.sc + self.phc) * isz
        self.s.width, self.s.height = width, height
        self.s.stride_y, self.s.stride_c = self.sy, self.sc
        self.s.pad_hor_y, self.s.pad_ver_y, self.s.pad_hor_c, self.s.pad_ver_c = pad_hor, pad_ver, self.phc, self.pvc
        self.s.sub, self.s.subsample, self.s.bitdepth, self.s.input_bitdepth = 1, 420, bitdepth, bitdepth

    # views of the visible area
    @property
    def y(self): return self.Y[self.pv:self.pv + self.height, self.ph:self.ph + self.width]
    @property
    def u(self): return self.U[self.pvc:self.pvc + self.height // 2, self.phc:self.phc + self.width // 2]
    @property
    def v(self): return self.V[self.pvc:self.pvc + self.height // 2, self.phc:self.phc + self.width // 2]

    def plane(self, p): return (self.y, self.u, self.v)[p]
    def full(self, p): return (self.Y, self.U, self.V)[p]
    def origin(self, p):
        """flat element index of the visible area's (0,0) in full(p)"""
        return (self.pv * self.sy + self.ph) if p == 0 else (self.pvc * self.sc + self.phc)
    def stride(self, p): return self.sy if p == 0 else self.sc

    def randomize(self, rng, smooth=True):
        maxv = (1 << self.bitdepth) - 1
        for p in range(3):
            a = self.plane(p)
            h, w = a.shape
            if smooth:
                yy, xx = np.mgrid[0:h, 0:w]
                v = (np.sin(xx / 9.0 + p) + np.cos(yy / 6.0)) * (maxv / 6.0) + maxv / 2.0 + rng.integers(-12, 13, (h, w))
                # blocky steps so that deblocking / CDEF have edges to work on
                v += ((xx // 8 + yy // 8) % 3 - 1) * (maxv / 24.0)
                a[...] = np.clip(v, 0, maxv).astype(a.dtype)
            else:
                a[...] = rng.integers(0, maxv + 1, (h, w)).astype(a.dtype)

    def copy(self):
        f = Frame(self.width, self.height, self.bitdepth, self.hbd, self.ph, self.pv)
        f.Y[...] = self.Y; f.U[...] = self.U; f.V[...] = self.V
        return f


def random_blkinfo(rng, width, height, p_skip=0.3, root=64, mv_range=9):
    """A plausible random coding-block partition on the 4x4 grid: returns (numpy BLKINFO [h/4, w/4], DeblockData array).
    root: the largest coding block (64, or 128 for the encoder's super blocks); motion vectors lie within +-mv_range."""
    bw, bh = width // 4, height // 4
    bi = np.zeros((bh, bw), dtype=BLKINFO)
    for y0 in range(0, height, root):
        for x0 in range(0, width, root):
            def fill(x, y, size):
                if size > 8 and (rng.random() < 0.5 or x + size > width or y + size > height):
                    h = size // 2
                    for dy in (0, h):
                        for dx in (0, h):
                            if x + dx < width and y + dy < height:
                                fill(x + dx, y + dy, h)
                    return
                r = rng.random()
                mode = 0 if r < p_skip else int(rng.integers(1, 5))
                rec = np.zeros((), dtype=BLKINFO)
                rec["mode"] = mode
                rec["size"] = size
                rec["cbp_y"] = 0 if mode == 0 else int(rng.integers(0, 2))
                rec["tb_split"] = int(rng.integers(0, 2)) if mode != 0 else 0
                rec["pb_part"] = int(rng.integers(0, 4)) if mode in (2, 3) else 0
                if mode != 1:
                    rec["mv0x"], rec["mv0y"] = int(rng.integers(-mv_range, mv_range + 1)), int(rng.integers(-mv_range, mv_range + 1))
                    if mode == 3:
                        rec["mv1x"], rec["mv1y"] = int(rng.integers(-mv_range, mv_range + 1)), int(rng.integers(-mv_range, mv_range + 1))
                bi[y // 4:min(bh, (y + size) // 4), x // 4:min(bw, (x + size) // 4)] = rec
            fill(x0, y0, root)
    return bi, deblock_data(bi)


def deblock_data(bi):
    """the DeblockData array of a BLKINFO grid (the fields the in-loop filters read)"""
    flat = bi.reshape(-1)
    dd = (DeblockData * flat.size)()
    for i in range(flat.size):
        d, r = dd[i], flat[i]
        d.mode = int(r["mode"]); d.cbp.y = int(r["cbp_y"]); d.size = int(r["size"]); d.tb_split = int(r["tb_split"])
        d.pb_part = int(r["pb_part"])
        d.inter_pred.mv0.x, d.inter_pred.mv0.y = int(r["mv0x"]), int(r["mv0y"])
        d.inter_pred.mv1.x, d.inter_pred.mv1.y = int(r["mv1x"]), int(r["mv1y"])
    return dd
