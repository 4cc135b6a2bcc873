"""ctypes loaders + helpers shared by the tests (test infrastructure only).

oracle()   -> oracle/libthor_oracle.so  (our plain-C restatement; built on demand with `make -C oracle port`)
ref()      -> oracle/_ref/libthorref.so (the compiled, unmodified reference; None if not built/travelled)
ref_enc(h) -> oracle/_ref/libthorref_enc_{lbd,hbd}.so (file-static reference kernels via trampolines)
"""
import ctypes as C
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
_cache = {}


def oracle():
    if "o" not in _cache:
        so = os.path.join(ORACLE_DIR, "libthor_oracle.so")
        src = [os.path.join(ORACLE_DIR, f) for f in ("thor_oracle.c", "thor_oracle.h", "thor_oracle_tmpl.h")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in src):
            subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "port"])
        lib = C.CDLL(so)
        for n in ("orc_ssd_lbd", "orc_ssd_hbd", "orc_dist_8x8_lbd", "orc_dist_8x8_hbd"):
            getattr(lib, n).restype = C.c_uint64
        for n in ("orc_dct_matrix", "orc_zigzag"):
            getattr(lib, n).restype = C.c_void_p
        _cache["o"] = lib
    return _cache["o"]


def ref():
    if "r" not in _cache:
        so = os.path.join(ORACLE_DIR, "_ref", "libthorref.so")
        lib = None
        if os.path.exists(so):
            lib = C.CDLL(so, mode=C.RTLD_GLOBAL)
            C.c_int.in_dll(lib, "use_simd").value = 1
            for n in ("ssd_calc_simd_lbd", "ssd_calc_simd_hbd"):
                getattr(lib, n).restype = C.c_uint64
        _cache["r"] = lib
    return _cache["r"]


def ref_enc(hbd):
    k = "re%d" % hbd
    if k not in _cache:
        so = os.path.join(ORACLE_DIR, "_ref", "libthorref_enc_%s.so" % ("hbd" if hbd else "lbd"))
        lib = None
        if os.path.exists(so) and ref() is not None:
            lib = C.CDLL(so)
            sfx = "hbd" if hbd else "lbd"
            getattr(lib, "ref_ssd_calc_" + sfx).restype = C.c_uint64
            getattr(lib, "ref_set_use_simd_" + sfx)(1)
        _cache[k] = lib
    return _cache[k]


def aligned(shape, dtype, align=64, fill=None):
    dtype = np.dtype(dtype)
    n = int(np.prod(shape))
    raw = np.zeros(n * dtype.itemsize + align, dtype=np.uint8)
    off = (-raw.ctypes.data) % align
    a = raw[off:off + n * dtype.itemsize].view(dtype).reshape(shape)
    if fill is not None:
        a[...] = fill
    return a


def P(a, off=0):
    """pointer to element `off` (flat index) of numpy array a"""
    return C.c_void_p(a.ctypes.data + off * a.itemsize)


def sdt(hbd):
    return np.uint16 if hbd else np.uint8


def sfx(hbd):
    return "hbd" if hbd else "lbd"


def rand_plane(rng, h, w, bitdepth, hbd, smooth=False):
    """random sample plane, 64-byte aligned; smooth=True gives low-gradient content (forces SAD ties etc.)"""
    a = aligned((h, w), sdt(hbd))
    maxv = (1 << bitdepth) - 1
    if smooth:
        y, x = np.mgrid[0:h, 0:w]
        v = (np.sin(x / 7.0) + np.cos(y / 5.0)) * (maxv / 8.0) + maxv / 2.0 + rng.integers(-3, 4, (h, w))
        a[...] = np.clip(v, 0, maxv).astype(a.dtype)
    else:
        a[...] = rng.integers(0, maxv + 1, (h, w)).astype(a.dtype)
    return a


ME_EXT = 160 - 16  # clip_mv: a vector takes a block at most PADDING_Y - 16 samples outside the picture (common/inter_prediction.c:51-63)


def edge_search(rng, padded, fw, fh, size, width, height, sign, bitdepth):
    """A motion search at the picture's edges, for the block searches of `size` (clip_mv's block) predicting width x height.
    Returns (xpos, ypos, org, mvc, mvp, near): the block sits in the first or last block row or column or a corner, and org (size x size)
    copies the padded reference (a 2-D array with a 160-sample border) at a displacement beyond or just inside clip_mv's limit on one or both
    axes (+-0..20 samples), wholly right of or below the picture (split_mv's pic_w - xpos / pic_h - ypos clamp), or, for left-column blocks,
    more than `height` rows up (split_mv's -xpos - height bound).  The content there is border-replicated, so it is also found past the
    limit: the cost minimum lies where clip_mv does not let the search go.  mvc and mvp are quarter-pel vectors with `sign` applied; mvp
    either sits at the target or thousands of quarter-pels away (the long mv_len codes).  near(n) draws n whole-sample candidates around it."""
    lastx, lasty = (fw - size) // size * size, (fh - size) // size * size
    kind = int(rng.integers(0, 4))
    if kind == 3:  # left column, vertical vector beyond -height
        xpos, ypos = 0, int(rng.integers(0, fh // size)) * size
    else:
        while True:
            xpos = [0, lastx, int(rng.integers(0, fw // size)) * size][int(rng.integers(0, 3))]
            ypos = [0, lasty, int(rng.integers(0, fh // size)) * size][int(rng.integers(0, 3))]
            if xpos in (0, lastx) or ypos in (0, lasty):
                break

    def at_limit(pos, f):
        k = int(rng.integers(0, 21)) * int(rng.choice([-1, 1]))
        return (-ME_EXT - pos - k) if rng.integers(0, 2) else (f + ME_EXT - size - pos + k)

    def outside(pos, f, b):  # wholly past the far edge or more than b samples before the near one, within clip_mv's reach
        return int(rng.integers(f - pos + 1, f + ME_EXT - size - pos + 1)) if rng.integers(0, 2) else int(rng.integers(-ME_EXT - pos, -pos - b))

    free = lambda: int(rng.integers(-6, 7))
    if kind == 0:
        tx, ty = [(at_limit(xpos, fw), free()), (free(), at_limit(ypos, fh)), (at_limit(xpos, fw), at_limit(ypos, fh))][int(rng.integers(0, 3))]
    elif kind == 1:
        tx, ty = [(outside(xpos, fw, width), free()), (free(), outside(ypos, fh, height)), (outside(xpos, fw, width), at_limit(ypos, fh))][int(rng.integers(0, 3))]
    elif kind == 2:
        tx, ty = at_limit(xpos, fw), outside(ypos, fh, height)
    else:
        tx, ty = free(), -height - int(rng.integers(1, 48))
    # the border replicates the edge samples, so a source clamped into the 160-sample border holds the same block
    sy, sx = min(max(ypos + ty, -160), fh + 160 - size), min(max(xpos + tx, -160), fw + 160 - size)
    org = np.clip(padded[160 + sy:160 + sy + size, 160 + sx:160 + sx + size].astype(int) + rng.integers(-2, 3, (size, size)), 0, (1 << bitdepth) - 1)
    s = -1 if sign else 1
    mvc = [s * (4 * tx + int(rng.integers(-3, 4))), s * (4 * ty + int(rng.integers(-3, 4)))]
    far = lambda: int(rng.integers(-4000, 4001)) if rng.integers(0, 2) else 0
    mvp = [max(-32768, min(32767, s * 4 * tx + far())), max(-32768, min(32767, s * 4 * ty + far()))]
    near = lambda n: [[s * (tx + int(rng.integers(-4, 5))), s * (ty + int(rng.integers(-4, 5)))] for _ in range(n)]
    return xpos, ypos, org, mvc, mvp, near


def edge_reach(mvx, mvy, sign, xpos, ypos, fw, fh, size, width, height):
    """(on a clip limit, through an active split_mv clamp) for a search result: whether the vector lies within the sub-pel stages' reach
    (3 quarter-pels) of clip_mv's limit on either axis, and whether predicting the block with it clamps the integer offset
    (common/inter_prediction.c:121-131, lower bounds on xpos for both axes as in the reference)"""
    x, y = (-mvx, -mvy) if sign else (mvx, mvy)
    lims = ((xpos, x, -ME_EXT), (xpos, x, fw + ME_EXT - size), (ypos, y, -ME_EXT), (ypos, y, fh + ME_EXT - size))
    on_limit = any(abs(4 * (pos - lim) + v) <= 3 for pos, v, lim in lims)
    hi, vi = x >> 2, y >> 2
    return on_limit, hi > fw - xpos or hi < -xpos - width or vi > fh - ypos or vi < -xpos - height


def full_scale_planes(h, w, maxv):
    """reconstructions whose intra neighbours sit at 0 and 2^bd-1: uniform, and stripes that put one of the top row and left column at 2^bd-1 and
    alternate the other (the planar pre-filter's int16 input reaches 8 (2^bd-1), 32760 at 12 bits)"""
    yy, xx = np.mgrid[0:h, 0:w]
    return {"max": np.full((h, w), maxv), "zero": np.zeros((h, w), int), "odd rows": (yy % 2) * maxv, "even rows": (1 - yy % 2) * maxv,
            "odd cols": (xx % 2) * maxv, "even cols": (1 - xx % 2) * maxv}


def rdo_hostcheck():
    """oracle/librdo_hostcheck.so: tb_rdo.h over the plain-C oracle on the CPU (built by `make -C oracle port`, no reference sources needed).  It
    exports tb_rdo_encode_frame like libthor_b200.so, so it is loaded through its own handle and never RTLD_GLOBAL."""
    if "h" not in _cache:
        so = os.path.join(ORACLE_DIR, "librdo_hostcheck.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "port"])
        lib = C.CDLL(so, mode=C.RTLD_LOCAL)
        lib.tb_rdo_encode_frame.argtypes = [C.c_void_p]
        _cache["h"] = lib
    return _cache["h"]


def host_decisions(jobs, alloc, warps=1):
    """every job decided by rdo_hostcheck() into fresh RJ.HostFrame buffers, frame by frame, with `warps` simulated warps (TBR_HOST_WARPS)"""
    from thor_b200 import rdo_jobs as RJ
    lib = rdo_hostcheck()
    old = os.environ.get("TBR_HOST_WARPS")
    os.environ["TBR_HOST_WARPS"] = str(warps)
    try:
        hosts = [RJ.HostFrame(j, alloc) for j in jobs]
        for hf in hosts:
            assert lib.tb_rdo_encode_frame(C.byref(hf.desc)) == 0
    finally:
        if old is None:
            del os.environ["TBR_HOST_WARPS"]
        else:
            os.environ["TBR_HOST_WARPS"] = old
    return hosts


def host_decisions_of_dir(directory):
    """host_decisions() of the jobs in `directory`, as plain arrays for another process: [(check(), leaves, leaf_count, coeffs)] per frame"""
    import sys
    if ROOT not in sys.path:  # a spawned worker process
        sys.path.insert(0, ROOT)
    from thor_b200 import rdo_jobs as RJ
    keep = []

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    return [(hf.check(), hf.leaves.copy(), hf.leaf_count.copy(), hf.coeffs.copy()) for hf in host_decisions(RJ.load_jobs(directory), alloc)]


def ref_frame(hbd):
    """oracle/_ref/libthorref_frame_{lbd,hbd}.so: cdef_search + dist_8x8 trampolines (enc/encode_frame.c included in place)"""
    k = "rf%d" % hbd
    if k not in _cache:
        so = os.path.join(ORACLE_DIR, "_ref", "libthorref_frame_%s.so" % ("hbd" if hbd else "lbd"))
        lib = None
        if os.path.exists(so) and ref() is not None:
            lib = C.CDLL(so)
            getattr(lib, "ref_dist_8x8_" + ("hbd" if hbd else "lbd")).restype = C.c_uint64
        _cache[k] = lib
    return _cache[k]
