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
