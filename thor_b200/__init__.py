"""thor_b200 — ctypes face of libthor_b200.so (the sm_90a CUDA implementation of the Thor per-block hot path).

This package is plumbing only: it loads the in-tree shared library built by thor_b200/build.py, declares the C ABI of
include/thor_b200.h, and offers numpy record dtypes for the work-item structs.  There is no CPU implementation here;
importing works without a GPU (so that symbol/ABI tests can run), but every compute entry point needs a CUDA device
and fails loudly otherwise (TB_ERR_CUDA from tb_*, abort() from the drop-in reference symbols).
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("THOR_B200_LIB") or os.path.join(_HERE, "libthor_b200.so")  # env override: A/B builds of the same sources

TB_OK, TB_ERR_CUDA, TB_ERR_ARG = 0, -1, -2


class ThorB200Error(RuntimeError):
    pass


def _load():
    if _build.stale() and not os.environ.get("THOR_B200_LIB"):
        try:
            _build.build()
        except Exception as e:  # no nvcc on this box: use the prebuilt library if there is one
            if not os.path.exists(LIB_PATH):
                raise ThorB200Error("libthor_b200.so is missing and could not be built: %s" % e)
    if not os.path.exists(LIB_PATH):
        raise ThorB200Error("libthor_b200.so not found at %s (run python thor_b200/build.py)" % LIB_PATH)
    return C.CDLL(LIB_PATH)


lib = _load()

from .records import *  # noqa: F401,F403  (work-item record layouts, must match include/thor_b200.h)
from .records import SAD_ITEM, ME_ITEM, ME_BI_ITEM, COMBINE_ITEM, ME_RESULT, INTERP_ITEM, TXFM_ITEM, TXFM_RESULT, TXFM_FAST, TXFM_BITS, INTRA_ITEM, BLKINFO  # noqa: F401

_vp, _i, _u64 = C.c_void_p, C.c_int, C.c_uint64
lib.tb_last_error.restype = C.c_char_p
lib.tb_launch_count.restype = _u64
lib.tb_stream.restype = _vp
lib.tb_malloc.restype = _vp
lib.tb_malloc.argtypes = [C.c_size_t]
lib.tb_free.argtypes = [_vp]
lib.tb_malloc_host.restype = _vp
lib.tb_malloc_host.argtypes = [C.c_size_t]
lib.tb_free_host.argtypes = [_vp]
lib.tb_memcpy_h2d.argtypes = [_vp, _vp, C.c_size_t]
lib.tb_memcpy_d2h.argtypes = [_vp, _vp, C.c_size_t]
lib.tb_memcpy_d2h_async.argtypes = [_vp, _vp, C.c_size_t]
lib.tb_memcpy_d2d.argtypes = [_vp, _vp, C.c_size_t]
lib.tb_set_stream.argtypes = [_vp]
lib.tb_frame_create.restype = _vp
lib.tb_frame_create.argtypes = [_i, _i, _i, _i]
lib.tb_frame_destroy.argtypes = [_vp]
lib.tb_frame_upload.argtypes = [_vp, _vp, _i, _vp, _vp, _i]
lib.tb_frame_download.argtypes = [_vp, _vp, _i, _vp, _vp, _i]
lib.tb_frame_download_async.argtypes = [_vp, _vp, _i, _vp, _vp, _i]
lib.tb_frame_plane.restype = _vp
lib.tb_frame_plane.argtypes = [_vp, _i, C.POINTER(_i)]
lib.tb_sad_batch.argtypes = [_vp, _i, _i, _i, _vp, _vp, _vp]
lib.tb_motion_estimate_batch.argtypes = [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp]
lib.tb_me_set_stats.argtypes = [_vp]
lib.tb_motion_estimate_bi_batch.argtypes = [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp]
lib.tb_block_combine_batch.argtypes = [_vp, _i, _i, _i, _i]
lib.tb_interp_batch.argtypes = [_vp, _i, _i, _i, _i]
lib.tb_txfm_chain_batch.argtypes = [_vp, _i, _i, _i, _vp]
lib.tb_intra_batch.argtypes = [_vp, _i, _i, _i]
lib.tb_deblock_frame.argtypes = [_vp, _vp, _i, _i]
lib.tb_clpf_frame.argtypes = [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i]
lib.tb_clpf_detect_frame.argtypes = [_vp, _vp, _vp, _i, _i, _i, _vp]
lib.tb_cdef_frame.argtypes = [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _i, _i]
lib.tb_cdef_search_mse.argtypes = [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]
lib.tb_pad_frame.argtypes = [_vp]
lib.tb_create_reference_frame.argtypes = [_vp, _vp]
lib.tb_scale_down2x2.argtypes = [_vp, _vp]
lib.tb_interpolate_frames.argtypes = [_vp, _vp, _vp, _i, _i]
lib.tb_quantize.argtypes = [_vp, _vp, _i, _i, _i]
lib.tb_dequantize.argtypes = [_vp, _vp, _i, _i]
lib.tb_improve_uv_prediction.argtypes = [_i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i]
for _s in ("lbd", "hbd"):
    getattr(lib, "ssd_calc_simd_" + _s).restype = _u64
    getattr(lib, "widesad_calc_simd_" + _s).restype = C.c_uint
    getattr(lib, "sad_calc_fasthalf_simd_" + _s).restype = C.c_uint
    getattr(lib, "sad_calc_fastquarter_simd_" + _s).restype = C.c_uint


def check(rc, what="thor_b200 call"):
    if rc != TB_OK:
        raise ThorB200Error("%s failed (%d): %s" % (what, rc, (lib.tb_last_error() or b"").decode()))


def init(device=-1):
    """Initialise CUDA for this process (device < 0: $LOCAL_RANK or 0).  Raises if no usable GPU: there is no CPU path."""
    check(lib.tb_init(device), "tb_init")


class DevBuf:
    """A raw HBM allocation with numpy upload/download helpers."""

    def __init__(self, nbytes):
        self.nbytes = int(nbytes)
        self.ptr = lib.tb_malloc(self.nbytes)
        if not self.ptr:
            raise ThorB200Error("tb_malloc(%d) failed: %s" % (nbytes, (lib.tb_last_error() or b"").decode()))

    @classmethod
    def from_array(cls, a):
        a = np.ascontiguousarray(a)
        b = cls(max(a.nbytes, 16))
        check(lib.tb_memcpy_h2d(b.ptr, a.ctypes.data, a.nbytes), "h2d")
        return b

    def upload(self, a):
        a = np.ascontiguousarray(a)
        check(lib.tb_memcpy_h2d(self.ptr, a.ctypes.data, a.nbytes), "h2d")

    def download(self, dtype, shape):
        out = np.empty(shape, dtype=dtype)
        check(lib.tb_memcpy_d2h(out.ctypes.data, self.ptr, out.nbytes), "d2h")
        return out

    def free(self):
        if self.ptr:
            lib.tb_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Frame:
    """An HBM-resident padded 4:2:0 frame (geometry of the reference's yuv_frame_t, common/common_frame.c:435-469)."""

    def __init__(self, width, height, sample_bytes=1, pad=160):
        self.width, self.height, self.sample_bytes, self.pad = width, height, sample_bytes, pad
        self.h = lib.tb_frame_create(width, height, pad, sample_bytes)
        if not self.h:
            raise ThorB200Error("tb_frame_create failed: %s" % (lib.tb_last_error() or b"").decode())
        self.dtype = np.uint8 if sample_bytes == 1 else np.uint16

    def upload(self, y, u=None, v=None):
        y = np.ascontiguousarray(y, self.dtype)
        u = None if u is None else np.ascontiguousarray(u, self.dtype)
        v = None if v is None else np.ascontiguousarray(v, self.dtype)
        check(lib.tb_frame_upload(self.h, y.ctypes.data, y.shape[1], None if u is None else u.ctypes.data, None if v is None else v.ctypes.data,
                                  0 if u is None else u.shape[1]), "frame upload")

    def download(self):
        y = np.empty((self.height, self.width), self.dtype)
        u = np.empty((self.height // 2, self.width // 2), self.dtype)
        v = np.empty_like(u)
        check(lib.tb_frame_download(self.h, y.ctypes.data, self.width, u.ctypes.data, v.ctypes.data, self.width // 2), "frame download")
        return y, u, v

    def plane(self, p):
        """(device pointer of sample (0,0), pitch in samples).  Pointers change after the in-loop filters swap planes."""
        st = C.c_int(0)
        ptr = lib.tb_frame_plane(self.h, p, C.byref(st))
        return ptr, st.value

    def destroy(self):
        if self.h:
            lib.tb_frame_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass
