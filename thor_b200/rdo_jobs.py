"""RD-loop jobs (SURVEY.md §8f.1): the ctypes mirror of tb_rdo_frame_t (include/thor_b200.h) and the reader of the frame_NNN.job files the
reference-side shim writes (thor_b200/csrc/tb_rdo_shim.c, TB_RDO_DUMP): one file = the RD-loop inputs of one frame of a real encode
(parameters, source planes, padded reference planes) + what the reference's own process_block() decided (reconstruction before the in-loop
filters, per-4x4 block state, RD cost per super block).  No library is loaded here (bench.py's CPU arm imports this module too).
"""
import ctypes as C
import os

import numpy as np

TB_RDO_MAX_REF, TB_RDO_MAX_LEAVES, TB_RDO_SB_COEFFS = 8, 256, 24576


class RdoFrame(C.Structure):
    """tb_rdo_frame_t"""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("log2_sb_size", C.c_int32), ("bitdepth", C.c_int32), ("sample_bytes", C.c_int32),
                ("frame_type", C.c_int32), ("qp", C.c_int32), ("num_ref", C.c_int32), ("interp_ref", C.c_int32), ("num_intra_modes", C.c_int32),
                ("lambda_", C.c_double),
                ("enable_bipred", C.c_int32), ("enable_tb_split", C.c_int32), ("enable_pb_split", C.c_int32), ("encoder_speed", C.c_int32), ("intra_rdo", C.c_int32),
                ("use_block_contexts", C.c_int32), ("cfl_intra", C.c_int32), ("cfl_inter", C.c_int32),
                ("early_skip_thr", C.c_float),
                ("ref_sign", C.c_int32 * TB_RDO_MAX_REF), ("ref_sign_ge", C.c_int32 * TB_RDO_MAX_REF),
                ("orig", C.c_void_p * 3), ("orig_stride", C.c_int32 * 2),
                ("ref", (C.c_void_p * 3) * TB_RDO_MAX_REF), ("ref_stride", C.c_int32 * 2), ("ref_pad", C.c_int32),
                ("rec", C.c_void_p * 3), ("rec_stride", C.c_int32 * 2),
                ("blk", C.c_void_p), ("leaves", C.c_void_p), ("leaf_count", C.c_void_p), ("coeffs", C.c_void_p)]


RDO_BLK = np.dtype([("mode", "u1"), ("size", "u1"), ("tb_split", "u1"), ("pb_part", "u1"), ("cbp_y", "u1"), ("cbp_u", "u1"), ("cbp_v", "u1"), ("bipred_flag", "i1"),
                    ("mv0x", "i2"), ("mv0y", "i2"), ("mv1x", "i2"), ("mv1y", "i2"), ("ref_idx0", "u1"), ("ref_idx1", "u1"), ("pad", "u1", 2)])
RDO_LEAF = np.dtype([("xpos", "u2"), ("ypos", "u2"), ("size", "u1"), ("mode", "u1"), ("intra_mode", "u1"), ("skip_idx", "u1"), ("pb_part", "u1"), ("tb_split", "u1"),
                     ("ref_idx0", "u1"), ("ref_idx1", "u1"), ("dir", "i1"), ("cbp_y", "u1"), ("cbp_u", "u1"), ("cbp_v", "u1"), ("num_skip_vec", "u1"),
                     ("num_merge_vec", "u1"), ("ctx_index", "i1"), ("ctx_cbp", "i1"), ("mv_arr0", "i2", (4, 2)), ("mv_arr1", "i2", (4, 2)), ("mvp", "i2", 2),
                     ("coeff_ofs", "i4"), ("cost", "u4")])
assert RDO_BLK.itemsize == 20 and RDO_LEAF.itemsize == 64


def coeff_count(size, tb_split):
    """tb_rdo_coeff_count (include/thor_b200.h): int16 coefficients stored for one plane of a coded block"""
    t = size // 2 if tb_split else size
    q = min(t, 16)
    return (4 if tb_split else 1) * q * q


def leaf_coeffs(leaf, coeffs):
    """the quantised coefficients of one leaf (Y, then U, then V) inside its super block's coefficient area; empty when it has none"""
    ofs, size, split = int(leaf["coeff_ofs"]), int(leaf["size"]), int(leaf["tb_split"])
    if ofs < 0:
        return coeffs[:0]
    sc = size >> 1
    return coeffs[ofs:ofs + coeff_count(size, split) + 2 * coeff_count(sc, int(split and sc > 4))]


# Which leaf fields the reference's bit writer reads, per block mode (SKIP 0, INTRA 1, INTER 2, BIPRED 3, MERGE 4), with the lines of enc/write_bits.c that
# read them (write_super_mode :257-358, write_block :360-600; tb_rdo_shim.c emit_node hands every field to them).  Outside these modes a field holds
# whichever candidate state the deciding warp held last, so two correct decisions may differ there.  `dir` is not read by the bit writer at all.
ALL_MODES = (0, 1, 2, 3, 4)
LEAF_FIELD_MODES = {
    "xpos": ALL_MODES, "ypos": ALL_MODES, "size": ALL_MODES,   # emit_node matches the leaf to its quad-tree node by position and size
    "mode": ALL_MODES,                                          # :291-349 mode code
    "cost": ALL_MODES,                                          # not written: the RD cost the super block's decisions add up to
    "coeff_ofs": ALL_MODES,                                     # where emit_node unpacks coeff_y/u/v from (-1: none)
    "ctx_index": ALL_MODES,                                     # :284, :315, :344 mode code order
    "intra_mode": (1,),                                         # :395-401
    "pb_part": (2, 3),                                          # :405-406, :410-429 (INTER); :441-465 which mv_arr1 entries (BIPRED)
    "mv_arr0": (2, 3),                                          # :410-429 (INTER); :441-445 (BIPRED)
    "mv_arr1": (3,),                                            # :446-465
    "mvp": (2, 3),                                              # :409, :440
    "ref_idx0": (2, 3),                                         # :300-304, :324-333 (INTER); :467-474 (BIPRED in P frames)
    "ref_idx1": (3,),                                           # :467-474
    "skip_idx": (0, 4),                                         # :477-498
    "num_skip_vec": (0,),                                       # :479-486
    "num_merge_vec": (4,),                                      # :490-497
    "ctx_cbp": (1, 2, 3, 4),                                    # :522, :551
    "tb_split": (1, 2, 3, 4),                                   # :509, :530, :542-594
    "cbp_y": (1, 2, 3, 4), "cbp_u": (1, 2, 3, 4), "cbp_v": (1, 2, 3, 4),   # :513-540, :545-591
}
# the motion vectors write_mv codes per pb_part (PART_NONE, PART_HOR, PART_VER, PART_QUAD): :410-428 and :446-464; BIPRED codes mv_arr0[0] only (:441-442)
MV_ENTRIES = {0: (0,), 1: (0, 2), 2: (0, 1), 3: (0, 1, 2, 3)}


def leaf_differences(got_leaves, got_count, got_coeffs, want_leaves, want_count, want_coeffs, limit=8):
    """what the bit writer would code differently from `got` than from `want` (one frame): leaf counts per super block, the fields of
    LEAF_FIELD_MODES where the block's mode reads them, and the quantised coefficients each leaf references.  Returns up to `limit` descriptions
    (super block, leaf index, position, mode, field, got, want), first difference first; empty when the frames code identically."""
    out = []
    for s in range(len(want_count)):
        if got_count[s] != want_count[s]:
            out.append("sb %d: leaf_count %d, want %d" % (s, got_count[s], want_count[s]))
            if len(out) >= limit:
                return out
            continue
        for i in range(int(want_count[s])):
            g, w = got_leaves[s, i], want_leaves[s, i]
            mode = int(w["mode"])
            where = "sb %d leaf %d (x %d y %d size %d mode %d)" % (s, i, w["xpos"], w["ypos"], w["size"], mode)
            for name, modes in LEAF_FIELD_MODES.items():
                if mode not in modes:
                    continue
                gv, wv = g[name], w[name]
                if name in ("mv_arr0", "mv_arr1"):
                    pb = int(w["pb_part"])
                    idx = (0,) if (name == "mv_arr0" and mode == 3) else MV_ENTRIES.get(pb, MV_ENTRIES[3])
                    gv, wv = gv[list(idx)], wv[list(idx)]
                if not np.array_equal(gv, wv):
                    out.append("%s: %s %s, want %s" % (where, name, np.asarray(gv).tolist(), np.asarray(wv).tolist()))
            if int(w["coeff_ofs"]) >= 0 and int(g["coeff_ofs"]) == int(w["coeff_ofs"]):
                gc, wc = leaf_coeffs(w, got_coeffs[s]), leaf_coeffs(w, want_coeffs[s])
                if not np.array_equal(gc, wc):
                    k = int(np.flatnonzero(gc != wc)[0])
                    out.append("%s: coefficient %d of %d is %d, want %d" % (where, k, wc.size, gc[k], wc[k]))
            if len(out) >= limit:
                return out[:limit]
    return out


class Job:
    """one frame_NNN.job: .hdr (RdoFrame with NULL pointers), .frame_num, .nsb, .orig[3], .refs[r][3] (whole padded planes), and the reference's
    results .rec[3], .blk, .sb_cost"""

    def __init__(self, path):
        raw = np.fromfile(path, dtype=np.uint8)
        assert bytes(raw[:8]) == b"TBJOB1\0\0", "%s is not an RD-loop job file" % path
        o = 8
        self.hdr = RdoFrame.from_buffer_copy(raw[o:o + C.sizeof(RdoFrame)].tobytes()); o += C.sizeof(RdoFrame)
        self.frame_num, self.nsb = [int(v) for v in raw[o:o + 8].view(np.int32)]; o += 8
        h = self.hdr
        w, hh, esz = h.width, h.height, h.sample_bytes
        self.sdt = np.uint8 if esz == 1 else np.uint16

        def take(n_samples, shape):
            nonlocal o
            a = raw[o:o + n_samples * esz].view(self.sdt).reshape(shape); o += n_samples * esz
            return a
        dims = [(hh, w), (hh >> 1, w >> 1), (hh >> 1, w >> 1)]
        self.orig = [take(a * b, (a, b)) for a, b in dims]
        pad, padc = h.ref_pad, h.ref_pad >> 1
        self.refs = []
        for _ in range(h.num_ref):
            planes = []
            for p in range(3):
                st, pd = h.ref_stride[1 if p else 0], padc if p else pad
                rows = dims[p][0] + 2 * pd
                planes.append(take(st * rows, (rows, st)))
            self.refs.append(planes)
        self.rec = [take(a * b, (a, b)) for a, b in dims]
        nblk = (hh // 4) * (w // 4)
        self.blk = raw[o:o + nblk * RDO_BLK.itemsize].view(RDO_BLK); o += nblk * RDO_BLK.itemsize
        self.sb_cost = raw[o:o + 4 * self.nsb].view(np.int32); o += 4 * self.nsb
        assert o == raw.size, "%s: %d trailing bytes" % (path, raw.size - o)
        self.pixels = w * hh

    def in_bytes(self):
        return sum(p.nbytes for p in self.orig) + sum(p.nbytes for r in self.refs for p in r)

    def out_bytes(self):
        h = self.hdr
        return sum(p.nbytes for p in self.rec) + self.blk.nbytes + self.nsb * (TB_RDO_MAX_LEAVES * RDO_LEAF.itemsize + 4 + 2 * TB_RDO_SB_COEFFS)


def load_jobs(directory):
    return [Job(os.path.join(directory, f)) for f in sorted(os.listdir(directory)) if f.endswith(".job")]


class HostFrame:
    """host buffers of one job in memory from `alloc(nbytes) -> address` (pinned for the bench), and the tb_rdo_frame_t that points into them.
    share_inputs: another HostFrame whose input planes are reused (replicas of a job upload from the same host memory)."""

    def __init__(self, job, alloc, share_inputs=None):
        self.job = job
        h = job.hdr
        esz, w, hh = h.sample_bytes, h.width, h.height
        self._keep = []

        def buf(nbytes, dtype, shape):
            p = alloc(nbytes)
            a = np.frombuffer((C.c_uint8 * nbytes).from_address(p), dtype=dtype).reshape(shape)
            self._keep.append(a)
            return p, a
        d = RdoFrame.from_buffer_copy(bytes(h))
        pad, padc = h.ref_pad, h.ref_pad >> 1
        if share_inputs is None:
            self.orig_ptr, self.ref_ptr = [], []
            for p in range(3):
                ptr, a = buf(job.orig[p].nbytes, job.sdt, job.orig[p].shape); a[...] = job.orig[p]; self.orig_ptr.append(ptr)
            for r in range(h.num_ref):
                ptrs = []
                for p in range(3):
                    ptr, a = buf(job.refs[r][p].nbytes, job.sdt, job.refs[r][p].shape); a[...] = job.refs[r][p]
                    st, pd = h.ref_stride[1 if p else 0], padc if p else pad
                    ptrs.append(ptr + (pd * st + pd) * esz)  # sample (0,0)
                self.ref_ptr.append(ptrs)
        else:
            self.orig_ptr, self.ref_ptr = share_inputs.orig_ptr, share_inputs.ref_ptr
        for p in range(3):
            d.orig[p] = self.orig_ptr[p]
        d.orig_stride[0], d.orig_stride[1] = w, w >> 1
        for r in range(h.num_ref):
            for p in range(3):
                d.ref[r][p] = self.ref_ptr[r][p]
        self.rec = []
        for p in range(3):
            ptr, a = buf(job.rec[p].nbytes, job.sdt, job.rec[p].shape); a[...] = 0; d.rec[p] = ptr; self.rec.append(a)
        d.rec_stride[0], d.rec_stride[1] = w, w >> 1
        nblk, nsb = (hh // 4) * (w // 4), job.nsb
        ptr, self.blk = buf(nblk * RDO_BLK.itemsize, RDO_BLK, (nblk,)); d.blk = ptr
        ptr, self.leaves = buf(nsb * TB_RDO_MAX_LEAVES * RDO_LEAF.itemsize, RDO_LEAF, (nsb, TB_RDO_MAX_LEAVES)); d.leaves = ptr
        ptr, self.leaf_count = buf(4 * nsb, np.int32, (nsb,)); d.leaf_count = ptr
        ptr, self.coeffs = buf(2 * nsb * TB_RDO_SB_COEFFS, np.int16, (nsb, TB_RDO_SB_COEFFS)); d.coeffs = ptr
        self.desc = d

    def clear_outputs(self):
        for a in self.rec:
            a[...] = 0
        self.blk.view(np.uint8)[...] = 0
        self.leaf_count[...] = 0

    def check(self):
        """the device's decisions against the reference's: reconstruction, block state, RD cost per super block"""
        j = self.job
        rec_ok = all(np.array_equal(self.rec[p], j.rec[p]) for p in range(3))
        names = [n for n in RDO_BLK.names if n != "pad"]
        blk_ok = all(np.array_equal(self.blk[n], j.blk[n]) for n in names)
        cost = np.array([int(self.leaves["cost"][s, :self.leaf_count[s]].astype(np.int64).sum()) for s in range(j.nsb)], dtype=np.int64)
        cost_ok = np.array_equal(cost, j.sb_cost.astype(np.int64))
        return {"rec": bool(rec_ok), "blk": bool(blk_ok), "sb_cost": bool(cost_ok)}

    def leaf_differences(self, want, limit=8):
        """leaf_differences() of this frame's leaf lists and coefficients against those of `want`, a HostFrame of the same job"""
        return leaf_differences(self.leaves, self.leaf_count, self.coeffs, want.leaves, want.leaf_count, want.coeffs, limit)
