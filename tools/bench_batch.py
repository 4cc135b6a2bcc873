#!/usr/bin/env python
"""bench.py — Thor per-block hot path on one GPU: encode-side hot-path throughput in Mpixel/s.

ONE STEP = one pass of the hot path over one inter frame's worth of work, in the quantities the reference's RD loop
generates for the chosen encoder configuration when no early termination fires (enc/encode_block.c:1835-2120, 2401-2565):
every coding block, every reference frame, the prediction-block motion searches per (block, reference) [a1,a2,a4,a5,a7],
the RD candidates' luma/chroma predictions [a7,a8], their residual -> DCT -> quant -> dequant -> inverse DCT ->
reconstruct -> SSD chains [a3,a10-a13], the intra predictors [a15], and the frame-level in-loop filters deblock ->
CDEF -> CLPF(+detect sums) -> reference copy + padding [a17-a20].  Work items are synthetic (seeded) but laid out exactly
as the reference lays them out; every kernel is the parity-tested one.

  --config hdb     1920x1080  8-bit  config_HDB_high_efficiency    (BASELINE.json configs[2], the headline; default)
  --config ldb     1920x1080  8-bit  config_LDB_low_complexity     (configs[1]: speed 2, 2 refs, no PB/TB split, no bipred, no CDEF)
  --config ra4k    3840x2160  8-bit  config_RA_high_efficiency     (configs[3])
  --config hdb10   1920x1080 10-bit  config_HDB16_high_efficiency  (configs[4]; --bitdepth 10 is an alias)

WHAT THIS NUMBER IS NOT: a complete encode.  The reference's serial RD control flow and bitstream writer run on the host
between these calls and are not part of the timed region; the dependency chain between neighbouring blocks is removed by
batching.  It is the throughput ceiling of the GPU hot path (the no-early-termination worst case: about the work the
reference does on noisy content, 2-3x what it does on the survey's synthetic clip), reported beside the SAME item lists
replayed through the reference's own CPU kernels on all host cores with a dynamic work queue (cpu_baseline / --impl reference).

PARITY: after timing, the search and transform-chain results the GPU produced on the FULL item lists are compared with the
CPU arm's results on the same lists ("parity" in the JSON line); a mismatch fails the run.

MULTI-GPU: frames shard across ranks (one frame per rank per step).  With N > 1 every step has a data plane inside the
timed region: rank 0 holds the N raw source frames in pinned host memory, uploads them and scatters them over NCCL; every
rank returns its frame's search decisions by an NCCL gather ("collective" in the JSON line).

  python bench.py --gpus 1 --steps 5 --warmup 3
  python bench.py --impl reference --steps 1 --warmup 0    (CPU arm: the reference's kernels on all host cores)
"""
import argparse
import ctypes as C
import importlib.util
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SQUARED_LAMBDA_QP = {32: 77.7672, 33: 98.6706, 34: 125.1926, 35: 158.8437}  # enc/encode_tables.c:29-36
CHROMA_QP = {32: 31, 33: 32, 34: 33, 35: 33}                                   # common/common_tables.c:67-72


class Cfg:
    """One BASELINE.json configuration: frame geometry + the encoder parameters that decide the work mix."""
    TABLE = {
        #        W     H    BD  config file                        nref speed bipred pb  tbs intra_rdo cdef qp
        "hdb":   (1920, 1080, 8, "config_HDB_high_efficiency",      4,   0,    1,     1,  1,  1,        1,   35),  # qp 32 + dqpB0 3
        "hdb10": (1920, 1080, 10, "config_HDB16_high_efficiency",   4,   0,    1,     1,  1,  1,        1,   34),  # qp 32 + dqpB0 2
        "ldb":   (1920, 1080, 8, "config_LDB_low_complexity",       2,   2,    0,     0,  0,  0,        0,   32),
        "ra4k":  (3840, 2160, 8, "config_RA_high_efficiency",       4,   0,    1,     1,  1,  1,        1,   35),
    }

    def __init__(self, name):
        self.name = name
        (self.W, self.H, self.BD, self.cfgfile, self.NREF, self.speed, self.bipred, self.pb_split, self.tb_split, self.intra_rdo, self.cdef,
         self.QP) = self.TABLE[name]
        self.ESZ = 1 if self.BD == 8 else 2
        self.SDT = np.uint8 if self.BD == 8 else np.uint16
        self.QPC = CHROMA_QP[self.QP]
        self.LAMBDA = (1.2 * SQUARED_LAMBDA_QP[self.QP]) ** 0.5  # sqrt(lambda_coeff * squared_lambda_QP[qp]) as passed to motion_estimate (encode_block.c:1981)
        self.NCAND = 8  # candidate MVs per (block, reference) (frame_info->mvcand grows up to 64 inside an SB)
        # coding-block sizes evaluated by mode_decision_rdo: "size < 128 || encoder_speed == 0" (encode_block.c:1912)
        self.SIZES = (8, 16, 32, 64, 128) if self.speed == 0 else (8, 16, 32, 64)
        # prediction blocks searched per (coding block, reference): PART_NONE [+ 2 HOR + 2 VER + 4 QUAD] (encode_block.c:1033-1098)
        self.PBS = PBS if self.pb_split else PBS[:1]
        # transform evaluations per coding block (mode_decision_rdo + encode_block):
        #   high efficiency: 31 unsplit + 30 tb_split (round 1's derivation: merge 2x2, inter 4 refs x 4 parts x {0-residual, unsplit, split},
        #                    bipred, intra 10 modes x 2 + final)
        #   low complexity : merge 2 + inter 2 refs (tb_param 0 only at speed >= 1) + final intra = 5 unsplit, no split
        self.N_UNSPLIT, self.N_SPLIT = (31, 30) if self.tb_split else (5, 0)
        self.PIXELS = self.W * self.H

    def describe(self, counts):
        return ("%dx%d %d-bit 4:2:0, %s hot-path batch for ONE inter frame per step: %d motion searches (blocks %d..%d x %d refs x %d PBs, speed %d%s), "
                "%d candidate predictions, %d DCT/quant/recon chains, %d intra predictions, deblock%s+CLPF(+detect)+reference pad; dependency-free "
                "batching, no early termination (not a complete encode)" %
                (self.W, self.H, self.BD, self.cfgfile, counts[0], self.SIZES[0], self.SIZES[-1], self.NREF, len(self.PBS), self.speed,
                 ", bipred taps" if self.bipred else "", counts[1], counts[2], counts[3], "+CDEF" if self.cdef else ""))


# the nine prediction blocks searched per (coding block, reference): PART_NONE, 2x HOR, 2x VER, 4x QUAD
# (search_inter_prediction_params, enc/encode_block.c:1033-1098) as (wnum, hnum, ox, oy) in halves of the block size
PBS = [(2, 2, 0, 0), (2, 1, 0, 0), (2, 1, 0, 1), (1, 2, 0, 0), (1, 2, 1, 0), (1, 1, 0, 0), (1, 1, 1, 0), (1, 1, 0, 1), (1, 1, 1, 1)]


def load_records():
    """record dtypes of include/thor_b200.h WITHOUT importing the package (which would dlopen libthor_b200.so): the CPU arm must not
    load the CUDA library"""
    spec = importlib.util.spec_from_file_location("thor_b200_records", os.path.join(ROOT, "thor_b200", "records.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


# ----------------------------------------------------------------------------------------------------------------------
# workload construction (host, numpy, seeded) — ONE function for the GPU arm and the CPU arm: the same seed gives the same
# lists (the random draws do not depend on the pointers bound into the items)
# ----------------------------------------------------------------------------------------------------------------------
def synth_frames(cfg, seed, n):
    """moving 8x8-block texture + low-frequency sinusoids + N(0,3) noise (SURVEY.md §8d synthetic input), 4:2:0"""
    rng = np.random.default_rng([seed, 1])
    W, H, BD = cfg.W, cfg.H, cfg.BD
    yy, xx = np.mgrid[0:H + 64, 0:W + 64]
    tex = rng.integers(0, 64, ((H + 64) // 8 + 1, (W + 64) // 8 + 1)).astype(np.float32)
    base = np.kron(tex, np.ones((8, 8), np.float32))[:H + 64, :W + 64] + 60 * np.sin(xx / 97.0) + 50 * np.cos(yy / 61.0) + 96
    frames = []
    for k in range(n):
        dy, dx = 2 * k, 3 * k
        sc, mx = 1 << (BD - 8), (1 << BD) - 1
        y = np.clip((base[dy:dy + H, dx:dx + W] + rng.normal(0, 3, (H, W))) * sc, 0, mx).astype(cfg.SDT)
        u = np.clip((128 + 30 * np.sin(xx[:H // 2, :W // 2] / 53.0 + k) + rng.normal(0, 2, (H // 2, W // 2))) * sc, 0, mx).astype(cfg.SDT)
        v = np.clip((128 + 30 * np.cos(yy[:H // 2, :W // 2] / 47.0 - k) + rng.normal(0, 2, (H // 2, W // 2))) * sc, 0, mx).astype(cfg.SDT)
        frames.append((y, u, v))
    return frames


def block_grid(cfg):
    """(size, xpos, ypos) of every square coding block fully inside the frame (process_block recursion), sizes ascending"""
    out = []
    for s in cfg.SIZES:
        xs = np.arange(0, cfg.W - s + 1, s); ys = np.arange(0, cfg.H - s + 1, s)
        gx, gy = np.meshgrid(xs, ys)
        out.append(np.stack([np.full(gx.size, s), gx.ravel(), gy.ravel()], axis=1))
    return np.concatenate(out).astype(np.int32)


def pb_geometry(cfg, blocks):
    npb, nb = len(cfg.PBS), len(blocks)
    size = np.repeat(blocks[:, 0], cfg.NREF * npb); xpos = np.repeat(blocks[:, 1], cfg.NREF * npb); ypos = np.repeat(blocks[:, 2], cfg.NREF * npb)
    ref = np.tile(np.repeat(np.arange(cfg.NREF), npb), nb)
    pb = np.tile(np.arange(npb), nb * cfg.NREF)
    pbt = np.array(cfg.PBS); half = size // 2
    return size, xpos, ypos, ref, pbt[pb, 0] * half, pbt[pb, 1] * half, pbt[pb, 2] * half, pbt[pb, 3] * half


def build_me(cfg, R, blocks, cur, refs, rng):
    """cur = (ptr, stride) of the luma plane; refs = [(ptr, stride)] per reference"""
    nb, npb, ESZ = len(blocks), len(cfg.PBS), cfg.ESZ
    size, xpos, ypos, ref, bw, bh, ox, oy = pb_geometry(cfg, blocks)
    n = len(size)
    items = np.zeros(n, R.ME_ITEM)
    refp = np.asarray([r[0] for r in refs], np.uint64)[ref]
    cur_st, ref_st = cur[1], refs[0][1]
    items["orig"] = np.uint64(cur[0]) + ((ypos + oy).astype(np.uint64) * np.uint64(cur_st) + (xpos + ox).astype(np.uint64)) * np.uint64(ESZ)
    items["ref"] = refp + ((ypos + oy).astype(np.uint64) * np.uint64(ref_st) + (xpos + ox).astype(np.uint64)) * np.uint64(ESZ)
    items["ostride"] = cur_st; items["rstride"] = ref_st
    items["xpos"] = xpos; items["ypos"] = ypos; items["size"] = size; items["width"] = bw; items["height"] = bh
    items["sign"] = (ref == cfg.NREF - 1) if cfg.bipred else 0  # one future reference, as in B frames
    grp = np.repeat(np.arange(nb * cfg.NREF), npb)  # one (block, ref) group shares centre, predictor and candidate list
    mvg = rng.integers(-24, 25, (nb * cfg.NREF, 4)).astype(np.int16)
    items["mvc_x"] = mvg[grp, 0]; items["mvc_y"] = mvg[grp, 1]; items["mvp_x"] = mvg[grp, 2]; items["mvp_y"] = mvg[grp, 3]
    items["cand_ofs"] = grp * cfg.NCAND; items["ncand"] = cfg.NCAND; items["lambda"] = cfg.LAMBDA
    cands = rng.integers(-12, 13, (nb * cfg.NREF * cfg.NCAND, 2)).astype(np.int16)
    return items, cands


def tu_list(cfg, blocks):
    """Transform blocks evaluated per coding block (mode_decision_rdo + encode_block, enc/encode_block.c:1340-1493, 1835-2120):
    N_UNSPLIT unsplit evaluations (luma size s, 2 chroma s/2) and N_SPLIT tb_split evaluations (4 luma s/2, 8 chroma s/4)."""
    rows = []
    for s in cfg.SIZES:
        b = blocks[blocks[:, 0] == s]

        def add(count, tsize, chroma, sub):
            if tsize < 4 or count == 0:
                return
            k = np.arange(sub * sub)  # sub x sub transform blocks tile the coding block (in the TU's own plane)
            tx = (k % sub) * tsize; ty = (k // sub) * tsize
            bx = (b[:, 1] >> chroma)[:, None] + tx[None, :]; by = (b[:, 2] >> chroma)[:, None] + ty[None, :]
            r = np.stack([np.full(bx.size, tsize), bx.ravel(), by.ravel(), np.full(bx.size, chroma)], axis=1)
            rows.append(np.tile(r, (count, 1)))
        add(cfg.N_UNSPLIT, s, 0, 1); add(2 * cfg.N_UNSPLIT, s // 2, 1, 1)
        add(cfg.N_SPLIT, s // 2, 0, 2); add(2 * cfg.N_SPLIT, s // 4, 1, 2)
    return np.concatenate(rows).astype(np.int32)


def build_txfm(cfg, R, tus, planes_cur, planes_ref, rec_ptr, rng):
    n, ESZ = len(tus), cfg.ESZ
    size, x, y, chroma = tus[:, 0], tus[:, 1], tus[:, 2], tus[:, 3]
    items = np.zeros(n, R.TXFM_ITEM)
    cp = np.array([planes_cur[0][0], planes_cur[1][0]], np.uint64)[chroma]; cs = np.array([planes_cur[0][1], planes_cur[1][1]])[chroma]
    rp = np.array([planes_ref[0][0], planes_ref[1][0]], np.uint64)[chroma]; rs = np.array([planes_ref[0][1], planes_ref[1][1]])[chroma]
    dx = rng.integers(-3, 4, n); dy = rng.integers(-3, 4, n)  # prediction = displaced reference block
    items["orig"] = cp + (y.astype(np.uint64) * cs.astype(np.uint64) + x.astype(np.uint64)) * np.uint64(ESZ)
    items["pred"] = (rp.astype(np.int64) + ((y + dy).astype(np.int64) * rs + (x + dx)) * ESZ).astype(np.uint64)
    if rec_ptr is not None:  # every candidate reconstructs into a block of its own: the kernel reads it back for the SSD
        ofs = np.concatenate([[0], np.cumsum(size.astype(np.int64) ** 2)[:-1]]).astype(np.uint64)
        items["rec"] = np.uint64(rec_ptr) + ofs * np.uint64(ESZ)
        items["rstride"] = size
    # else rec = NULL: the CPU replay reconstructs into a private scratch block per thread
    items["coeffq"] = 0
    items["ostride"] = cs; items["pstride"] = rs
    items["size"] = size; items["qp"] = np.where(chroma == 1, cfg.QPC, cfg.QP)
    items["coeff_type"] = rng.integers(0, 2, n) * 2 + chroma
    items["fast"] = 1 if cfg.speed > 1 else 0  # TB_TXFM_FAST: 16-point transform for 32x32 (common/transform.c:252)
    return items


def interp_geometry(cfg, blocks):
    size, xpos, ypos, ref, bw, bh, ox, oy = pb_geometry(cfg, blocks)
    parts, total = [], 0
    for plane in range(3):
        c = 1 if plane else 0
        w_, h_ = bw >> c, bh >> c
        keep = (w_ >= (2 if c else 4)) & (h_ >= (2 if c else 4))
        area = (w_[keep] * h_[keep]).astype(np.int64)
        start = total + np.concatenate([[0], np.cumsum(area)[:-1]])
        total += int(area.sum())
        parts.append((plane, c, keep, w_[keep], h_[keep], ((xpos + ox)[keep]) >> c, ((ypos + oy)[keep]) >> c, ref[keep], start))
    return parts, total, len(size)


def build_interp(cfg, R, blocks, ref_planes, out_ptr, rng):
    """predictions of the inter RD candidates: per (block, ref): the prediction blocks, luma + U + V"""
    parts, total, n_pb = interp_geometry(cfg, blocks)
    mv = rng.integers(-40, 41, (n_pb, 2))
    out = []
    for plane, c, keep, w_, h_, px, py, ref, start in parts:
        it = np.zeros(len(w_), R.INTERP_ITEM)
        ptrs = np.array([ref_planes[r][plane][0] for r in range(cfg.NREF)], np.uint64)[ref]
        st = ref_planes[0][plane][1]
        it["ref"] = ptrs + (py.astype(np.uint64) * np.uint64(st) + px.astype(np.uint64)) * np.uint64(cfg.ESZ)
        it["dst"] = np.uint64(out_ptr) + start.astype(np.uint64) * np.uint64(cfg.ESZ)
        it["rstride"] = st; it["dstride"] = w_
        it["xpos"] = px; it["ypos"] = py; it["mvx"] = mv[keep, 0]; it["mvy"] = mv[keep, 1]
        it["width"] = w_; it["height"] = h_; it["sign"] = (ref == cfg.NREF - 1) if cfg.bipred else 0; it["chroma"] = c
        it["pic_w"] = cfg.W >> c; it["pic_h"] = cfg.H >> c
        out.append(it)
    return np.concatenate(out)


def intra_geometry(cfg, blocks):
    """10 modes on the block and (intra_rdo = 1 with tb_split) on its four tb_split quadrants (enc/encode_block.c:2073-2114)"""
    rows = []
    for s in cfg.SIZES:
        b = blocks[blocks[:, 0] == s]
        for (ts, sub) in ((s, 1), (s // 2, 2)) if (cfg.intra_rdo and cfg.tb_split) else ((s, 1),):
            if ts < 4:
                continue
            k = np.arange(sub * sub)
            bx = b[:, 1][:, None] + (k % sub)[None, :] * ts; by = b[:, 2][:, None] + (k // sub)[None, :] * ts
            r = np.stack([np.full(bx.size, ts), bx.ravel(), by.ravel()], axis=1)
            rows.append(np.repeat(r, 10, axis=0))
    r = np.concatenate(rows)
    return r, int((r[:, 0].astype(np.int64) ** 2).sum())


def build_intra(cfg, R, blocks, rec, out_ptr):
    r, total = intra_geometry(cfg, blocks)
    n = len(r)
    items = np.zeros(n, R.INTRA_ITEM)
    size, x, y = r[:, 0], r[:, 1], r[:, 2]
    area = (size * size).astype(np.int64)
    start = np.concatenate([[0], np.cumsum(area)[:-1]])
    items["rec"] = np.uint64(rec[0]) + (y.astype(np.uint64) * np.uint64(rec[1]) + x.astype(np.uint64)) * np.uint64(cfg.ESZ)
    items["dst"] = np.uint64(out_ptr) + start.astype(np.uint64) * np.uint64(cfg.ESZ)
    items["rstride"] = rec[1]; items["xpos"] = x; items["ypos"] = y; items["size"] = size
    items["mode"] = np.tile(np.arange(10), n // 10)
    items["upright"] = ((y > 0) & (x + size < cfg.W)); items["downleft"] = ((x > 0) & (y + size < cfg.H))
    return items


def build_blkinfo(cfg, R, rng):
    W, H = cfg.W, cfg.H
    bi = np.zeros((H // 4, W // 4), R.BLKINFO)

    def fill(x, y, s):  # random quad-tree: 64x64 leaves split with p=0.6 down to 8x8
        if s > 8 and (rng.random() < 0.6 or x + s > W or y + s > H):
            for dy in (0, s // 2):
                for dx in (0, s // 2):
                    if x + dx < W and y + dy < H:
                        fill(x + dx, y + dy, s // 2)
            return
        mode = 0 if rng.random() < 0.3 else int(rng.integers(1, 5))
        rec = np.zeros((), R.BLKINFO)
        rec["mode"] = mode; rec["size"] = s; rec["cbp_y"] = 0 if mode == 0 else int(rng.integers(0, 2))
        rec["tb_split"] = int(rng.integers(0, 2)) if mode else 0
        rec["pb_part"] = int(rng.integers(0, 4)) if mode in (2, 3) else 0
        if mode != 1:
            rec["mv0x"], rec["mv0y"] = int(rng.integers(-9, 10)), int(rng.integers(-9, 10))
        bi[y // 4:min(H // 4, (y + s) // 4), x // 4:min(W // 4, (x + s) // 4)] = rec
    for y0 in range(0, H, 64):
        for x0 in range(0, W, 64):
            fill(x0, y0, 64)
    return bi


class Workload:
    """Everything one step needs, built from (cfg, seed) only; `bind` supplies the buffer addresses of the arm."""

    def __init__(self, cfg, R, seed):
        self.cfg, self.R, self.seed = cfg, R, seed
        self.blocks = block_grid(cfg)
        self.tus = tu_list(cfg, self.blocks)
        _, self.ip_total, _ = interp_geometry(cfg, self.blocks)
        _, self.in_total = intra_geometry(cfg, self.blocks)

    def bind(self, cur_planes, ref_planes, rec_plane0, cand_rec_ptr, pred_ptr, intra_ptr):
        """cur_planes: [(ptr, stride)] x 2 (Y, U); ref_planes: [[(ptr, stride)] x 3] x NREF; rec_plane0: (ptr, stride); cand_rec_ptr:
        tx_samples() samples for the candidates' reconstructions, or None"""
        cfg, R = self.cfg, self.R
        rng = np.random.default_rng([self.seed, 2])
        self.me, self.cands = build_me(cfg, R, self.blocks, cur_planes[0], [r[0] for r in ref_planes], rng)
        self.tx = build_txfm(cfg, R, self.tus, cur_planes, [ref_planes[0][0], ref_planes[0][1]], cand_rec_ptr, rng)
        self.ip = build_interp(cfg, R, self.blocks, ref_planes, pred_ptr, rng)
        self.intra = build_intra(cfg, R, self.blocks, rec_plane0, intra_ptr)
        self.bi = build_blkinfo(cfg, R, rng)
        nfb = ((cfg.W + 63) // 64) * ((cfg.H + 63) // 64)
        self.pri = rng.integers(0, 16, (2, nfb)).astype(np.int8); self.sec = rng.integers(0, 4, (2, nfb)).astype(np.int8)
        return self

    def counts(self):
        return len(self.me), len(self.ip), len(self.tx), len(self.intra)

    def tx_samples(self):
        return int((self.tus[:, 0].astype(np.int64) ** 2).sum())

    def txfm_alg_bytes(self):
        """SURVEY.md §8d for the chain: orig + pred read, rec written (3 N^2 s) + the 48-byte item + the 16-byte result"""
        n2 = (self.tx["size"].astype(np.int64) ** 2).sum()
        return int(3 * n2 * self.cfg.ESZ + len(self.tx) * (self.R.TXFM_ITEM.itemsize + self.R.TXFM_RESULT.itemsize))


# ----------------------------------------------------------------------------------------------------------------------
# clocks sampling
# ----------------------------------------------------------------------------------------------------------------------
class ClockSampler:
    """SM clock and throttle reasons sampled DURING the timed region: NVML from a thread every 5 ms (nvidia-smi -lms as fallback)."""
    REASONS = ((0x8, "hw_slowdown"), (0x40, "hw_thermal_slowdown"), (0x20, "sw_thermal_slowdown"), (0x4, "sw_power_cap"))

    def __init__(self, index=0):
        self.sm, self.mx, self.reasons, self.index = [], [], set(), index
        self.proc, self.thread, self.stop_flag, self.nvml = None, None, threading.Event(), None

    def _nvml_loop(self):
        import pynvml as nv
        h = self.nvml
        while not self.stop_flag.is_set():
            try:
                self.sm.append(int(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)))
                mask = int(nv.nvmlDeviceGetCurrentClocksThrottleReasons(h))
                for bit, name in self.REASONS:
                    if mask & bit:
                        self.reasons.add(name)
            except Exception:
                pass
            time.sleep(0.005)

    def start(self):
        try:
            import pynvml as nv
            nv.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(vis.split(",")[self.index]) if vis and all(t.strip().isdigit() for t in vis.split(",")) else self.index
            self.nvml = nv.nvmlDeviceGetHandleByIndex(phys)
            self.mx.append(int(nv.nvmlDeviceGetMaxClockInfo(self.nvml, nv.NVML_CLOCK_SM)))
            self.thread = threading.Thread(target=self._nvml_loop, daemon=True); self.thread.start()
            return
        except Exception:
            self.nvml = None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,"
                                          "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap",
                                          "--format=csv,noheader,nounits", "-lms", "50"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._smi_read, daemon=True); self.thread.start()
        except Exception:
            self.proc = None

    def _smi_read(self):
        names = [n for _, n in self.REASONS]
        for line in self.proc.stdout:
            r = [c.strip() for c in line.split(",")]
            if r and r[0].isdigit():
                self.sm.append(int(r[0]))
            if len(r) > 1 and r[1].isdigit():
                self.mx.append(int(r[1]))
            for i in range(4):
                if len(r) >= 6 and r[2 + i].lower().startswith("active"):
                    self.reasons.add(names[i])

    def stop(self):
        self.stop_flag.set()
        if self.proc:
            self.proc.terminate()
        if self.thread:
            self.thread.join(timeout=1.0)
        return {"sm_mhz": int(np.median(self.sm)) if self.sm else None, "sm_max_mhz": max(self.mx) if self.mx else None, "reasons": sorted(self.reasons),
                "samples": len(self.sm), "source": "nvml" if self.nvml is not None else "nvidia-smi"}


def metric_name(cfg):
    return "encode hot-path Mpixels/s (%dp %s work mix, batched; host RD control flow excluded)" % (cfg.H, cfg.cfgfile.replace("config_", ""))


# ----------------------------------------------------------------------------------------------------------------------
# GPU arm
# ----------------------------------------------------------------------------------------------------------------------
def run_gpu(args, cfg):
    import torch
    import torch.distributed as dist
    import thor_b200 as tb

    W, H, BD, ESZ, NREF, QP = cfg.W, cfg.H, cfg.BD, cfg.ESZ, cfg.NREF, cfg.QP
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1)); local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    tb.init(local)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    tb.check(tb.lib.tb_set_stream(C.c_void_p(stream.cuda_stream)))
    L = tb.lib
    seed = 2026 + rank  # every rank encodes its own frame (frames shard across ranks)

    # ---- resident frames: current, NREF references (padded), reconstruction + scratch + "original" for the filters
    fr = synth_frames(cfg, seed, NREF + 1)
    cur = tb.Frame(W, H, ESZ); cur.upload(*fr[0])
    refs = []
    tmp = tb.Frame(W, H, ESZ)
    for k in range(NREF):
        tmp.upload(*fr[k + 1])
        r = tb.Frame(W, H, ESZ)
        tb.check(L.tb_create_reference_frame(r.h, tmp.h))
        refs.append(r)
    pristine = tb.Frame(W, H, ESZ); pristine.upload(*fr[1])  # un-filtered reconstruction, restored device-side every step
    rec = tb.Frame(W, H, ESZ); rec.upload(*fr[1]); scratch = tb.Frame(W, H, ESZ); newref = tb.Frame(W, H, ESZ)

    wl = Workload(cfg, tb, seed)
    pred_buf = tb.DevBuf(wl.ip_total * ESZ + 64); intra_buf = tb.DevBuf(wl.in_total * ESZ + 64)
    cand_rec = tb.DevBuf(wl.tx_samples() * ESZ)  # where RD candidates write their reconstructions
    wl.bind([cur.plane(0), cur.plane(1)], [[r.plane(p) for p in range(3)] for r in refs], rec.plane(0), cand_rec.ptr, pred_buf.ptr, intra_buf.ptr)
    me_items, cands, tx_items, ip_items, in_items = wl.me, wl.cands, wl.tx, wl.ip, wl.intra
    nfb = ((W + 63) // 64) * ((H + 63) // 64)

    d_me = tb.DevBuf.from_array(me_items); d_cand = tb.DevBuf.from_array(cands); d_me_out = tb.DevBuf(8 * len(me_items))
    d_tx = tb.DevBuf.from_array(tx_items); d_tx_out = tb.DevBuf(16 * len(tx_items))
    d_ip = tb.DevBuf.from_array(ip_items); d_in = tb.DevBuf.from_array(in_items)
    d_bi = tb.DevBuf.from_array(wl.bi)
    d_pri = [tb.DevBuf.from_array(wl.pri[k]) for k in range(2)]; d_sec = [tb.DevBuf.from_array(wl.sec[k]) for k in range(2)]
    d_dv = tb.DevBuf(nfb * 2 * 64 * 4); d_sums = tb.DevBuf(16 * (W // 8) * (H // 8))
    resident_bytes = sum(b.nbytes for b in (d_me, d_cand, d_me_out, d_tx, d_tx_out, d_ip, d_in, pred_buf, intra_buf))

    # pinned host staging for the end-to-end leg
    def pinned(a):
        p = L.tb_malloc_host(a.nbytes)
        buf = (C.c_uint8 * a.nbytes).from_address(p)
        arr = np.frombuffer(buf, dtype=np.uint8)
        arr[...] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        return p, a.nbytes

    def pinned_view(p, dtype, n):
        return np.frombuffer((C.c_uint8 * (np.dtype(dtype).itemsize * n)).from_address(p), dtype=dtype)
    h_y, h_u, h_v = [pinned(p)[0] for p in fr[0]]
    h_me, me_bytes = pinned(me_items); h_cand, cand_bytes = pinned(cands)
    h_me_out = L.tb_malloc_host(8 * len(me_items)); h_tx_out = L.tb_malloc_host(16 * len(tx_items))
    h_rec = [L.tb_malloc_host(W * H * ESZ), L.tb_malloc_host(W * H // 4 * ESZ), L.tb_malloc_host(W * H // 4 * ESZ)]

    ev = lambda: torch.cuda.Event(enable_timing=True)
    me_ev, tx_ev, coll_ev = [], [], []
    TXF = 0  # TB_TXFM_* flags live in the items

    # ---- multi-GPU data plane (N > 1): rank 0 owns the raw source frames of ALL ranks in pinned host memory; each step it uploads them and
    # scatters them over NCCL; every rank returns its frame's search decisions (8 bytes per search) by an NCCL gather
    frame_elems = W * H * 3 // 2
    tdt = torch.uint8 if ESZ == 1 else torch.int16
    if world > 1:
        recv_yuv = torch.empty(frame_elems, dtype=tdt, device="cuda")
        me_out_t = torch.empty(8 * len(me_items), dtype=torch.uint8, device="cuda")
        if rank == 0:
            srcs = []
            for r in range(world):
                f0 = fr[0] if r == 0 else synth_frames(cfg, 2026 + r, 1)[0]
                srcs.append(torch.from_numpy(np.concatenate([p.reshape(-1) for p in f0]).view(np.uint8 if ESZ == 1 else np.int16)).pin_memory())
            scat = [torch.empty(frame_elems, dtype=tdt, device="cuda") for _ in range(world)]
            gath = [torch.empty(8 * len(me_items), dtype=torch.uint8, device="cuda") for _ in range(world)]
            h_gath = torch.empty(world * 8 * len(me_items), dtype=torch.uint8).pin_memory()
        esz_t = recv_yuv.element_size()

    def scatter_frames():
        if rank == 0:
            for r in range(world):
                scat[r].copy_(srcs[r], non_blocking=True)
        dist.scatter(recv_yuv, scat if rank == 0 else None, src=0)
        base = recv_yuv.data_ptr()
        tb.check(L.tb_frame_upload(cur.h, base, W, base + W * H * esz_t, base + (W * H + W * H // 4) * esz_t, W // 2))

    def gather_results():
        tb.check(L.tb_memcpy_d2d(me_out_t.data_ptr(), d_me_out.ptr, 8 * len(me_items)))
        dist.gather(me_out_t, gath if rank == 0 else None, dst=0)
        if rank == 0:
            for r in range(world):
                h_gath[r * 8 * len(me_items):(r + 1) * 8 * len(me_items)].copy_(gath[r], non_blocking=True)

    def filters_and_ref():
        tb.check(L.tb_deblock_frame(rec.h, d_bi.ptr, QP, BD))
        if cfg.cdef:
            for plane in range(3):
                tb.check(L.tb_cdef_frame(rec.h, scratch.h, d_bi.ptr, d_pri[int(plane > 0)].ptr, d_sec[int(plane > 0)].ptr, 5, 5, d_dv.ptr, BD, plane))
        for plane in range(3):
            tb.check(L.tb_clpf_detect_frame(rec.h, cur.h, d_bi.ptr, plane, BD, QP, d_sums.ptr))
        for plane, (fbl, strength) in enumerate(((6, 2), (4, 1), (4, 2))):
            tb.check(L.tb_clpf_frame(rec.h, scratch.h, d_bi.ptr, None, fbl, strength, BD, plane, QP))
        tb.check(L.tb_create_reference_frame(newref.h, rec.h))

    def step(timed=False):
        if world > 1:
            if timed:
                c0, c1 = ev(), ev(); c0.record(stream)
            scatter_frames()
            if timed:
                c1.record(stream)
        tb.check(L.tb_create_reference_frame(rec.h, pristine.h))  # the filters run in place: restore their input (device-side copy)
        if timed:
            a, b = ev(), ev(); a.record(stream)
        tb.check(L.tb_motion_estimate_batch(d_me.ptr, len(me_items), d_cand.ptr, ESZ, BD, cfg.speed, cfg.bipred, W, H, d_me_out.ptr))
        if timed:
            b.record(stream); me_ev.append((a, b))
        tb.check(L.tb_interp_batch(d_ip.ptr, len(ip_items), ESZ, BD, cfg.bipred))
        if timed:
            a, b = ev(), ev(); a.record(stream)
        tb.check(L.tb_txfm_chain_batch(d_tx.ptr, len(tx_items), ESZ, BD, d_tx_out.ptr))
        if timed:
            b.record(stream); tx_ev.append((a, b))
        tb.check(L.tb_intra_batch(d_in.ptr, len(in_items), ESZ, BD))
        filters_and_ref()
        if world > 1:
            if timed:
                c2, c3 = ev(), ev(); c2.record(stream)
            gather_results()
            if timed:
                c3.record(stream); coll_ev.append((c0, c1, c2, c3))

    # End-to-end step: the same work fed from pinned host memory and drained to pinned host memory INSIDE the step.  Three
    # streams: uploads (source frame, candidate lists, search items in chunks), compute, downloads (search results,
    # transform results per chunk, filtered frame); chunk i of a kernel waits only for chunk i of its upload and chunk i of a
    # download waits only for chunk i of its kernel, so PCIe traffic hides behind the kernels.  Nothing is carried over from
    # one step to the next: the step ends when the last download has landed.
    up, down = torch.cuda.Stream(), torch.cuda.Stream()
    use = lambda st: tb.check(L.tb_set_stream(C.c_void_p(st.cuda_stream)))
    # search items: a small first chunk so the first kernel starts early; transform results: eight chunks so the last download is short
    mb = [int(len(me_items) * f) for f in (0, 1 / 16, 1 / 4, 1 / 2, 1)]
    xb = [len(tx_items) * k // 8 for k in range(9)]
    ME_SZ, TX_SZ = me_items.dtype.itemsize, tx_items.dtype.itemsize

    def step_e2e():
        start = torch.cuda.Event(); start.record(stream)
        up.wait_event(start); down.wait_event(start)
        use(up)
        tb.check(L.tb_frame_upload(cur.h, h_y, W, h_u, h_v, W // 2))
        tb.check(L.tb_memcpy_h2d(d_cand.ptr, h_cand, cand_bytes))
        up_done = []
        for k in range(len(mb) - 1):
            tb.check(L.tb_memcpy_h2d(d_me.ptr + mb[k] * ME_SZ, h_me + mb[k] * ME_SZ, (mb[k + 1] - mb[k]) * ME_SZ))
            e = torch.cuda.Event(); e.record(up); up_done.append(e)
        use(stream)
        tb.check(L.tb_create_reference_frame(rec.h, pristine.h))
        for k in range(len(mb) - 1):
            stream.wait_event(up_done[k])
            tb.check(L.tb_motion_estimate_batch(d_me.ptr + mb[k] * ME_SZ, mb[k + 1] - mb[k], d_cand.ptr, ESZ, BD, cfg.speed, cfg.bipred, W, H, d_me_out.ptr + 8 * mb[k]))
        me_done = torch.cuda.Event(); me_done.record(stream)
        tb.check(L.tb_interp_batch(d_ip.ptr, len(ip_items), ESZ, BD, cfg.bipred))
        tx_done = []
        for k in range(len(xb) - 1):
            tb.check(L.tb_txfm_chain_batch(d_tx.ptr + xb[k] * TX_SZ, xb[k + 1] - xb[k], ESZ, BD, d_tx_out.ptr + 16 * xb[k]))
            e = torch.cuda.Event(); e.record(stream); tx_done.append(e)
        tb.check(L.tb_intra_batch(d_in.ptr, len(in_items), ESZ, BD))
        filters_and_ref()
        all_done = torch.cuda.Event(); all_done.record(stream)
        use(down)
        down.wait_event(me_done)
        tb.check(L.tb_memcpy_d2h_async(h_me_out, d_me_out.ptr, 8 * len(me_items)))
        for k in range(len(xb) - 1):
            down.wait_event(tx_done[k])
            tb.check(L.tb_memcpy_d2h_async(h_tx_out + 16 * xb[k], d_tx_out.ptr + 16 * xb[k], 16 * (xb[k + 1] - xb[k])))
        down.wait_event(all_done)
        tb.check(L.tb_frame_download_async(rec.h, h_rec[0], W, h_rec[1], h_rec[2], W // 2))
        landed = torch.cuda.Event(); landed.record(down)
        use(stream)
        stream.wait_event(landed)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        step()
    barrier()
    l0 = L.tb_launch_count()
    sampler = ClockSampler(local); sampler.start()
    t0, t1 = ev(), ev()
    t0.record(stream)
    for _ in range(args.steps):
        step(timed=True)
    t1.record(stream)
    barrier()
    clocks = sampler.stop()
    launches = int(L.tb_launch_count() - l0)
    ms = t0.elapsed_time(t1)
    me_ms = float(np.mean([a.elapsed_time(b) for a, b in me_ev]))
    tx_ms = float(np.mean([a.elapsed_time(b) for a, b in tx_ev]))
    coll_ms = float(np.mean([c0.elapsed_time(c1) + c2.elapsed_time(c3) for c0, c1, c2, c3 in coll_ev])) if coll_ev else 0.0
    if args.breakdown:
        names = ["restore", "motion_estimate", "interp", "txfm_chain", "intra", "deblock", "cdef x3", "clpf_detect x3", "clpf x3", "create_reference"]
        calls = [lambda: L.tb_create_reference_frame(rec.h, pristine.h),
                 lambda: L.tb_motion_estimate_batch(d_me.ptr, len(me_items), d_cand.ptr, ESZ, BD, cfg.speed, cfg.bipred, W, H, d_me_out.ptr),
                 lambda: L.tb_interp_batch(d_ip.ptr, len(ip_items), ESZ, BD, cfg.bipred),
                 lambda: L.tb_txfm_chain_batch(d_tx.ptr, len(tx_items), ESZ, BD, d_tx_out.ptr),
                 lambda: L.tb_intra_batch(d_in.ptr, len(in_items), ESZ, BD),
                 lambda: L.tb_deblock_frame(rec.h, d_bi.ptr, QP, BD),
                 lambda: [L.tb_cdef_frame(rec.h, scratch.h, d_bi.ptr, d_pri[int(p > 0)].ptr, d_sec[int(p > 0)].ptr, 5, 5, d_dv.ptr, BD, p) for p in range(3)],
                 lambda: [L.tb_clpf_detect_frame(rec.h, cur.h, d_bi.ptr, p, BD, QP, d_sums.ptr) for p in range(3)],
                 lambda: [L.tb_clpf_frame(rec.h, scratch.h, d_bi.ptr, None, f_, s_, BD, p, QP) for p, (f_, s_) in enumerate(((6, 2), (4, 1), (4, 2)))],
                 lambda: L.tb_create_reference_frame(newref.h, rec.h)]
        bd_ms = {}
        for nm, fn in zip(names, calls):
            a, b = ev(), ev(); a.record(stream); fn(); b.record(stream); torch.cuda.synchronize()
            bd_ms[nm] = round(a.elapsed_time(b), 3)
        sys.stderr.write("breakdown_ms " + json.dumps(bd_ms) + "\n")
    # end-to-end leg (host buffers in, host results out)
    for _ in range(2):
        step_e2e()
    barrier()
    e0, e1 = ev(), ev(); e0.record(stream)
    for _ in range(args.steps):
        step_e2e()
    e1.record(stream); barrier()
    ems = e0.elapsed_time(e1)
    # work counters of the motion-search kernel (one extra untimed launch)
    d_stats = tb.DevBuf.from_array(np.zeros(5, np.uint64))
    L.tb_me_set_stats(d_stats.ptr)
    tb.check(L.tb_motion_estimate_batch(d_me.ptr, len(me_items), d_cand.ptr, ESZ, BD, cfg.speed, cfg.bipred, W, H, d_me_out.ptr)); barrier()
    L.tb_me_set_stats(None)
    st = d_stats.download(np.uint64, 5)

    if world > 1:
        t = torch.tensor([ms, ems, me_ms, tx_ms, coll_ms], device="cuda"); dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms, ems, me_ms, tx_ms, coll_ms = [float(v) for v in t.tolist()]
    if rank != 0:
        return
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", 3350.0))
    peak_source = "MEASURED_PEAKS.json hbm_gbs" if peaks else "H100 SXM data sheet, 3.35 TB/s HBM3"

    def ncu_of(kernel):
        """DRAM bytes per launch + the binding ncu roofs of this kernel from an `ncu --set full` capture of the same workload
        (profiles/ncu_traffic.json, keyed by config and kernel; None when there is no capture)"""
        try:
            tr = json.load(open(os.path.join(ROOT, "profiles", "ncu_traffic.json")))[cfg.name][kernel]
            return tr
        except Exception:
            return None

    def roof(kernel, label, alg_bytes, k_ms, extra):
        tr = ncu_of(kernel)
        traffic = int(tr["dram_bytes_read"] + tr["dram_bytes_write"]) if tr and tr.get("items") == extra.get("items") else None
        achieved = alg_bytes / (k_ms * 1e-3) / 1e9
        r = {"kernel": label,
             # `achieved`/`frac` follow the bench contract: ALGORITHMIC bytes (SURVEY.md §8d) / launch time vs the HBM peak.  These bytes are
             # mostly served from L1/L2, not HBM, so an ncu capture's real DRAM rate is reported beside it when one is given.
             "bound": "issue+l1 (by design; not profiled on this GPU)", "achieved": round(achieved, 1), "peak": peak, "peak_source": peak_source, "unit": "GB/s",
             "frac": round(achieved / peak, 4), "l1_stream_gbs": round(achieved, 1), "traffic": traffic,
             "dram_gbs": round(traffic / (k_ms * 1e-3) / 1e9, 1) if traffic else None, "dram_frac": round(traffic / (k_ms * 1e-3) / 1e9 / peak, 4) if traffic else None,
             "ncu": {k: tr[k] for k in tr if k.endswith("_pct")} if tr else None,
             "algorithmic_bytes": int(alg_bytes), "ms_per_launch": round(k_ms, 3), "share_of_step": round(k_ms / (ms / args.steps), 3)}
        r.update(extra)
        return r
    alg_bytes = float(st[3] + st[4]) * ESZ  # SURVEY.md §8d: w*h*s per integer candidate (+ one read of the original), ((w+5)(h+5)+w*h)*s per sub-pel probe
    S = "uint8_t" if ESZ == 1 else "uint16_t"
    value = world * args.steps * cfg.PIXELS / (ms * 1e-3) / 1e6
    e2e_value = world * args.steps * cfg.PIXELS / (ems * 1e-3) / 1e6
    h2d = 3 * W * H // 2 * ESZ + me_bytes + cand_bytes
    d2h = 8 * len(me_items) + 16 * len(tx_items) + 3 * W * H // 2 * ESZ
    workload = cfg.describe(wl.counts())
    line = {
        "metric": metric_name(cfg),
        "value": round(value, 3), "unit": "Mpixel/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": round(ms / args.steps, 3), "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8" if ESZ == 1 else "u16", "data": "synthetic",
        "config": {"workload": workload,
                   "parallelism": ("frame-per-GPU x%d; per step rank 0 scatters the raw frames and gathers the search decisions over NCCL" % world) if world > 1 else
                                  "frame-per-GPU x1, no collective",
                   "l2_policy": "per-step inputs+outputs %.0f MB, L2 %.0f MB" % (resident_bytes / 1e6, torch.cuda.get_device_properties(local).L2_cache_size / 1e6)},
        "e2e": {"value": round(e2e_value, 3), "unit": "Mpixel/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h), "ms_per_step": round(ems / args.steps, 3)},
        "gpu_launches": launches,
        "clocks": clocks,
        "roofline": roof("me_batch_kernel", "me_batch_kernel<%s> (a1/a2/a4/a5/a7 fused motion search)" % S, alg_bytes, me_ms,
                         {"items": len(me_items), "searches": int(st[0]), "int_block_sads": int(st[1]), "subpel_probes": int(st[2])}),
        "roofline_txfm": roof("txfm_chain_kernel", "txfm_chain_kernel<%s> (a3/a10-a13 residual->DCT->quant->dequant->IDCT->recon->SSD)" % S, wl.txfm_alg_bytes(), tx_ms,
                              {"items": len(tx_items)}),
    }
    if world > 1:
        line["collective"] = {"backend": "nccl", "scatter_bytes_per_step": int((world - 1) * frame_elems * ESZ), "gather_bytes_per_step": int((world - 1) * 8 * len(me_items)),
                              "ms_per_step": round(coll_ms, 3), "share_of_step": round(coll_ms / (ms / args.steps), 4),
                              "what": "dist.scatter of the raw 4:2:0 source frames from rank 0 (pinned host -> HBM -> NVLink) + dist.gather of each rank's search results"}
    if not args.no_cpu:
        res, cpu_me, cpu_tx, sub = cpu_arm(args, cfg, brief=True)
        line["cpu_baseline"] = res
        # full-size parity: the GPU's results on the item lists (downloaded by the e2e leg) vs the reference's on the same lists
        g_me = pinned_view(h_me_out, tb.ME_RESULT, len(me_items))[::sub]; g_tx = pinned_view(h_tx_out, tb.TXFM_RESULT, len(tx_items))[::sub]
        me_eq = int(((g_me["mvx"] == cpu_me["mvx"]) & (g_me["mvy"] == cpu_me["mvy"]) & (g_me["cost"] == cpu_me["cost"])).sum())
        tx_eq = int(((g_tx["ssd"] == cpu_tx["ssd"]) & (g_tx["cbp"] == cpu_tx["cbp"])).sum())
        line["parity"] = {"me": "%d/%d" % (me_eq, len(cpu_me)), "txfm": "%d/%d" % (tx_eq, len(cpu_tx)), "sample": "every %d-th item of the full lists" % sub,
                          "checker": res["kind"], "ok": me_eq == len(cpu_me) and tx_eq == len(cpu_tx)}
    print(json.dumps(line))
    if not args.no_cpu and not line["parity"]["ok"]:
        sys.stderr.write("PARITY FAILURE: GPU results differ from the %s on the bench lists\n" % res["kind"])
        sys.exit(3)


# ----------------------------------------------------------------------------------------------------------------------
# CPU arm: the same item lists through the reference's own kernels (oracle/_ref) on all host cores
# ----------------------------------------------------------------------------------------------------------------------
def cpu_arm(args, cfg, brief=False):
    R = load_records()  # item dtypes only: this arm never loads libthor_b200.so
    W, H, BD, ESZ, NREF = cfg.W, cfg.H, cfg.BD, cfg.ESZ, cfg.NREF
    refso = os.path.join(ROOT, "oracle", "_ref", "libcpubench_ref.so"); portso = os.path.join(ROOT, "oracle", "libcpubench_port.so")
    if os.path.exists(refso):
        C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libthorref.so"), mode=C.RTLD_GLOBAL)
        lib = C.CDLL(refso)
    else:
        if not os.path.exists(portso):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "port"])
        lib = C.CDLL(portso)
    lib.cpu_bench_run.restype = C.c_double
    lib.cpu_bench_run.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p] + [C.c_int] * 7
    lib.cpu_bench_imbalance.restype = C.c_double
    lib.cpu_bench_core_seconds.restype = C.c_double
    lib.cpu_bench_cpu_seconds.restype = C.c_double
    lib.cpu_bench_kind.restype = C.c_char_p
    kind = lib.cpu_bench_kind().decode()
    cores = len(os.sched_getaffinity(0))
    try:
        import psutil
        phys = psutil.cpu_count(logical=False)
    except Exception:
        phys = None
    sub = max(1, args.cpu_subsample)  # every sub-th work item of each list (1 = the full frame)
    fr = synth_frames(cfg, 2026, NREF + 1)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from _refstructs import Frame as HFrame
    from _libs import oracle, P
    O = oracle()

    def hframe(planes):
        f = HFrame(W, H, BD, int(ESZ == 2))
        f.y[...] = planes[0]; f.u[...] = planes[1]; f.v[...] = planes[2]
        for p, (pw, ph, pad) in enumerate(((W, H, 160), (W // 2, H // 2, 80), (W // 2, H // 2, 80))):
            (O.orc_pad_plane_lbd if ESZ == 1 else O.orc_pad_plane_hbd)(P(f.full(p), f.origin(p)), f.stride(p), pw, ph, pad, pad)
        return f
    cur = hframe(fr[0]); refs = [hframe(fr[k + 1]) for k in range(NREF)]; rec = hframe(fr[1])
    pl = lambda f, p: (f.full(p).ctypes.data + f.origin(p) * ESZ, f.stride(p))
    wl = Workload(cfg, R, 2026)
    pred = np.empty(wl.ip_total + 64, cfg.SDT); ibuf = np.empty(wl.in_total + 64, cfg.SDT)
    pred.fill(0); ibuf.fill(0)  # touch the pages now: first-touch faults are not part of the reference's kernel time
    wl.bind([pl(cur, 0), pl(cur, 1)], [[pl(r, p) for p in range(3)] for r in refs], pl(rec, 0), None, pred.ctypes.data, ibuf.ctypes.data)
    full_counts = wl.counts()
    me, cd, tx, ip, it = [np.ascontiguousarray(a[::sub]) if sub > 1 else a for a in (wl.me, wl.cands, wl.tx, wl.ip, wl.intra)]
    if sub > 1:
        cd = wl.cands  # candidate lists are addressed through cand_ofs: keep them whole
    me_out = np.zeros(len(me), R.ME_RESULT); tx_out = np.zeros(len(tx), R.TXFM_RESULT)
    hbd = int(ESZ == 2)
    imb, core_s, cpu_s, by_list = [], [0.0], [0.0], {}

    def run_once():
        t = 0.0
        for name, kind_, items, cands_, out in (("search", 0, me, cd, me_out), ("interp", 3, ip, None, None), ("txfm", 1, tx, None, tx_out), ("intra", 2, it, None, None)):
            dt = lib.cpu_bench_run(kind_, items.ctypes.data, len(items), None if cands_ is None else cands_.ctypes.data, None if out is None else out.ctypes.data,
                                   hbd, BD, cfg.speed, cfg.bipred, W, H, cores)
            t += dt; by_list[name] = by_list.get(name, 0.0) + dt
            imb.append((dt, lib.cpu_bench_imbalance())); core_s[0] += lib.cpu_bench_core_seconds(); cpu_s[0] += lib.cpu_bench_cpu_seconds()
        return t

    steps = max(1, args.steps if args.impl == "reference" else 1)
    for _ in range(args.warmup if args.impl == "reference" else 0):
        run_once()
    imb.clear(); core_s[0] = 0.0; cpu_s[0] = 0.0; by_list.clear()
    total = 0.0
    for _ in range(steps):
        total += run_once()
    value = steps * cfg.PIXELS / sub / total / 1e6
    imbalance = max([b for dt, b in imb if dt > 0.1] or [1.0])  # lists that ran long enough for thread start-up not to matter
    sample = ("%s of one %dx%d frame (%d motion searches, %d predictions, %d transform chains, %d intra predictions) through the %s on %d threads, "
              "dynamic work queue (largest blocks first); frame-level filters not included in the CPU sample" %
              ("every work item" if sub == 1 else "every %d-th work item of each list" % sub, W, H, len(me), len(ip), len(tx), len(it),
               "reference's own kernels (oracle/_ref, SIMD path, gcc -O3 -march=x86-64-v3; the reference Makefile uses -march=native)" if kind == "reference" else "oracle port",
               cores))
    res = {"value": round(value, 4), "unit": "Mpixel/s", "cores": cores, "physical_cores": phys, "kind": kind, "sample": sample, "seconds": round(total, 2),
           "thread_wall_seconds_per_frame": round(core_s[0] / steps * sub, 2), "cpu_seconds_per_frame": round(cpu_s[0] / steps * sub, 2),
           "effective_cores": round(cpu_s[0] / total, 1),
           "ideal_value_all_threads": round(cfg.PIXELS / (cpu_s[0] / steps * sub / cores) / 1e6, 3),
           "note": "value = measured wall throughput of this host; cpu_seconds_per_frame = CPU time the threads consumed (CLOCK_THREAD_CPUTIME_ID); effective_cores = "
                   "cpu seconds / wall seconds: when it is far below `cores` the box did not grant the threads that many cores (shared host / SMT); "
                   "ideal_value_all_threads = pixels / (cpu_seconds_per_frame / cores): what perfect scaling over every hardware thread would give", "seconds_by_list": {k: round(v, 3) for k, v in by_list.items()}, "imbalance_max_over_mean": round(imbalance, 3)}
    assert imbalance < 1.3, "CPU arm is load-imbalanced (max/mean thread time %.2f): its throughput is not a fair baseline" % imbalance
    if brief:
        return res, me_out, tx_out, sub
    line = {"impl": "reference", "metric": metric_name(cfg),
            "value": res["value"], "unit": "Mpixel/s", "n_gpus": int(os.environ.get("WORLD_SIZE", args.gpus)), "steps": steps, "warmup": args.warmup,
            "ms_per_step": round(1e3 * total / steps * sub, 1), "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8" if ESZ == 1 else "u16", "data": "synthetic",
            "config": {"workload": cfg.describe(full_counts), "parallelism": "all host threads, dynamic queue", "sample": "1/%d of the lists per step" % sub},
            "cpu_baseline": res, "e2e": {"value": res["value"], "unit": "Mpixel/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", default="hdb", choices=sorted(Cfg.TABLE), help="BASELINE.json configuration (default: the headline 1080p HDB_high_efficiency)")
    ap.add_argument("--bitdepth", type=int, default=8, choices=[8, 10], help="10 = --config hdb10")
    ap.add_argument("--cpu-subsample", type=int, default=1, help="CPU arm: every k-th work item (1 = the full lists; the parity check then covers every item)")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--breakdown", action="store_true")
    args = ap.parse_args()
    cfg = Cfg("hdb10" if args.bitdepth == 10 and args.config == "hdb" else args.config)
    if args.impl == "reference":
        if int(os.environ.get("RANK", 0)) == 0:
            cpu_arm(args, cfg)
        return
    run_gpu(args, cfg)


if __name__ == "__main__":
    main()
