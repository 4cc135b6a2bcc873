// rdo_hostcheck.cpp — TEST INFRASTRUCTURE ONLY (never linked into libthor_b200.so, never on a product path).
//
// The RD-loop control flow of thor_b200/csrc/tb_rdo.h instantiated over the plain-C oracle's primitives (oracle/thor_oracle.h), on the CPU.
// Purpose: this container has no GPU, and the control flow (process_block / mode_decision_rdo / early skip / bit counting / MV
// predictors) is the part of SURVEY §8f.1 that no existing kernel test covers.  oracle/_ref/Thorenc_rdocheck = the reference's
// unmodified objects + thor_b200/csrc/tb_rdo_shim.c + this library; with TB_RDO_VERIFY=1 every super block of a real encode is decided by
// this code AND by the reference's process_block() on the same state and compared (bits, reconstruction, deblock_data), and without it
// the whole encode runs through tb_rdo_encode_frame() below and the .bit file must equal the reference's.  tests/test_rdo_host.py.
// The CUDA build of the same header (thor_b200/csrc/tb_rdo.cu) differs only in the backend, whose primitives are parity-tested separately.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>
#include "../thor_b200/csrc/tb_rdo.h"
#include "thor_oracle.h"

using namespace tbr;

template <class S> struct Orc;
#define ORC_FWD(S, SFX)                                                                                                                                        \
  template <> struct Orc<S> {                                                                                                                                  \
    static unsigned sad(const S *a, const S *b, int as, int bs, int w, int h) { return orc_sad_##SFX(a, b, as, bs, w, h); }                                     \
    static uint64_t ssd(const S *a, const S *b, int as, int bs, int w, int h) { return orc_ssd_##SFX(a, b, as, bs, w, h); }                                     \
    static void luma(S *p, const S *r, int w, int h, int st, int ps, const orc_mv_t *mv, int sign, int bip, int pw, int ph, int x, int y, int bd) {             \
      orc_get_inter_prediction_luma_##SFX(p, r, w, h, st, ps, mv, sign, bip, pw, ph, x, y, bd);                                                                 \
    }                                                                                                                                                          \
    static void chroma(S *p, const S *r, int w, int h, int st, int ps, const orc_mv_t *mv, int sign, int pw, int ph, int x, int y, int bd) {                    \
      orc_get_inter_prediction_chroma_##SFX(p, r, w, h, st, ps, mv, sign, pw, ph, x, y, bd);                                                                    \
    }                                                                                                                                                          \
    static void residual(int16_t *b, const S *p, const S *o, int size, int ps, int os) { orc_residual_##SFX(b, p, o, size, ps, os); }                           \
    static void reconstruct(const int16_t *b, const S *p, S *r, int size, int ps, int rs, int bd) { orc_reconstruct_##SFX(b, p, r, size, ps, rs, bd); }         \
    static void tl(S *l, S *t, S *c, const S *rf, int fs, const S *rb, int rbs, int i, int j, int y, int x, int size, int ur, int dl, int tbs, int bd) {        \
      orc_make_top_and_left_##SFX(l, t, c, rf, fs, rb, rbs, i, j, y, x, size, ur, dl, tbs, bd);                                                                 \
    }                                                                                                                                                          \
    static void ipred(const S *l, const S *t, S c, int y, int x, int size, S *p, int ps, int mode, int bd) { orc_intra_pred_##SFX(l, t, c, y, x, size, p, ps, mode, bd); } \
    static void cfl(const S *y, S *u, S *v, const S *ry, int n, int cs, int st, int sub, int bd) { orc_cfl_##SFX(y, u, v, ry, n, cs, st, sub, bd); }            \
    static int me(const S *o, const S *r, int size, int rs, int w, int h, orc_mv_t *mv, const orc_mv_t *mvc, const orc_mv_t *mvp, double lam, int speed, int bd, \
                  int sign, int fw, int fh, int x, int y, const orc_mv_t *cand, int n, int bip) {                                                               \
      return orc_motion_estimate_##SFX(o, r, size, rs, w, h, mv, mvc, mvp, lam, speed, bd, sign, fw, fh, x, y, cand, n, bip);                                   \
    }                                                                                                                                                          \
    static int me_bi(const S *o, const S *r0, const S *r1, int size, int rs, int w, int h, orc_mv_t *mv, const orc_mv_t *mvc, const orc_mv_t *mvp, double lam,  \
                     int bd, int sign, int fw, int fh, int x, int y, const orc_mv_t *cand, int n, int bip) {                                                    \
      return orc_motion_estimate_bi_##SFX(o, r0, r1, size, rs, w, h, mv, mvc, mvp, lam, bd, sign, fw, fh, x, y, cand, n, bip);                                  \
    }                                                                                                                                                          \
  };
ORC_FWD(uint8_t, lbd)
ORC_FWD(uint16_t, hbd)

// "warps" simulated by host threads (TBR_HOST_WARPS=N): the exchange area and the barrier of one simulated CTA
struct Exchange {
  int nw = 1;
  std::mutex m;
  std::condition_variable cv;
  int waiting = 0, phase = 0;
  uint32_t cost[16];
  int idx[16];
  uint32_t rng[16][2];
  int flag[16];
  Mv mv[TB_RDO_MAX_REF][16];
  uint32_t sad[TB_RDO_MAX_REF];
  unsigned char buf[256];
  int queue[4] = {0, 0, 0, 0};
  // The oracle's functions keep static scratch buffers (not re-entrant), so the simulated warps never run at the same time: a thread
  // holds `run` while it executes and gives it up only while it waits at a barrier.  The interleaving is arbitrary, the semantics are
  // those of warps that only communicate at CTA barriers.
  std::mutex run;
  void barrier() {
    if (nw == 1) return;
    run.unlock();
    {
      std::unique_lock<std::mutex> lk(m);
      const int ph = phase;
      if (++waiting == nw) { waiting = 0; phase++; cv.notify_all(); }
      else cv.wait(lk, [&] { return phase != ph; });
    }
    run.lock();
  }
};

template <class S> struct OracleBackend {
  const FrameCtx<S> *F;
  Exchange *X = nullptr;
  int wid = 0;
  // ---- SPMD over simulated warps (see tb_rdo.h)
  int warp() const { return wid; }
  bool mine(int k) const { return (k % X->nw) == wid; }
  void cta_sync() const { X->barrier(); }
  void mark(int) const {}  // phase timers exist only on the device
  void mark2(int) const {}
  int nwarps() const { return X->nw; }
  void queue_reset() const { X->barrier(); if (wid == 0) for (int q = 0; q < 4; q++) X->queue[q] = 0; X->barrier(); }
  // shared counters; the simulated warp gives the others a chance to run at every draw, so the distribution of the items varies from run to run
  int next(int q) const {
    const int v = X->queue[q]++;
    if (X->nw > 1) { X->run.unlock(); std::this_thread::yield(); X->run.lock(); }
    return v;
  }
  void copy_words(void *dst, const void *src, int nwords) const { memcpy(dst, src, (size_t)nwords * 4); }
  void put_me(int ref, const Mv *mv16, uint32_t sad) const { memcpy(X->mv[ref], mv16, 16 * sizeof(Mv)); X->sad[ref] = sad; }
  void get_me(int ref, Mv *mv16, uint32_t *sad) const { memcpy(mv16, X->mv[ref], 16 * sizeof(Mv)); *sad = X->sad[ref]; }
  int reduce_best(uint32_t *cost, int *idx) const {
    X->cost[wid] = *cost; X->idx[wid] = *idx;
    X->barrier();
    int w = 0;
    for (int k = 1; k < X->nw; k++)
      if (X->cost[k] < X->cost[w] || (X->cost[k] == X->cost[w] && X->idx[k] < X->idx[w])) w = k;
    *cost = X->cost[w]; *idx = X->idx[w];
    X->barrier();
    return w;
  }
  void bcast(void *p, int nbytes, int owner) const {
    if (wid == owner) memcpy(X->buf, p, nbytes);
    X->barrier();
    if (wid != owner) memcpy(p, X->buf, nbytes);
    X->barrier();
  }
  void reduce_range(uint32_t *worst, uint32_t *best) const {
    X->rng[wid][0] = *worst; X->rng[wid][1] = *best;
    X->barrier();
    for (int k = 0; k < X->nw; k++) { if (X->rng[k][0] > *worst) *worst = X->rng[k][0]; if (X->rng[k][1] < *best) *best = X->rng[k][1]; }
    X->barrier();
  }
  int reduce_or(int f) const {
    X->flag[wid] = f;
    X->barrier();
    int r = 0;
    for (int k = 0; k < X->nw; k++) r |= X->flag[k];
    X->barrier();
    return r;
  }
  // scratch
  int16_t block[128 * 128], coeff[128 * 128], rcoeff[128 * 128], rblock[128 * 128], tmp[32 * 32];
  S compact[128 * 128], left[2 * 128 + 16], top[2 * 128 + 16];

  tb_rdo_blk_t ld_blk(const tb_rdo_blk_t *p) const { return *p; }
  void clip_mv(Mv &mv, int ypos, int xpos, int fw, int fh, int bw, int bh, int sign) const { orc_clip_mv((orc_mv_t *)&mv, ypos, xpos, fw, fh, bw, bh, sign); }
  void interp_luma(S *dst, int ds, const S *ref, int rs, int w, int h, Mv mv, int sign, int bip, int pw, int ph, int xpos, int ypos) const {
    Orc<S>::luma(dst, ref, w, h, rs, ds, (const orc_mv_t *)&mv, sign, bip, pw, ph, xpos, ypos, F->bitdepth);
  }
  void interp_chroma(S *dst, int ds, const S *ref, int rs, int w, int h, Mv mv, int sign, int pw, int ph, int xc, int yc) const {
    Orc<S>::chroma(dst, ref, w, h, rs, ds, (const orc_mv_t *)&mv, sign, pw, ph, xc, yc, F->bitdepth);
  }
  void avg(S *dst, const S *a, const S *b, int stride, int w, int h) const {
    for (int i = 0; i < h; i++)
      for (int j = 0; j < w; j++) dst[i * stride + j] = (S)(((int)a[i * stride + j] + (int)b[i * stride + j]) >> 1);
  }
  void sat2ab(S *dst, const S *org, int os, const S *pred, int size) const {  // enc/encode_block.c:1780-1782
    const int maxv = (1 << F->bitdepth) - 1;
    for (int i = 0; i < size; i++)
      for (int j = 0; j < size; j++) {
        int v = 2 * (int16_t)org[i * os + j] - (int16_t)pred[i * size + j];
        dst[i * size + j] = (S)(v < 0 ? 0 : (v > maxv ? maxv : v));
      }
  }
  void copy(S *dst, int ds, const S *src, int ss, int w, int h) const {
    for (int i = 0; i < h; i++) memcpy(dst + i * ds, src + i * ss, (size_t)w * sizeof(S));
  }
  void copy_coeff(int16_t *dst, const int16_t *src) const { memcpy(dst, src, 1024 * sizeof(int16_t)); }
  void intra_predict(S *dst, int ds, const S *recf, int rfs, const S *rblock_, int rbs, int i, int j, int ypos, int xpos, int size, int ur, int dl, int tbs, int mode) {
    S tl;
    Orc<S>::tl(left, top, &tl, recf, rfs, rblock_, rbs, i, j, ypos, xpos, size, ur, dl, tbs, F->bitdepth);
    if (mode == 10) Orc<S>::ipred(left, top, tl, 1, 1, size, dst, ds, 0, F->bitdepth);  // DC from (left, top) as gathered
    else Orc<S>::ipred(left, top, tl, ypos + i, xpos + j, size, dst, ds, mode, F->bitdepth);
  }
  void cfl(const S *y, S *u, S *v, const S *ry, int n, int cstride, int stride) const { Orc<S>::cfl(y, u, v, ry, n, cstride, stride, 1, F->bitdepth); }
  void tx_multi(const tb_txfm_item_t *jobs, int n, int *bit) {  // the device runs these side by side; here one after the other
    for (int k = 0; k < n; k++) {
      const tb_txfm_item_t &q = jobs[k];
      bit[k] = tx_chain((const S *)q.orig, q.ostride, (const S *)q.pred, q.pstride, (S *)q.rec, q.rstride, q.coeffq, q.size, q.qp, q.coeff_type, q.fast & TB_TXFM_FAST);
    }
  }
  int tx_chain(const S *orig, int os, const S *pred, int ps, S *rec, int rs, int16_t *cq, int size, int qp, int coeff_type, int fast) {
    Orc<S>::residual(block, pred, orig, size, ps, os);
    orc_transform(block, coeff, size, fast, F->bitdepth);
    const int cbp = orc_quantize(coeff, cq, qp, size, coeff_type, nullptr);
    if (cbp) {
      orc_dequantize(cq, rcoeff, qp, size, nullptr);
      orc_inverse_transform(rcoeff, rblock, size, F->bitdepth);
      Orc<S>::reconstruct(rblock, pred, rec, size, ps, rs, F->bitdepth);
    } else
      copy(rec, rs, pred, ps, size, size);
    return cbp;
  }
  int coeff_bits(const int16_t *cq, int size, int type) const { return orc_coeff_bits(cq, size, type); }
  uint64_t ssd(const S *a, int as, const S *b, int bs, int w, int h) const { return Orc<S>::ssd(a, b, as, bs, w, h); }
  unsigned sad(const S *a, int as, const S *b, int bs, int w, int h) const { return Orc<S>::sad(a, b, as, bs, w, h); }
  // the reference searches a compact copy of the original (pitch = coding-block size, enc/encode_block.c:2457)
  int me(const S *org, int os, const S *ref, int rs, int size, int w, int h, Mv *mv, Mv mvc, Mv mvp, double lambda, int sign, int xpos, int ypos, const Mv *cand, int ncand) {
    for (int i = 0; i < h; i++) memcpy(compact + i * size, org + i * os, (size_t)w * sizeof(S));
    return Orc<S>::me(compact, ref, size, rs, w, h, (orc_mv_t *)mv, (const orc_mv_t *)&mvc, (const orc_mv_t *)&mvp, lambda, F->speed, F->bitdepth, sign, F->width, F->height, xpos,
                      ypos, (const orc_mv_t *)cand, ncand, F->enable_bipred);
  }
  int me_bi(const S *org, int os, const S *ref0, const S *ref1, int rs, int size, Mv *mv, Mv mvc, Mv mvp, double lambda, int sign, int xpos, int ypos, const Mv *cand, int ncand, S *, S *) {
    for (int i = 0; i < size; i++) memcpy(compact + i * size, org + i * os, (size_t)size * sizeof(S));
    return Orc<S>::me_bi(compact, ref0, ref1, size, rs, size, size, (orc_mv_t *)mv, (const orc_mv_t *)&mvc, (const orc_mv_t *)&mvp, lambda, F->bitdepth, sign, F->width, F->height,
                         xpos, ypos, (const orc_mv_t *)cand, ncand, 1);
  }
  // check_early_skip_sub_block (enc/encode_block.c:2147-2180): 2x2 average, (size/2)-point transform, any |c| > threshold
  int es_luma(const S *orig, int os, const S *pred, int ps, int size, int threshold) {
    Orc<S>::residual(block, pred, orig, size, ps, os);
    const int s2 = size / 2;
    for (int i = 0; i < s2; i++)
      for (int j = 0; j < s2; j++)
        tmp[i * s2 + j] = (int16_t)((block[(2 * i) * size + 2 * j] + block[(2 * i) * size + 2 * j + 1] + block[(2 * i + 1) * size + 2 * j] + block[(2 * i + 1) * size + 2 * j + 1] + 2) >> 2);
    orc_transform(tmp, coeff, s2, 0, F->bitdepth);
    for (int i = 0; i < s2 * s2; i++)
      if (abs((int)coeff[i]) > threshold) return 1;
    return 0;
  }
  // check_early_skip_sub_blockC :2214-2229 with calc_cbp_simd (use_simd = 1)
  int es_chroma(const S *orig, int os, const S *pred, int ps, int size, int threshold) {
    Orc<S>::residual(block, pred, orig, size, ps, os);
    return orc_calc_cbp(block, size, threshold);
  }
  // copy_deblock_data, enc/encode_block.c:1568-1613
  void store_blk(tb_rdo_blk_t *blk, int stride, int by, int bx, int nbw, int nbh, int div, tb_rdo_blk_t v, const Mv *mv0, const Mv *mv1) const {
    for (int m = 0; m < nbh; m++)
      for (int n = 0; n < nbw; n++) {
        const int m0 = div > 0 ? m / div : 0, n0 = div > 0 ? n / div : 0, index = 2 * m0 + n0;
        tb_rdo_blk_t w = v;
        w.mv0 = mv0[index]; w.mv1 = mv1[index];
        blk[(by + m) * stride + bx + n] = w;
      }
  }
  void pack_coeff(int16_t *dst, const int16_t *q, int size, int tb_split, int nonzero) const {
    const int t = tb_split ? size / 2 : size, qs = t < 16 ? t : 16, n = tb_split ? 4 : 1;
    for (int k = 0; k < n; k++)
      for (int i = 0; i < qs * qs; i++) dst[k * qs * qs + i] = nonzero ? q[k * 256 + i] : 0;
  }
  void store_leaf(tb_rdo_leaf_t *p, const tb_rdo_leaf_t &L) const { *p = L; }
  void store_count(int *p, int n) const { *p = n; }
};

template <class S> static void make_ctx(FrameCtx<S> &C, const tb_rdo_frame_t *f) {
  static const int8_t chroma_qp_mid[13] = {29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37};
  C.width = f->width; C.height = f->height; C.sb_size = 1 << f->log2_sb_size; C.bitdepth = f->bitdepth; C.frame_type = f->frame_type; C.qp = f->qp;
  C.qpc = f->qp < 30 ? f->qp : (f->qp >= 43 ? f->qp - 6 : chroma_qp_mid[f->qp - 30]);
  C.num_ref = f->num_ref; C.interp_ref = f->interp_ref; C.num_intra_modes = f->num_intra_modes; C.lambda = f->lambda; C.sqrt_lambda = sqrt(f->lambda);
  C.enable_bipred = f->enable_bipred; C.enable_tb_split = f->enable_tb_split; C.enable_pb_split = f->enable_pb_split; C.speed = f->encoder_speed; C.intra_rdo = f->intra_rdo;
  C.use_block_contexts = f->use_block_contexts; C.cfl_intra = f->cfl_intra; C.cfl_inter = f->cfl_inter; C.early_skip_thr = f->early_skip_thr;
  for (int r = 0; r < TB_RDO_MAX_REF; r++) {
    C.ref_sign[r] = f->ref_sign[r]; C.ref_sign_ge[r] = f->ref_sign_ge[r];
    for (int p = 0; p < 3; p++) C.ref[r][p] = (const S *)f->ref[r][p];
  }
  for (int p = 0; p < 3; p++) { C.org[p] = (const S *)f->orig[p]; C.rec[p] = (S *)f->rec[p]; }
  C.org_stride[0] = f->orig_stride[0]; C.org_stride[1] = f->orig_stride[1]; C.ref_stride[0] = f->ref_stride[0]; C.ref_stride[1] = f->ref_stride[1];
  C.rec_stride[0] = f->rec_stride[0]; C.rec_stride[1] = f->rec_stride[1];
  C.blk = f->blk; C.blk_stride = f->width / 4; C.leaves = f->leaves; C.leaf_count = f->leaf_count; C.coeffs = f->coeffs;
}

template <class S> static int run(const tb_rdo_frame_t *f, int sbx0, int sby0, int one) {
  static FrameCtx<S> C;
  const char *e = getenv("TBR_HOST_WARPS");
  const int nw = e ? atoi(e) : 1;
  if (nw < 1 || nw > 16) return TB_ERR_ARG;
  static std::vector<Work<S>> W;
  static std::vector<OracleBackend<S>> be;
  static Exchange X;
  if ((int)W.size() != nw) { W.resize(nw); be.resize(nw); }
  make_ctx(C, f);
  X.nw = nw;
  for (int k = 0; k < nw; k++) { be[k].F = &C; be[k].X = &X; be[k].wid = k; }
  const int nsbx = (C.width + C.sb_size - 1) / C.sb_size, nsby = (C.height + C.sb_size - 1) / C.sb_size;
  for (int sby = one ? sby0 : 0; sby < (one ? sby0 + 1 : nsby); sby++)
    for (int sbx = one ? sbx0 : 0; sbx < (one ? sbx0 + 1 : nsbx); sbx++) {
      auto body = [&](int k) {
        if (nw > 1) X.run.lock();
        Rdo<S, OracleBackend<S>> R(C, W[k], W[0], be[k]);
        R.process_sb(sbx, sby);
        if (nw > 1) X.run.unlock();
      };
      if (nw == 1) body(0);
      else {
        std::vector<std::thread> th;
        for (int k = 0; k < nw; k++) th.emplace_back(body, k);
        for (auto &t : th) t.join();
      }
    }
  return TB_OK;
}

static int check(const tb_rdo_frame_t *f) {
  if (!f || f->num_ref > TB_RDO_MAX_REF || f->log2_sb_size > 7 || (f->sample_bytes != 1 && f->sample_bytes != 2)) return TB_ERR_ARG;
  return TB_OK;
}

extern "C" {
// same C ABI as libthor_b200.so's entry point, computed on the CPU by the oracle (test infrastructure)
int tb_rdo_encode_frame(const tb_rdo_frame_t *f) {
  if (check(f) != TB_OK) return TB_ERR_ARG;
  return f->sample_bytes == 1 ? run<uint8_t>(f, 0, 0, 0) : run<uint16_t>(f, 0, 0, 0);
}
// one super block on the caller's current state (rec planes and blk grid are in/out): the in-situ comparison of tb_rdo_shim.c
int tb_rdo_encode_sb(const tb_rdo_frame_t *f, int sbx, int sby) {
  if (check(f) != TB_OK) return TB_ERR_ARG;
  return f->sample_bytes == 1 ? run<uint8_t>(f, sbx, sby, 1) : run<uint16_t>(f, sbx, sby, 1);
}
}
