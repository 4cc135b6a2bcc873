/* thor_oracle.c — TEST INFRASTRUCTURE ONLY (see thor_oracle.h).  Bit-depth independent half of the plain-C
 * restatement of the Thor hot path, plus the two instantiations of thor_oracle_tmpl.h. */
#include "thor_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

static int orc_log2i(int x) { int r = 0; while (x > 1) { x >>= 1; r++; } return r; } /* common/simd.h:86 */
static int orc_sat(int v, int maxv) { return v < 0 ? 0 : v > maxv ? maxv : v; }        /* common/global.h:128 */

/* ---- tables ---- */
/* HEVC core-transform magnitudes at angle k*pi/64, k = 0..32 (k = 0 is the DC row's 64).  The NxN matrices of
 * common/transform.c:37-241 are M_N[i][j] = +-T[fold((2j+1)*i*32/N mod 128)]. */
static const int8_t orc_T[33] = {64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64,
                                 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9,  4,  0};
static int16_t orc_mats[4][32 * 32];
static int orc_zz[3][256];
static int orc_tables_ready;
static void orc_init_tables(void) {
  if (orc_tables_ready) return;
  for (int l = 2; l <= 5; l++) {
    int n = 1 << l;
    for (int i = 0; i < n; i++)
      for (int j = 0; j < n; j++) {
        int m = ((2 * j + 1) * i * (32 / n)) & 127;
        if (m > 64) m = 128 - m;
        orc_mats[l - 2][i * n + j] = (int16_t)(m > 32 ? -orc_T[64 - m] : orc_T[m]);
      }
  }
  for (int t = 0; t < 3; t++) { /* classic zig-zag: scan index of each (row, col) */
    int n = 4 << t, idx = 0;
    for (int d = 0; d <= 2 * (n - 1); d++)
      for (int k = 0; k <= d; k++) {
        int r = (d & 1) ? k : d - k, c = d - r;
        if (r < n && c < n) orc_zz[t][r * n + c] = idx++;
      }
  }
  orc_tables_ready = 1;
}
const int16_t *orc_dct_matrix(int log2size) { orc_init_tables(); return orc_mats[log2size - 2]; }
const int *orc_zigzag(int qsize) { orc_init_tables(); return orc_zz[qsize == 4 ? 0 : qsize == 8 ? 1 : 2]; }
int orc_chroma_qp(int qp) {
  static const int8_t mid[13] = {29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37};
  return qp < 30 ? qp : qp >= 43 ? qp - 6 : mid[qp - 30];
}
static const uint16_t orc_quant[6] = {26214, 23302, 20560, 18396, 16384, 14564}; /* common/common_tables.c:72 */
static const uint16_t orc_dequant[6] = {40, 45, 51, 57, 64, 72};                 /* common/common_tables.c:73 */
/* common/common_frame.c:36-45 */
static const uint8_t orc_beta_table[52] = {0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15,
                                           16, 17, 18, 20, 22, 24, 26, 28, 30, 32, 34, 36, 38, 40, 42, 44, 46, 48, 50, 52, 54, 56, 58, 60, 62, 64};
static const uint8_t orc_tc_table[56] = {0,  0,  1,  1,  2,  3,  4,  5,  6,  7,  8,  9,  10,  11,  12,  13,  14,  15,  16,
                                         17, 18, 20, 22, 24, 26, 28, 30, 32, 36, 40, 44, 48,  52,  56,  60,  64,  68,  72,
                                         80, 88, 96, 104, 112, 128, 144, 152, 160, 168, 176, 184, 192, 200, 208, 216, 224, 232};

/* ---- a10: forward transform.  common/transform.c:245-308 (C path; int16 intermediates), box sum as in transform_simd ---- */
void orc_transform(const int16_t *block, int16_t *coeff, int size, int fast, int bitdepth) {
  static int16_t tmp[32][32], tmp2[32 * 32];
  const int16_t *in = block;
  int qsize = size < 16 ? size : 16, size1 = size, scale = 1;
  if (size > (32 >> fast)) {
    size1 = 32 >> fast;
    scale = size / size1;
    /* The box sum is formed as the encoder's transform_simd forms it.  64x64 and 128x128 with `fast` saturate to [-16384, 16383] after every
       addition (common/common_kernels.c:1524-1529).  The 2x2 sums of 32x32 with `fast` (:1501-1503) and the sums of 64x64 and 128x128 without
       it (:1544-1549) wrap in int16.  The C transform saturates everywhere (common/transform.c:261-278).  The two rules differ only when a
       partial sum leaves [-16384, 16383]: 4 residuals never do (4 x 4095 = 16380), and 16 residuals only above 10 bits (16 x 1023 = 16368),
       so only 128x128 without `fast` at 12 bits tells them apart. */
    const int sat = fast && size >= 64;
    for (int i = 0; i < size1; i++)
      for (int j = 0; j < size1; j++) {
        int16_t sum = 0;
        for (int m = 0; m < scale; m++)
          for (int n = 0; n < scale; n++) {
            int v = sum + block[(i * scale + m) * size + j * scale + n];
            sum = (int16_t)(!sat ? v : v < -16384 ? -16384 : v > 16383 ? 16383 : v); /* !sat: modulo 2^16 */
          }
        tmp2[i * size1 + j] = sum;
      }
    in = tmp2;
  }
  const int16_t *M = orc_dct_matrix(orc_log2i(size1));
  int shift1 = orc_log2i(size) + orc_log2i(scale) + bitdepth - 8, add1 = 1 << (shift1 - 1);
  int shift2 = orc_log2i(size1) + 5, add2 = 1 << (shift2 - 1);
  for (int i = 0; i < qsize; i++)
    for (int j = 0; j < size1; j++) {
      int sum = 0;
      for (int k = 0; k < size1; k++) sum += M[i * size1 + k] * in[j * size1 + k];
      tmp[i][j] = (int16_t)((sum + add1) >> shift1);
    }
  for (int i = 0; i < qsize; i++)
    for (int j = 0; j < qsize; j++) {
      int sum = 0;
      for (int k = 0; k < size1; k++) sum += M[i * size1 + k] * tmp[j][k];
      coeff[i * size + j] = (int16_t)((sum + add2) >> shift2);
    }
}

/* ---- a11: inverse transform.  common/transform.c:411-494 ---- */
static void orc_inverse_core(const int16_t *coeff, int16_t *block, int size, int bitdepth) {
  static int16_t tmp[32 * 32];
  int qsize = size < 16 ? size : 16, shift2 = 20 - bitdepth;
  const int16_t *M = orc_dct_matrix(orc_log2i(size));
  for (int i = 0; i < qsize; i++)
    for (int j = 0; j < size; j++) {
      int o = 0;
      for (int k = 0; k < qsize; k++) o += M[k * size + j] * coeff[k * size + i];
      o = (o + 64) >> 7;
      tmp[i * size + j] = (int16_t)(o < -32768 ? -32768 : o > 32767 ? 32767 : o);
    }
  for (int i = 0; i < size; i++)
    for (int j = 0; j < size; j++) {
      int o = 0;
      for (int k = 0; k < qsize; k++) o += M[k * size + j] * tmp[k * size + i];
      o = (o + (1 << (shift2 - 1))) >> shift2;
      block[i * size + j] = (int16_t)(o < -32768 ? -32768 : o > 32767 ? 32767 : o);
    }
}
void orc_inverse_transform(const int16_t *coeff, int16_t *block, int size, int bitdepth) {
  if (size < 64) { orc_inverse_core(coeff, block, size, bitdepth); return; }
  static int16_t c2[32 * 32], b2[32 * 32];
  int scale = size / 32;
  for (int i = 0; i < 32; i++) memcpy(c2 + i * 32, coeff + i * size, 32 * sizeof(int16_t));
  orc_inverse_core(c2, b2, 32, bitdepth);
  for (int i = 0; i < size; i++)
    for (int j = 0; j < size; j++) block[i * size + j] = b2[(i / scale) * 32 + j / scale];
}

/* ---- a12: quantisation.  enc/encode_block.c:84-160 ---- */
int orc_quantize(const int16_t *coeff, int16_t *coeffq, int qp, int size, int coeff_block_type, const uint16_t *wmatrix) {
  int intra = (coeff_block_type >> 1) & 1, qsize = size < 16 ? size : 16, nq = qsize * qsize;
  int64_t scale = orc_quant[qp % 6];
  int shift2 = 21 - orc_log2i(size) + qp / 6 + (wmatrix ? 6 : 0);
  const int *zz = orc_zigzag(qsize);
  int sc[256], sq[256];
  memset(sq, 0, sizeof(int) * (size_t)nq);
  for (int i = 0; i < qsize; i++)
    for (int j = 0; j < qsize; j++) {
      int v = coeff[i * size + j];
      if (wmatrix) v *= wmatrix[i * qsize + j];
      sc[zz[i * qsize + j]] = v;
    }
  int64_t offset = (int64_t)(intra ? 38 : -26) << (shift2 - 8);
  int level = 0, pos = nq - 1;
  while (level == 0 && pos >= 0) {
    int64_t l64 = (int64_t)abs(sc[pos]) * scale + offset;
    level = (int)((l64 > 0 ? l64 : -l64) >> shift2);
    pos--;
  }
  int last_pos = level ? pos + 1 : pos, cbp = 0, level_mode = 1;
  int off0 = intra ? 102 : 51, off1 = intra ? 115 : 90;
  for (pos = 0; pos <= last_pos; pos++) {
    int c = sc[pos], sign = c < 0 ? -1 : 1;
    int64_t ac = scale * abs(c);
    int level0 = (int)(ac >> shift2);
    int off = ((level0 > (1 - level_mode)) ? off1 : off0) << (shift2 - 8);
    level = (int)((ac + off) >> shift2);
    sq[pos] = sign * level;
    cbp |= level != 0;
    if (level_mode) { if (level == 0) level_mode = 0; }
    else if (level > 1) level_mode = 1;
  }
  for (int i = 0; i < nq; i++) coeffq[i] = (int16_t)sq[zz[i]];
  return cbp;
}

/* ---- a13: de-quantisation.  common/common_block.c:45-73 ---- */
void orc_dequantize(const int16_t *coeff, int16_t *rcoeff, int qp, int size, const uint16_t *wm) {
  int lshift = qp / 6, qsize = size < 16 ? size : 16, rshift = orc_log2i(size) - 1 + (wm ? 6 : 0);
  int64_t scale = orc_dequant[qp % 6], add = lshift < rshift ? (1 << (rshift - lshift - 1)) : 0;
  for (int i = 0; i < qsize; i++)
    for (int j = 0; j < qsize; j++) {
      int c = coeff[i * qsize + j];
      if (wm) c *= wm[i * qsize + j];
      rcoeff[i * size + j] = lshift >= rshift ? (int16_t)((c * scale) << (lshift - rshift)) : (int16_t)((c * scale + add) >> (rshift - lshift));
    }
}

/* ---- a14: chroma early-skip test ---- */
int orc_calc_cbp_c(const int16_t *block, int size, int thr) { /* enc/encode_block.c:2182-2212 */
  int step = size == 4 ? 2 : 1;
  for (int j = 0; j < size; j += step) {
    int sum = 0;
    for (int i = 0; i < size; i++) sum += block[i * size + j] + (step == 2 ? block[i * size + j + 1] : 0);
    if (abs(sum) > thr) return 1;
  }
  return 0;
}
int orc_calc_cbp(const int16_t *block, int size, int thr) { /* enc/enc_kernels.c:828-909: int16 column sums; 4x4 = odd + |even| */
  int16_t col[16];
  for (int j = 0; j < size; j++) {
    int16_t s = 0;
    for (int i = 0; i < size; i++) s = (int16_t)(s + block[i * size + j]);
    col[j] = s;
  }
  if (size == 4) {
    for (int j = 0; j < 4; j += 2) {
      int16_t a = (int16_t)(col[j] < 0 ? -col[j] : col[j]);
      if ((int)col[j + 1] + (int)a > thr) return 1;
    }
    return 0;
  }
  for (int j = 0; j < size; j++) {
    int16_t a = (int16_t)(col[j] < 0 ? -col[j] : col[j]);
    if (a > (int16_t)thr) return 1;
  }
  return 0;
}

/* common/common_kernels.c:127-161: 0 DC only, 1 only the top-left 4x4, 2 only the top-left 8x8, 3 otherwise */
int orc_check_nz_area(const int16_t *coeff, int size) {
  int qs = size < 16 ? size : 16, dc = 1, in4 = 1, in8 = 1;
  for (int i = 0; i < qs; i++)
    for (int j = 0; j < qs; j++) {
      if (!coeff[i * size + j]) continue;
      if (i || j) dc = 0;
      if (i >= 4 || j >= 4) in4 = 0;
      if (i >= 8 || j >= 8) in8 = 0;
    }
  if (size == 4) return dc ? 0 : 3;
  if (size == 8) return dc ? 0 : in4 ? 1 : 2;
  return dc ? 0 : in4 ? 1 : in8 ? 2 : 3;
}

/* ---- a6 ---- */
static int orc_mv_len(int d) { /* enc/encode_block.c:467-515 */
  int a = abs(d);
  if (a < 1) return 2;
  if (a < 2) return 4;
  if (a < 4) return 5;
  if (a < 36) return 5 + ((a - 4) >> 3) + 1;
  return 10 + ((a - 36) >> 4) + 1;
}
int orc_quote_mv_bits(int dy, int dx) { return orc_mv_len(dx) + orc_mv_len(dy); }

void orc_clip_mv(orc_mv_t *mv, int ypos, int xpos, int fwidth, int fheight, int bwidth, int bheight, int sign) { /* common/inter_prediction.c:51-63 */
  const int ext = 160 - 16;
  int mvy = sign ? -mv->y : mv->y, mvx = sign ? -mv->x : mv->x;
  if (ypos + mvy / 4 < -ext) mvy = 4 * (-ext - ypos);
  if (ypos + mvy / 4 + bheight > fheight + ext) mvy = 4 * (fheight + ext - ypos - bheight);
  if (xpos + mvx / 4 < -ext) mvx = 4 * (-ext - xpos);
  if (xpos + mvx / 4 + bwidth > fwidth + ext) mvx = 4 * (fwidth + ext - xpos - bwidth);
  mv->y = (int16_t)(sign ? -mvy : mvy);
  mv->x = (int16_t)(sign ? -mvx : mvx);
}

/* ---- a18/a19 shared scalar pieces.  common/common_block.c:214-220, 315-321 ---- */
static int orc_constrain(int diff, int threshold, unsigned damping) {
  if (!threshold) return 0;
  int a = abs(diff), lim = threshold - (a >> (damping - (unsigned)orc_log2i(threshold)));
  if (lim < 0) lim = 0;
  if (a < lim) lim = a;
  return diff < 0 ? -lim : lim;
}
int orc_clpf_sample(int X, int A, int B, int C, int D, int E, int F, int G, int H, int s, unsigned dmp) {
  int delta = orc_constrain(A - X, s, dmp) + 3 * orc_constrain(B - X, s, dmp) + orc_constrain(C - X, s, dmp) + 3 * orc_constrain(D - X, s, dmp) +
              3 * orc_constrain(E - X, s, dmp) + orc_constrain(F - X, s, dmp) + 3 * orc_constrain(G - X, s, dmp) + orc_constrain(H - X, s, dmp);
  return (8 + delta - (delta < 0)) >> 4;
}
int orc_adjust_strength(int strength, int32_t var) { /* common/common_frame.h:61-65 */
  int i = (var >> 6) ? (orc_log2i(var >> 6) < 12 ? orc_log2i(var >> 6) : 12) : 0;
  return var ? (strength * (4 + i) + 8) >> 4 : 0;
}
/* common/common_block.c:169-281 with CDEF_FULL = 0.  Tap offsets as (dy,dx) pairs, cdef_directions_x/y :189-208 */
static const int8_t orc_cdef_dx[8][2] = {{1, 2}, {1, 2}, {1, 2}, {1, 2}, {1, 2}, {0, 1}, {0, 0}, {0, -1}};
static const int8_t orc_cdef_dy[8][2] = {{-1, -2}, {0, -1}, {0, 0}, {0, 1}, {1, 2}, {1, 2}, {1, 2}, {1, 2}};
void orc_cdef_filter_block(uint8_t *dst8, uint16_t *dst16, int dstride, const uint16_t *in, int sstride, int pri_strength, int sec_strength,
                           int dir, int pri_damping, int sec_damping, int bsize, int coeff_shift) {
  static const int pri_taps[2][2] = {{4, 2}, {3, 3}}, sec_taps[2][2] = {{2, 1}, {2, 1}};
  const int *pt = pri_taps[(pri_strength >> coeff_shift) & 1], *st = sec_taps[(pri_strength >> coeff_shift) & 1];
  for (int i = 0; i < bsize; i++)
    for (int j = 0; j < bsize; j++) {
      int16_t sum = 0, x = (int16_t)in[i * sstride + j];
      int mx = x, mn = x;
      for (int k = 0; k < 2; k++) {
        int o0 = orc_cdef_dy[dir][k] * sstride + orc_cdef_dx[dir][k];
        int o1 = orc_cdef_dy[(dir + 2) & 7][k] * sstride + orc_cdef_dx[(dir + 2) & 7][k];
        int o2 = orc_cdef_dy[(dir + 6) & 7][k] * sstride + orc_cdef_dx[(dir + 6) & 7][k];
        int16_t p[2] = {(int16_t)in[i * sstride + j + o0], (int16_t)in[i * sstride + j - o0]};
        int16_t s[4] = {(int16_t)in[i * sstride + j + o1], (int16_t)in[i * sstride + j - o1], (int16_t)in[i * sstride + j + o2], (int16_t)in[i * sstride + j - o2]};
        for (int t = 0; t < 2; t++) {
          sum = (int16_t)(sum + pt[k] * orc_constrain(p[t] - x, pri_strength, (unsigned)pri_damping));
          if (p[t] != 30000 && p[t] > mx) mx = p[t];
          if (p[t] < mn) mn = p[t];
        }
        for (int t = 0; t < 4; t++) {
          sum = (int16_t)(sum + st[k] * orc_constrain(s[t] - x, sec_strength, (unsigned)sec_damping));
          if (s[t] != 30000 && s[t] > mx) mx = s[t];
          if (s[t] < mn) mn = s[t];
        }
      }
      int y = x + ((8 + sum - (sum < 0)) >> 4);
      y = y < mn ? mn : y > mx ? mx : y;
      if (dst8) dst8[i * dstride + j] = (uint8_t)y;
      else dst16[i * dstride + j] = (uint16_t)y;
    }
}

/* ---- a19 (encoder): preset selection of cdef_search.  enc/encode_frame.c:58-192 (greedy joint search, dual = luma + chroma)
 * and :378-470 (sort, de-duplicate, per-block assignment).  mse0/mse1: [sb_count][64] for the non-all-skip filter blocks.
 * Outputs: strengths[8], uv_strengths[8] (already mapped through priconv), selected[sb_count]; returns nb_strength_bits. */
static uint64_t orc_search_one_dual(int *lev0, int *lev1, int nb, const uint64_t *m0, const uint64_t *m1, int sb_count, int total) {
  static uint64_t tot[64][64];
  memset(tot, 0, sizeof(tot));
  for (int i = 0; i < sb_count; i++) {
    uint64_t best = (uint64_t)1 << 63;
    for (int g = 0; g < nb; g++) {
      uint64_t c = m0[i * 64 + lev0[g]] + m1[i * 64 + lev1[g]];
      if (c < best) best = c;
    }
    for (int j = 0; j < total; j++)
      for (int k = 0; k < total; k++) {
        uint64_t c = m0[i * 64 + j] + m1[i * 64 + k];
        tot[j][k] += c < best ? c : best;
      }
  }
  uint64_t bt = (uint64_t)1 << 63;
  int b0 = 0, b1 = 0;
  for (int j = 0; j < total; j++)
    for (int k = 0; k < total; k++)
      if (tot[j][k] < bt) { bt = tot[j][k]; b0 = j; b1 = k; }
  lev0[nb] = b0;
  lev1[nb] = b1;
  return bt;
}
static int orc_u32_cmp(const void *a, const void *b) { return *(const uint32_t *)a < *(const uint32_t *)b ? -1 : *(const uint32_t *)a > *(const uint32_t *)b; }
int orc_cdef_select(const uint64_t *mse0, const uint64_t *mse1, int sb_count, int speed, int cdef_bits, double lambda, int *strengths, int *uv_strengths, int *selected) {
  static const int priconv[3][16] = {{0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {0, 1, 2, 3, 5, 7, 10, 13}, {0, 1, 3, 6}};
  static const int pristrengths[3] = {64, 32, 16};
  const int total = pristrengths[speed], nb = 1 << cdef_bits;
  int lev0[16], lev1[16] = {0};
  uint64_t tot = 0;
  for (int i = 0; i < nb; i++) tot = orc_search_one_dual(lev0, lev1, i, mse0, mse1, sb_count, total);
  for (int i = 0; i < 4 * nb; i++) {
    for (int j = 0; j < nb - 1; j++) { lev0[j] = lev0[j + 1]; lev1[j] = lev1[j + 1]; }
    tot = orc_search_one_dual(lev0, lev1, nb - 1, mse0, mse1, sb_count, total);
  }
  tot += (uint64_t)(sb_count * lambda * cdef_bits);
  tot += (uint64_t)(nb * lambda * 6);
  (void)tot;  /* a single bit budget is tried (encode_frame.c:385), so the total only mirrors the reference */
  for (int j = 0; j < nb; j++) { strengths[j] = lev0[j]; uv_strengths[j] = lev1[j]; }
  int gi_trans[8];
  uint32_t list[8];
  for (int i = 0; i < nb; i++) list[i] = ((uint32_t)strengths[i] << 16) + ((uint32_t)uv_strengths[i] << 8) + (uint32_t)i;
  qsort(list, (size_t)nb, sizeof(*list), orc_u32_cmp);
  int j = 0;
  for (int i = 0; i < nb; i++) {
    gi_trans[list[i] & 255] = j;
    if (!i || (list[i] & ~255u) != (list[i - 1] & ~255u)) {
      strengths[j] = (int)(list[i] >> 16);
      uv_strengths[j++] = (int)((list[i] >> 8) & 255);
    }
  }
  const int bits = orc_log2i(j), nstr = 1 << bits;
  for (int i = 0; i < sb_count; i++) {
    uint64_t best = (uint64_t)1 << 63;
    int bg = 0;
    for (int g = 0; g < (1 << bits); g++) {
      uint64_t c = mse0[i * 64 + strengths[gi_trans[g]]] + mse1[i * 64 + uv_strengths[gi_trans[g]]];
      if (c < best) { bg = gi_trans[g] < nstr - 1 ? gi_trans[g] : nstr - 1; best = c; }
    }
    selected[i] = bg;
  }
  for (int q = 0; q < nstr; q++) {
    strengths[q] = priconv[speed][strengths[q] / 4] * 4 + strengths[q] % 4;
    uv_strengths[q] = priconv[speed][uv_strengths[q] / 4] * 4 + uv_strengths[q] % 4;
  }
  return bits;
}

#define S uint8_t
#define FN(x) x##_lbd
#include "thor_oracle_tmpl.h"
#undef S
#undef FN
#define S uint16_t
#define FN(x) x##_hbd
#include "thor_oracle_tmpl.h"
#undef S
#undef FN

/* ------------------------------------------------------------------------------------------------------------------
 * SURVEY 8f.2 (first part): number of bits write_coeff() emits for one transform block.  enc/write_bits.c:145-242 with the
 * code lengths of put_vlc(), enc/putvlc.c:73-161 (tables 0/1: Golomb-like with e = 5; 6: cn+1 on table 2 with a 2-bit zero;
 * 10: Elias-gamma of cn+1).  coeff: min(size,16)^2 quantised coefficients in raster order.  Returns 0 for an all-zero block
 * (the reference never calls write_coeff for one).
 * ------------------------------------------------------------------------------------------------------------------ */
static int orc_log2u(unsigned x) { int n = 0; while (x >>= 1) n++; return n; }
int orc_vlc_len(int n, unsigned cn) {
  if (n == 6) {
    if (!cn) return 2;
    cn++;
    n = 2;
  } else if (n == 10)
    return 1 + 2 * orc_log2u(cn + 1);
  if ((int)cn < 5 * (1 << n)) return 1 + n + (int)(cn >> n);
  return (5 - n) + 1 + 2 * orc_log2u(cn - 5u * (1u << n) + (1u << n));
}
int orc_coeff_bits(const int16_t *coeff, int size, int type) {
  int16_t sc[256];
  const int qsize = size < 16 ? size : 16, N = qsize * qsize;
  const int chroma = type & 1, intra = (type >> 1) & 1;
  int vlc_adaptive = intra && !chroma;
  const unsigned eob_pos = chroma ? 0 : 2;
  const int run_tab = chroma && size <= 8 ? 10 : 6;
  const int *zz = orc_zigzag(qsize);
  int bits = 0, pos, last_pos, level_mode = 1, level = 1, c = 0;
  for (int i = 0; i < N; i++) sc[zz[i]] = coeff[i];
  for (pos = N - 1; !sc[pos] && pos; pos--);
  if (!pos && !sc[0]) return 0;
  last_pos = pos;
  pos = 0;
  if (chroma) {
    if (last_pos == 0 && (sc[0] == 1 || sc[0] == -1)) { bits += 2; pos = N; }
    else bits += 1;
  }
  while (pos <= last_pos) {
    if (level_mode) {
      while (pos <= last_pos && level > 0) {
        c = sc[pos++];
        level = c < 0 ? -c : c;
        bits += orc_vlc_len(vlc_adaptive, (unsigned)level);
        if (level > 0) bits += 1;
        if (!chroma) vlc_adaptive = level > 3;
      }
    }
    int run = 0;
    c = 0;
    while (c == 0 && pos <= last_pos) {
      c = sc[pos++];
      run += !c;
      if (c) {
        unsigned cn;
        level = c < 0 ? -c : c;
        cn = level == 1 ? (unsigned)(run * 5) / 4 : (unsigned)(run * 5 + 4);
        bits += orc_vlc_len(run_tab, cn + (cn >= eob_pos));
        level_mode = level > 1;
        bits += level > 1 ? orc_vlc_len(0, (unsigned)((level - 2) * 2 + (c < 0))) : 1;
        run = 0;
      }
    }
  }
  if (pos < N && level_mode) { bits += orc_vlc_len(vlc_adaptive, 0); pos++; }
  if (pos < N) bits += orc_vlc_len(run_tab, eob_pos);
  return bits;
}
