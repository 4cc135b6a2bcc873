/* thor_oracle_tmpl.h — TEST INFRASTRUCTURE ONLY; included twice by thor_oracle.c with
 *   S = uint8_t,  FN(x) = x##_lbd     and     S = uint16_t, FN(x) = x##_hbd.
 * Scalar restatement of the sample-typed half of the Thor hot path.  Citations are /root/reference paths.
 */

/* ---- a1: SAD.  enc/encode_block.c:417-428 (C), enc/enc_kernels.c:36-81 (SIMD, same value) ---- */
unsigned FN(orc_sad)(const S *a, const S *b, int astride, int bstride, int width, int height) {
  unsigned sad = 0;
  for (int i = 0; i < height; i++)
    for (int j = 0; j < width; j++) sad += (unsigned)abs((int)a[i * astride + j] - (int)b[i * bstride + j]);
  return sad;
}

/* ---- a2: five-position wide SAD.  enc/encode_block.c:430-453; SIMD tie rule enc/enc_kernels.c:110-114
 * (lowest packed (sad<<3)|idx) == first strict minimum in offset order -3,-1,0,1,3. ---- */
unsigned FN(orc_widesad)(const S *a, const S *b, int astride, int bstride, int width, int height, int *x) {
  static const int off[5] = {-3, -1, 0, 1, 3};
  unsigned best = 1u << 31;
  int bestx = 0;
  for (int k = 0; k < 5; k++) {
    unsigned sad = FN(orc_sad)(a, b + off[k], astride, bstride, width, height);
    if (sad < best) { best = sad; bestx = off[k]; }
  }
  *x = bestx;
  return best;
}

/* ---- a3: SSD.  enc/encode_block.c:455-465, enc/enc_kernels.c:119 ---- */
uint64_t FN(orc_ssd)(const S *a, const S *b, int astride, int bstride, int width, int height) {
  uint64_t ssd = 0;
  for (int i = 0; i < height; i++)
    for (int j = 0; j < width; j++) {
      int d = (int)a[i * astride + j] - (int)b[i * bstride + j];
      ssd += (uint64_t)(d * d);
    }
  return ssd;
}

/* ---- a4: bilinear half-pel SAD approximation.  enc/encode_block.c:174-283.
 * up(x,y) = (x+y+1)>>1 (SIMD avg), dn(x,y) = (x+y)>>1 (SIMD rdavg), common/simd/v64_intrinsics_c.h:736-750.
 * Eight positions; winner chosen in the fixed order top,down,right,left,tl,tr,br,bl with strict '<'. ---- */
#define ORC_UP(x, y) (((int)(x) + (int)(y) + 1) >> 1)
#define ORC_DN(x, y) (((int)(x) + (int)(y)) >> 1)
unsigned FN(orc_sad_fasthalf)(const S *a, const S *b, int astride, int bstride, int width, int height, int *x, int *y) {
  unsigned acc[8] = {0}; /* top, down, right, left, tl, tr, br, bl */
  for (int i = 0; i < height; i++) {
    const S *r = b + i * bstride;
    for (int j = 0; j < width; j++) {
      int o = a[i * astride + j];
#define P(dy, dx) ((int)r[(dy) * bstride + j + (dx)])
      /* horizontal / vertical half-pels of the four pixels around each diagonal position */
      int hL = ORC_UP(P(0, -1), P(0, 0));   /* left  of centre, row 0 */
      int hR = ORC_UP(P(0, 0), P(0, 1));    /* right of centre, row 0 */
      int hLu = ORC_UP(P(-1, -1), P(-1, 0)), hRu = ORC_UP(P(-1, 0), P(-1, 1));
      int hLd = ORC_UP(P(1, -1), P(1, 0)), hRd = ORC_UP(P(1, 0), P(1, 1));
      /* column pairs two rows apart (outer taps), for columns j-1, j, j+1; upper (-2,+1) and lower (-1,+2) */
      int vU_m = ORC_UP(P(-2, -1), P(1, -1)), vU_0 = ORC_UP(P(-2, 0), P(1, 0)), vU_p = ORC_UP(P(-2, 1), P(1, 1));
      int vD_m = ORC_UP(P(-1, -1), P(2, -1)), vD_0 = ORC_UP(P(-1, 0), P(2, 0)), vD_p = ORC_UP(P(-1, 1), P(2, 1));
      /* row pairs three columns apart, rows -1, 0, +1; left (-2,+1) and right (-1,+2) */
      int wL_u = ORC_UP(P(-1, -2), P(-1, 1)), wL_0 = ORC_UP(P(0, -2), P(0, 1)), wL_d = ORC_UP(P(1, -2), P(1, 1));
      int wR_u = ORC_UP(P(-1, -1), P(-1, 2)), wR_0 = ORC_UP(P(0, -1), P(0, 2)), wR_d = ORC_UP(P(1, -1), P(1, 2));
      int ptl = ORC_DN(ORC_DN(ORC_DN(vU_m, vU_0), ORC_DN(wL_u, wL_0)), ORC_DN(hLu, hL));
      int ptr = ORC_DN(ORC_DN(ORC_DN(vU_0, vU_p), ORC_DN(wR_0, wR_u)), ORC_DN(hRu, hR));
      int pbl = ORC_DN(ORC_DN(ORC_DN(vD_0, vD_m), ORC_DN(wL_0, wL_d)), ORC_DN(hLd, hL));
      int pbr = ORC_DN(ORC_DN(ORC_DN(vD_0, vD_p), ORC_DN(wR_0, wR_d)), ORC_DN(hR, hRd));
      acc[0] += (unsigned)abs(o - ORC_UP(P(0, 0), P(-1, 0)));
      acc[1] += (unsigned)abs(o - ORC_UP(P(0, 0), P(1, 0)));
      acc[2] += (unsigned)abs(o - hR);
      acc[3] += (unsigned)abs(o - hL);
      acc[4] += (unsigned)abs(o - ptl);
      acc[5] += (unsigned)abs(o - ptr);
      acc[6] += (unsigned)abs(o - pbr);
      acc[7] += (unsigned)abs(o - pbl);
#undef P
    }
  }
  static const int bx[8] = {0, 0, 2, -2, -2, 2, 2, -2};
  static const int by[8] = {-2, 2, 0, 0, -2, -2, 2, 2};
  int best = 0;
  for (int k = 1; k < 8; k++)
    if (acc[k] < acc[best]) best = k;
  *x = bx[best];
  *y = by[best];
  return acc[best];
}

/* ---- a4: bilinear quarter-pel SAD approximation.  enc/encode_block.c:286-414.  *x,*y are in/out: on entry the
 * half-pel offset of the current best (only their low bits select the formula set). ---- */
unsigned FN(orc_sad_fastquarter)(const S *o, const S *r, int os, int rs, int width, int height, int *x, int *y) {
  unsigned acc[8] = {0}; /* top, tl, tr, left, right, bl, down, br : evaluation order of the final compare */
  int fx = *x, fy = *y;
  for (int i = 0; i < height; i++) {
    const S *q = r + i * rs;
    for (int j = 0; j < width; j++) {
      int org = o[i * os + j];
      int a = q[j], d = q[j + 1], f = q[j + rs], e = q[j + rs + 1];
      int vtop, vtl, vtr, vleft, vright, vbl, vdown, vbr;
      if (fx & fy) {
        int ad = ORC_UP(a, d), de = ORC_UP(d, e), af = ORC_UP(a, f), fe = ORC_UP(f, e);
        vtl = ORC_DN(ad, af); vtop = ORC_DN(de, a); vtr = ORC_DN(ad, de); vleft = ORC_DN(ad, f);
        vright = ORC_DN(ad, e); vbl = ORC_DN(af, fe); vdown = ORC_DN(de, f); vbr = ORC_DN(de, fe);
      } else if (fx) {
        int b = q[j - rs], c = q[j - rs + 1];
        int ad = ORC_UP(a, d), de = ORC_UP(d, e), dc = ORC_UP(d, c), af = ORC_UP(a, f), ab = ORC_UP(a, b);
        vtl = ORC_DN(ad, ab); vtop = ORC_DN(dc, a); vtr = ORC_DN(ad, dc); vleft = ORC_DN(ad, a);
        vright = ORC_DN(ad, d); vbl = ORC_DN(ad, af); vdown = ORC_DN(af, d); vbr = ORC_DN(ad, de);
      } else if (fy) {
        int g = q[j + rs - 1], h = q[j - 1];
        int ad = ORC_UP(a, d), af = ORC_UP(a, f), fe = ORC_UP(f, e), ah = ORC_UP(a, h), gf = ORC_UP(g, f);
        vtl = ORC_DN(ah, af); vtop = ORC_DN(af, a); vtr = ORC_DN(ad, af); vleft = ORC_DN(gf, a);
        vright = ORC_DN(ad, f); vbl = ORC_DN(af, gf); vdown = ORC_DN(af, f); vbr = ORC_DN(af, fe);
      } else {
        int b = q[j - rs], h = q[j - 1];
        int ad = ORC_UP(a, d), af = ORC_UP(a, f), ah = ORC_UP(a, h), ab = ORC_UP(a, b);
        vtl = ORC_DN(ah, ab); vtop = ORC_DN(ab, a); vtr = ORC_DN(ad, ab); vleft = ORC_DN(ah, a);
        vright = ORC_DN(ad, a); vbl = ORC_DN(ah, af); vdown = ORC_DN(af, a); vbr = ORC_DN(af, ad);
      }
      acc[0] += (unsigned)abs(org - vtop);  acc[1] += (unsigned)abs(org - vtl);
      acc[2] += (unsigned)abs(org - vtr);   acc[3] += (unsigned)abs(org - vleft);
      acc[4] += (unsigned)abs(org - vright); acc[5] += (unsigned)abs(org - vbl);
      acc[6] += (unsigned)abs(org - vdown); acc[7] += (unsigned)abs(org - vbr);
    }
  }
  static const int bx[8] = {0, -1, 1, -1, 1, -1, 0, 1};
  static const int by[8] = {-1, -1, -1, 0, 0, 1, 1, 1};
  int best = 0;
  for (int k = 1; k < 8; k++)
    if (acc[k] < acc[best]) best = k;
  *x = bx[best];
  *y = by[best];
  return acc[best];
}

/* ---- a9: rounding block average, (a+b+1)>>1.  common/common_kernels.c:38-66 ---- */
void FN(orc_block_avg)(S *p, const S *r0, const S *r1, int sp, int s0, int s1, int width, int height) {
  for (int i = 0; i < height; i++)
    for (int j = 0; j < width; j++) p[i * sp + j] = (S)ORC_UP(r0[i * s0 + j], r1[i * s1 + j]);
}

/* ---- a7: quarter-pel luma interpolation at a fractional position (xoff,yoff), ip already at the integer
 * position.  common/inter_prediction.c:146-180 (C), common/common_kernels.c:1930-2190 (SIMD; same values). ---- */
static const int8_t FN(orc_luma_taps)[2][4][6] = {
    {{0, 0, 64, 0, 0, 0}, {1, -7, 55, 19, -5, 1}, {1, -7, 38, 38, -7, 1}, {1, -5, 19, 55, -7, 1}},
    {{0, 0, 64, 0, 0, 0}, {2, -10, 59, 17, -5, 1}, {1, -8, 39, 39, -8, 1}, {1, -5, 17, 59, -10, 2}}};
static const int8_t FN(orc_chroma_taps)[8][4] = {{0, 64, 0, 0},  {-2, 58, 10, -2}, {-4, 54, 16, -2}, {-4, 44, 28, -4},
                                                 {-4, 36, 36, -4}, {-4, 28, 44, -4}, {-2, 16, 54, -4}, {-2, 10, 58, -2}};

/* The SIMD edge filters (exactly one fraction non-zero; common/common_kernels_gen.c:1964-1999 luma, :2222-2253 chroma) shift 16-bit
 * samples right by bitdepth - 10.  At bit depth 8 that count is -2, which the x86 shift takes as a huge unsigned count: every lane becomes
 * 0 or -1, and the saturating pack makes the prediction 0.  The reference's encoder predicts these zeros (-frame_bitdepth 16 with 8-bit
 * input); its decoder works in 8-bit samples at bit depth 8 and filters normally, so it does not reconstruct what such an encoder did. */
static int FN(orc_edge_zero)(int xoff, int yoff, int bitdepth) { return sizeof(S) == 2 && bitdepth == 8 && !xoff != !yoff; }

void FN(orc_interp_luma)(int width, int height, int xoff, int yoff, S *qp, int qstride, const S *ip, int istride, int bipred, int bitdepth) {
  int maxv = (1 << bitdepth) - 1;
  if (FN(orc_edge_zero)(xoff, yoff, bitdepth)) {
    for (int i = 0; i < height; i++) memset(qp + i * qstride, 0, (size_t)width * sizeof(S));
    return;
  }
  if (xoff == 2 && yoff == 2 && bipred < 2) {
    /* 12-tap 4x4 low-pass at the centre position: corners 0, edges 1, middle 2; (sum+8)>>4 */
    static const int8_t w[4][4] = {{0, 1, 1, 0}, {1, 2, 2, 1}, {1, 2, 2, 1}, {0, 1, 1, 0}};
    for (int i = 0; i < height; i++)
      for (int j = 0; j < width; j++) {
        int sum = 0;
        for (int m = 0; m < 4; m++)
          for (int n = 0; n < 4; n++) sum += w[m][n] * (int)ip[(i + m - 1) * istride + j + n - 1];
        sum = (sum + 8) >> 4;
        qp[i * qstride + j] = (S)(sum < 0 ? 0 : sum > maxv ? maxv : sum);
      }
    return;
  }
  const int8_t *fv = FN(orc_luma_taps)[bipred ? 1 : 0][yoff];
  const int8_t *fh = FN(orc_luma_taps)[bipred ? 1 : 0][xoff];
  for (int i = 0; i < height; i++)
    for (int j = 0; j < width; j++) {
      int sum = 0;
      for (int n = 0; n < 6; n++) {
        int col = 0;
        for (int m = 0; m < 6; m++) col += fv[m] * (int)ip[(i + m - 2) * istride + j + n - 2];
        sum += fh[n] * col;
      }
      sum = (sum + 2048) >> 12;
      qp[i * qstride + j] = (S)(sum < 0 ? 0 : sum > maxv ? maxv : sum);
    }
}

/* ---- a8: eighth-pel 4-tap chroma.  common/inter_prediction.c:94-114, common/common_kernels.c:2192-2375 ---- */
void FN(orc_interp_chroma)(int width, int height, int xoff, int yoff, S *qp, int qstride, const S *ip, int istride, int bitdepth) {
  int maxv = (1 << bitdepth) - 1;
  if (width > 2 && FN(orc_edge_zero)(xoff, yoff, bitdepth)) { /* 2-wide blocks take the C filter (common/inter_prediction.c:92) */
    for (int i = 0; i < height; i++) memset(qp + i * qstride, 0, (size_t)width * sizeof(S));
    return;
  }
  const int8_t *fh = FN(orc_chroma_taps)[xoff], *fv = FN(orc_chroma_taps)[yoff];
  for (int i = 0; i < height; i++)
    for (int j = 0; j < width; j++) {
      int sum = 0;
      for (int m = 0; m < 4; m++) {
        int row = 0;
        for (int n = 0; n < 4; n++) row += fh[n] * (int)ip[(i + m - 1) * istride + j + n - 1];
        sum += fv[m] * row;
      }
      sum = (sum + 2048) >> 12;
      qp[i * qstride + j] = (S)(sum < 0 ? 0 : sum > maxv ? maxv : sum);
    }
}

/* ---- a7: full get_inter_prediction_luma incl. the normative clamp (note: lower clamps use xpos for both axes).
 * common/inter_prediction.c:117-180 ---- */
void FN(orc_get_inter_prediction_luma)(S *pblock, const S *ref, int width, int height, int stride, int pstride, const orc_mv_t *mv,
                                       int sign, int bipred, int pic_width, int pic_height, int xpos, int ypos, int bitdepth) {
  int mvx = sign ? -mv->x : mv->x, mvy = sign ? -mv->y : mv->y;
  int ver_frac = mvy & 3, hor_frac = mvx & 3, ver_int = mvy >> 2, hor_int = mvx >> 2;
  if (ver_int > pic_height - ypos) ver_int = pic_height - ypos;
  if (ver_int < -xpos - height) ver_int = -xpos - height;
  if (hor_int > pic_width - xpos) hor_int = pic_width - xpos;
  if (hor_int < -xpos - width) hor_int = -xpos - width;
  const S *ip = ref + ver_int * stride + hor_int;
  if (!ver_frac && !hor_frac) {
    for (int i = 0; i < height; i++) memcpy(pblock + i * pstride, ip + i * stride, (size_t)width * sizeof(S));
    return;
  }
  FN(orc_interp_luma)(width, height, hor_frac, ver_frac, pblock, pstride, ip, stride, bipred, bitdepth);
}

/* common/inter_prediction.c:65-114 */
void FN(orc_get_inter_prediction_chroma)(S *pblock, const S *ref, int width, int height, int stride, int pstride, const orc_mv_t *mv,
                                         int sign, int pic_width2, int pic_height2, int xpos, int ypos, int bitdepth) {
  int mvx = sign ? -mv->x : mv->x, mvy = sign ? -mv->y : mv->y;
  int ver_frac = mvy & 7, hor_frac = mvx & 7, ver_int = mvy >> 3, hor_int = mvx >> 3;
  if (ver_int > pic_height2 - ypos) ver_int = pic_height2 - ypos;
  if (ver_int < -xpos - height) ver_int = -xpos - height;
  if (hor_int > pic_width2 - xpos) hor_int = pic_width2 - xpos;
  if (hor_int < -xpos - width) hor_int = -xpos - width;
  const S *ip = ref + ver_int * stride + hor_int;
  if (!ver_frac && !hor_frac) {
    for (int i = 0; i < height; i++) memcpy(pblock + i * pstride, ip + i * stride, (size_t)width * sizeof(S));
    return;
  }
  FN(orc_interp_chroma)(width, height, hor_frac, ver_frac, pblock, pstride, ip, stride, bitdepth);
}

/* ---- a13: residual / reconstruct.  enc/encode_block.c:162-171, common/common_block.c:75-83 ---- */
void FN(orc_residual)(int16_t *block, const S *pblock, const S *orig, int size, int pred_stride, int orig_stride) {
  for (int i = 0; i < size; i++)
    for (int j = 0; j < size; j++) block[i * size + j] = (int16_t)((int)orig[i * orig_stride + j] - (int)pblock[i * pred_stride + j]);
}
void FN(orc_reconstruct)(const int16_t *block, const S *pblock, S *rec, int size, int pstride, int stride, int bitdepth) {
  int maxv = (1 << bitdepth) - 1;
  for (int i = 0; i < size; i++)
    for (int j = 0; j < size; j++) {
      int v = block[i * size + j] + (int16_t)pblock[i * pstride + j];
      rec[i * stride + j] = (S)(v < 0 ? 0 : v > maxv ? maxv : v);
    }
}

/* ---- a15: intra neighbour gather.  common/intra_prediction.c:57-183.  (i,j) = TU offset inside the coding
 * block at (ypos,xpos); rec_frame points at the TU's top-left sample in the frame, rblock likewise in the
 * block-local reconstruction buffer. ---- */
void FN(orc_make_top_and_left)(S *left, S *top, S *top_left, const S *rec_frame, int fstride, const S *rblock, int rbstride, int i, int j,
                               int ypos, int xpos, int size, int cb_upright, int cb_downleft, int tb_split, int bitdepth) {
  S mid = (S)(128 << (bitdepth - 8));
  int downleft, upright;
  if (!tb_split) { downleft = cb_downleft; upright = cb_upright; }
  else {
    downleft = (j == 0 && (i == 0 || cb_downleft)) ? 1 : 0;
    upright = (j == 0 || (i == 0 && cb_upright)) ? 1 : 0;
  }
  int leftlen = downleft ? size + 1 : size, toplen = upright ? size + 1 : size;
  /* rec_frame = the coding block's top-left sample in the frame; rblock = this TU's top-left sample in the
   * block-local reconstruction.  The non-split branch asserts i == j == 0, so one set of formulas serves both. */
  if (ypos + i == 0) {
    for (int k = 0; k < 2 * size; k++) top[k] = mid;
    *top_left = mid;
  } else {
    const S *src = (i == 0) ? rec_frame - fstride + j : rblock - rbstride;
    for (int k = 0; k < toplen; k++) top[k] = src[k];
    S val = top[toplen - 1];
    for (int k = 0; k < size; k++) top[size + k] = val;
    if (xpos > 0) {
      if (i == 0) *top_left = rec_frame[-fstride + j - 1];
      else *top_left = (j > 0) ? rblock[-rbstride - 1] : rec_frame[(i - 1) * fstride - 1];
    } else
      *top_left = top[0];
  }
  if (xpos + j == 0) {
    for (int k = 0; k < 2 * size; k++) left[k] = mid;
  } else {
    for (int k = 0; k < leftlen; k++) left[k] = (j == 0) ? rec_frame[(i + k) * fstride - 1] : rblock[k * rbstride - 1];
    S val = left[leftlen - 1];
    for (int k = 0; k < size; k++) left[size + k] = val;
  }
  if (ypos + i == 0) *top_left = left[0];
}

static void FN(orc_f121)(const S *in, S *out, int len) {
  out[0] = (S)((in[0] + 2 * in[0] + in[1] + 2) >> 2);
  for (int k = 1; k < len - 1; k++) out[k] = (S)((in[k - 1] + 2 * in[k] + in[k + 1] + 2) >> 2);
  out[len - 1] = (S)((in[len - 2] + 2 * in[len - 1] + in[len - 1] + 2) >> 2);
}

/* ---- a15: the ten predictors + dispatcher.  common/intra_prediction.c:185-428.  mode numbering
 * common/types.h:189-201: 0 DC,1 PLANAR,2 HOR,3 VER,4 UPLEFT,5 UPRIGHT,6 UPUPRIGHT,7 UPUPLEFT,8 UPLEFTLEFT,9 DOWNLEFTLEFT */
void FN(orc_intra_pred)(const S *left, const S *top, S top_left, int ypos, int xpos, int size, S *pblock, int pstride, int mode, int bitdepth) {
  S tF[2 * 128], lF[2 * 128], tlF = 0;
  int maxv = (1 << bitdepth) - 1;
  if (mode < 0 || mode > 9) mode = 0;
  if (mode == 4 || mode == 7 || mode == 8) {
    FN(orc_f121)(left, lF, size);
    FN(orc_f121)(top, tF, size);
    tlF = (S)((2 * top_left + left[0] + top[0] + 2) >> 2);
  } else if (mode == 5 || mode == 6) FN(orc_f121)(top, tF, 2 * size);
  else if (mode == 9) FN(orc_f121)(left, lF, 2 * size);
  int16_t ptF[128], plF[128], ptlF = 0;
  unsigned dc = 0;
  if (mode == 0) {
    const S *l = xpos != 0 ? left : top, *t = ypos != 0 ? top : left;
    unsigned sum = 0;
    for (int k = 0; k < size; k++) sum += t[k];
    for (int k = 0; k < size; k++) sum += l[k];
    dc = (sum + (unsigned)size) / (2u * (unsigned)size);
  } else if (mode == 1) {
    /* 5-tap (1,2,2,2,1) smoothing with edge replication; int16 like the reference */
    for (int k = 0; k < size; k++) {
      int a = k - 2 < 0 ? 0 : k - 2, b = k - 1 < 0 ? 0 : k - 1, c = k + 1 > size - 1 ? size - 1 : k + 1, d = k + 2 > size - 1 ? size - 1 : k + 2;
      ptF[k] = (int16_t)(top[a] + 2 * top[b] + 2 * top[k] + 2 * top[c] + top[d]);
      plF[k] = (int16_t)(left[a] + 2 * left[b] + 2 * left[k] + 2 * left[c] + left[d]);
    }
    ptlF = (int16_t)(left[1] + 2 * left[0] + 2 * top_left + 2 * top[0] + top[1]);
  }
  for (int i = 0; i < size; i++)
    for (int j = 0; j < size; j++) {
      int v, d;
      switch (mode) {
        case 0: v = (int)dc; break;
        case 1: { v = (plF[i] + ptF[j] - ptlF + 4) / 8; v = v < 0 ? 0 : v > maxv ? maxv : v; } break;
        case 2: v = left[i]; break;
        case 3: v = top[j]; break;
        case 4: d = i - j; v = d > 0 ? lF[d - 1] : d == 0 ? tlF : tF[-d - 1]; break;
        case 5: v = tF[i + j + 1]; break;
        case 6: d = i + 2 * j; v = (d & 1) ? tF[(d + 1) / 2] : (tF[d / 2] + tF[d / 2 + 1]) >> 1; break;
        case 7: d = i - 2 * j;
          if (d > 1) v = lF[d - 2]; else if (d == 1) v = tlF; else if (d == 0) v = (tlF + tF[0]) >> 1;
          else v = (d & 1) ? tF[(-d) / 2] : (tF[(-d) / 2] + tF[(-d) / 2 - 1]) >> 1;
          break;
        case 8: d = 2 * i - j;
          if (d < -1) v = tF[-d - 2]; else if (d == -1) v = tlF; else if (d == 0) v = (tlF + lF[0]) >> 1;
          else v = (d & 1) ? lF[d / 2] : (lF[d / 2] + lF[d / 2 - 1]) >> 1;
          break;
        default: d = 2 * i + j; v = (d & 1) ? lF[(d + 1) / 2] : (lF[d / 2] + lF[d / 2 + 1]) >> 1; break;
      }
      pblock[i * pstride + j] = (S)v;
    }
}

/* ---- a16: chroma-from-luma.  common/common_block.c:347-427 ---- */
void FN(orc_cfl)(const S *y, S *u, S *v, const S *ry, int n, int cstride, int stride, int sub, int bitdepth) {
  int nc = n >> sub, lognc = orc_log2i(nc), cs = cstride >> sub, maxv = (1 << bitdepth) - 1;
  int64_t sq = 0;
  for (int i = 0; i < n; i++)
    for (int j = 0; j < n; j++) { int d = (int)ry[i * stride + j] - (int)y[i * n + j]; sq += d * d; }
  if ((sq >> (2 * orc_log2i(n))) <= (64 << 2 * (bitdepth - 8))) return;
  int64_t ysum = 0, usum = 0, vsum = 0, yy = 0, yu = 0, yv = 0, uu = 0, vv = 0;
  for (int i = 0; i < nc; i++)
    for (int j = 0; j < nc; j++) {
      int us = u[i * cs + j], vs = v[i * cs + j];
      int ys = sub ? (y[(2 * i) * n + 2 * j] + y[(2 * i) * n + 2 * j + 1] + y[(2 * i + 1) * n + 2 * j] + y[(2 * i + 1) * n + 2 * j + 1] + 2) >> 2
                   : y[i * cstride + j];
      ysum += ys; usum += us; vsum += vs;
      yy += ys * ys; yu += ys * us; yv += ys * vs; uu += us * us; vv += vs * vs;
    }
  int sh = lognc * 2;
  int64_t ssyy = yy - (ysum * ysum >> sh), ssuu = uu - (usum * usum >> sh), ssvv = vv - (vsum * vsum >> sh);
  int64_t ssyu = yu - (ysum * usum >> sh), ssyv = yv - (ysum * vsum >> sh);
  if (!ssyy) return;
  for (int c = 0; c < 2; c++) {
    int64_t sc = c ? ssyv : ssyu, scc = c ? ssvv : ssuu, csum = c ? vsum : usum;
    S *dst = c ? v : u;
    if (!(sc * sc * 2 > ssyy * scc)) continue;
    int64_t a64 = (sc << 16) / ssyy;
    int64_t b64 = ((csum << 16) - a64 * ysum) >> sh;
    int64_t lim = (int64_t)1 << (31 - bitdepth);
    int32_t a = (int32_t)(a64 < -lim ? -lim : a64 > lim ? lim : a64);
    int64_t bb = b64 + (1 << 15);
    int32_t b = (int32_t)(bb < -((int64_t)1 << 31) ? -((int64_t)1 << 31) : bb > (((int64_t)1 << 31) - 1) ? (((int64_t)1 << 31) - 1) : bb);
#define ORC_MAP(px) orc_sat((a * (int)(px) + b) >> 16, maxv)
    for (int i = 0; i < nc; i++)
      for (int j = 0; j < nc; j++)
        dst[i * cs + j] = sub ? (S)((ORC_MAP(ry[(2 * i) * stride + 2 * j]) + ORC_MAP(ry[(2 * i) * stride + 2 * j + 1]) +
                                     ORC_MAP(ry[(2 * i + 1) * stride + 2 * j]) + ORC_MAP(ry[(2 * i + 1) * stride + 2 * j + 1]) + 2) >> 2)
                              : (S)ORC_MAP(ry[i * stride + j]);
#undef ORC_MAP
  }
}

/* ---- a17: luma deblocking, vertical edges of the whole frame then horizontal edges.
 * common/common_frame.c:47-352 with the compile-time switches of common/global.h:80-85 (all on). ---- */
static void FN(orc_deblock_edge_y)(S *p, int along, int across, const orc_blkinfo_t *bq, const orc_blkinfo_t *bp_, int bstep,
                                   int pos_mod_base, int vertical, int beta, int tc, int maxv) {
  /* p: first sample on the q side of the edge; 'along' steps along the edge, 'across' steps across it */
  int d15 = 0, d26 = 0;
  for (int t = 0; t < 2; t++) {
    const S *l1 = p + (1 + 4 * t) * along, *l2 = p + (2 + 4 * t) * along;
    d15 += abs((int)l1[-2 * across] - (int)l1[-across]) + abs((int)l1[across] - (int)l1[0]);
    d26 += abs((int)l2[-2 * across] - (int)l2[-across]) + abs((int)l2[across] - (int)l2[0]);
  }
  for (int m = 0; m < 8; m += 4) {
    const orc_blkinfo_t *q = bq + (m / 4) * bstep, *pp = bp_ + (m / 4) * bstep;
    int q_size = q->size;
    int part_hit = vertical ? (q->pb_part == 2 || q->pb_part == 3) : (q->pb_part == 1 || q->pb_part == 3);
    if ((q->tb_split || part_hit) && q_size > 8) q_size /= 2;
    int mv = abs(pp->mv0y) >= 4 || abs(q->mv0y) >= 4 || abs(pp->mv0x) >= 4 || abs(q->mv0x) >= 4 ||
             abs(pp->mv1y) >= 4 || abs(q->mv1y) >= 4 || abs(pp->mv1x) >= 4 || abs(q->mv1x) >= 4;
    int cbp = pp->cbp_y || q->cbp_y;
    int intra = pp->mode == 1 || q->mode == 1;
    int interior = (pos_mod_base % q_size) > 0;
    if (interior || !(mv || cbp || intra)) continue;
    for (int k = m; k < m + 4; k++) {
      int d = (k & 1) ? d26 : d15;
      if (d >= beta) continue;
      S *s = p + k * along;
      int p1 = s[-2 * across], p0 = s[-across], q0 = s[0], q1 = s[across];
      int delta = (18 * (q0 - p0) - 6 * (q1 - p1) + 16) >> 5;
      delta = delta < -tc ? -tc : delta > tc ? tc : delta;
      s[-2 * across] = (S)orc_sat(p1 + delta / 2, maxv);
      s[-across] = (S)orc_sat(p0 + delta, maxv);
      s[0] = (S)orc_sat(q0 - delta, maxv);
      s[across] = (S)orc_sat(q1 - delta / 2, maxv);
    }
  }
}

void FN(orc_deblock_y)(S *rec, int stride, const orc_blkinfo_t *bi, int width, int height, int qp, int bitdepth) {
  int bw = width / 4, maxv = (1 << bitdepth) - 1;
  int beta = (S)(orc_beta_table[qp] << (bitdepth - 8));
  int tc = (S)(bitdepth > 12 ? orc_tc_table[qp] << (bitdepth - 12) : orc_tc_table[qp] >> (12 - bitdepth));
  for (int i = 0; i < height; i += 8)
    for (int j = 8; j < width; j += 8)
      FN(orc_deblock_edge_y)(rec + i * stride + j, stride, 1, bi + (i / 4) * bw + j / 4, bi + (i / 4) * bw + j / 4 - 1, bw, j, 1, beta, tc, maxv);
  for (int i = 8; i < height; i += 8)
    for (int j = 0; j < width; j += 8)
      FN(orc_deblock_edge_y)(rec + i * stride + j, 1, stride, bi + (i / 4) * bw + j / 4, bi + (i / 4 - 1) * bw + j / 4, 1, i, 0, beta, tc, maxv);
}

/* common/common_frame.c:354-432.  width,height are LUMA dimensions; chroma filtered only next to intra blocks. */
void FN(orc_deblock_uv)(S *recU, S *recV, int stride, const orc_blkinfo_t *bi, int width, int height, int sub, int qp, int bitdepth) {
  int bw = width / 4, maxv = (1 << bitdepth) - 1;
  int tc = (S)(bitdepth > 12 ? orc_tc_table[qp] << (bitdepth - 12) : orc_tc_table[qp] >> (12 - bitdepth));
  for (int uv = 0; uv < 2; uv++) {
    S *c = uv ? recV : recU;
    for (int pass = 0; pass < 2; pass++)
      for (int i = pass ? 8 : 0; i < height; i += 8)
        for (int j = pass ? 0 : 8; j < width; j += 8) {
          const orc_blkinfo_t *q = bi + (i / 4) * bw + j / 4, *p = pass ? q - bw : q - 1;
          int intra = p->mode == 1 || q->mode == 1;
          int interior = ((pass ? i : j) % q->size) > 0;
          if (interior || !intra) continue;
          S *s = c + (i >> sub) * stride + (j >> sub);
          int along = pass ? 1 : stride, across = pass ? stride : 1;
          for (int k = 0; k < (8 >> sub); k++, s += along) {
            int p1 = s[-2 * across], p0 = s[-across], q0 = s[0], q1 = s[across];
            int delta = (4 * (q0 - p0) + (p1 - q1) + 4) >> 3;
            delta = delta < -tc ? -tc : delta > tc ? tc : delta;
            s[-across] = (S)orc_sat(p0 + delta, maxv);
            s[0] = (S)orc_sat(q0 - delta, maxv);
          }
        }
  }
}

/* ---- a18: CLPF.  common/common_block.c:324-345 ---- */
void FN(orc_clpf_block)(const S *src, S *dst, int sstride, int dstride, int x0, int y0, int sizex, int sizey, int bt, unsigned strength, unsigned damping) {
  int xmin = x0 - !(bt & 1) * 2, ymin = y0 - !(bt & 4) * 2;
  int xmax = x0 + sizex + !(bt & 2) * 2 - 1, ymax = y0 + sizey + !(bt & 8) * 2 - 1;
#define MX(a, b) ((a) > (b) ? (a) : (b))
#define MN(a, b) ((a) < (b) ? (a) : (b))
  for (int y = y0; y < y0 + sizey; y++)
    for (int x = x0; x < x0 + sizex; x++) {
      int X = src[y * sstride + x];
      int d = orc_clpf_sample(X, src[MX(ymin, y - 2) * sstride + x], src[MX(ymin, y - 1) * sstride + x], src[y * sstride + MX(xmin, x - 2)],
                              src[y * sstride + MX(xmin, x - 1)], src[y * sstride + MN(xmax, x + 1)], src[y * sstride + MN(xmax, x + 2)],
                              src[MN(ymax, y + 1) * sstride + x], src[MN(ymax, y + 2) * sstride + x], (int)strength, damping);
      dst[y * dstride + x] = (S)(X + d);
    }
}

/* Whole-plane CLPF with the reference's semantics made explicit: every read sees unfiltered samples
 * (the block cache of common/common_frame.c:1005-1155 delays write-back by one filter-block row), so src->dst
 * out of place.  dst must be pre-filled with src.  width,height = dimensions of THIS plane.  fb_on = per filter
 * block decision (NULL = filter every non-all-skip block).  The skip lookup reproduces the reference's index
 * arithmetic, including its use of the plane width as the grid pitch (common_frame.c:1049, 1073). */
void FN(orc_clpf_plane)(const S *src, S *dst, int stride, int width, int height, const orc_blkinfo_t *bi, int bi_stride_unused, int sub,
                        const uint8_t *fb_on, int fb_size_log2, unsigned strength, int bitdepth, int plane, int qp) {
  (void)bi_stride_unused;
  int bs = sub ? 4 : 8, fb = 1 << fb_size_log2;
  int nh = (width + fb - 1) >> fb_size_log2, nv = (height + fb - 1) >> fb_size_log2;
  unsigned damping = (unsigned)(bitdepth - 4 - (plane != 0) + (qp >> 4));
  strength <<= bitdepth - 8;
  for (int k = 0; k < nv; k++)
    for (int l = 0; l < nh; l++) {
      int xoff = l << fb_size_log2, yoff = k << fb_size_log2, allskip = 1;
      for (int m = 0; allskip && m < fb / bs; m++)
        for (int n = 0; allskip && n < fb / bs; n++) {
          int xpos = xoff + n * bs, ypos = yoff + m * bs;
          if (xpos < width && ypos < height) allskip &= bi[((ypos << sub) / 4) * (width / 4) + ((xpos << sub) / 4)].mode == 0;
        }
      int h = MN(height, (k + 1) << fb_size_log2) & (fb - 1), w = MN(width, (l + 1) << fb_size_log2) & (fb - 1);
      h += !h << fb_size_log2;
      w += !w << fb_size_log2;
      if (allskip || (fb_on && !fb_on[k * nh + l])) continue;
      for (int m = 0; m < (h + bs - 1) / bs; m++)
        for (int n = 0; n < (w + bs - 1) / bs; n++) {
          int xpos = xoff + n * bs, ypos = yoff + m * bs;
          int sizex = MN(width - xpos, bs), sizey = MN(height - ypos, bs);
          if (bi[((ypos << sub) / 4) * (width / 4) + ((xpos << sub) / 4)].mode == 0) continue;
          int bt = (xpos == 0 ? 1 : 0) | (ypos == 0 ? 4 : 0) | (xpos == width - sizex ? 2 : 0) | (ypos == height - sizey ? 8 : 0);
          FN(orc_clpf_block)(src, dst, stride, stride, xpos, ypos, sizex, sizey, bt, strength, damping);
        }
    }
}

/* enc/encode_block.c:2568-2624 (C forms; the SIMD detect_clpf doubles both sums, enc/enc_kernels.c:259) */
void FN(orc_detect_clpf)(const S *rec, const S *org, int x0, int y0, int width, int height, int ostride, int rstride, int *sum0, int *sum1,
                         unsigned strength, unsigned shift, unsigned size, unsigned dmp) {
  uint32_t s0 = 0, s1 = 0;
  for (int y = y0; y < y0 + (int)size; y++)
    for (int x = x0; x < x0 + (int)size; x++) {
      int O = org[y * ostride + x], X = rec[y * rstride + x];
      int d = orc_clpf_sample(X, rec[MX(0, y - 2) * rstride + x], rec[MX(0, y - 1) * rstride + x], rec[y * rstride + MX(0, x - 2)],
                              rec[y * rstride + MX(0, x - 1)], rec[y * rstride + MN(width - 1, x + 1)], rec[y * rstride + MN(width - 1, x + 2)],
                              rec[MN(height - 1, y + 1) * rstride + x], rec[MN(height - 1, y + 2) * rstride + x], (int)strength, dmp);
      s0 += (uint32_t)((O - X) * (O - X));
      s1 += (uint32_t)((O - X - d) * (O - X - d));
    }
  *sum0 += (int)(s0 >> (shift * 2));
  *sum1 += (int)(s1 >> (shift * 2));
}
void FN(orc_detect_multi_clpf)(const S *rec, const S *org, int x0, int y0, int width, int height, int ostride, int rstride, int *sum,
                               unsigned shift, unsigned size, unsigned dmp) {
  uint32_t s[4] = {0, 0, 0, 0};
  for (int y = y0; y < y0 + (int)size; y++)
    for (int x = x0; x < x0 + (int)size; x++) {
      int O = org[y * ostride + x], X = rec[y * rstride + x];
      int A = rec[MX(0, y - 2) * rstride + x], B = rec[MX(0, y - 1) * rstride + x], C = rec[y * rstride + MX(0, x - 2)], D = rec[y * rstride + MX(0, x - 1)];
      int E = rec[y * rstride + MN(width - 1, x + 1)], F = rec[y * rstride + MN(width - 1, x + 2)];
      int G = rec[MN(height - 1, y + 1) * rstride + x], H = rec[MN(height - 1, y + 2) * rstride + x];
      s[0] += (uint32_t)((O - X) * (O - X));
      for (int t = 0; t < 3; t++) {
        int Y = X + orc_clpf_sample(X, A, B, C, D, E, F, G, H, (1 << t) << shift, dmp);
        s[t + 1] += (uint32_t)((O - Y) * (O - Y));
      }
    }
  for (int t = 0; t < 4; t++) sum[t] += (int)(s[t] >> (shift * 2));
}
#undef MX
#undef MN

/* ---- a19: CDEF direction search.  common/common_block.c:94-167 ---- */
int FN(orc_cdef_find_dir)(const S *img, int stride, int32_t *var, int coeff_shift) {
  static const int div_table[9] = {0, 840, 420, 280, 210, 168, 140, 120, 105};
  int32_t cost[8] = {0};
  int partial[8][15];
  memset(partial, 0, sizeof(partial));
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) {
      int x = (img[i * stride + j] >> coeff_shift) - 128;
      partial[0][i + j] += x;
      partial[1][i + j / 2] += x;
      partial[2][i] += x;
      partial[3][3 + i - j / 2] += x;
      partial[4][7 + i - j] += x;
      partial[5][3 - i / 2 + j] += x;
      partial[6][j] += x;
      partial[7][i / 2 + j] += x;
    }
  for (int i = 0; i < 8; i++) {
    cost[2] += partial[2][i] * partial[2][i];
    cost[6] += partial[6][i] * partial[6][i];
  }
  cost[2] *= div_table[8];
  cost[6] *= div_table[8];
  for (int i = 0; i < 7; i++) {
    cost[0] += (partial[0][i] * partial[0][i] + partial[0][14 - i] * partial[0][14 - i]) * div_table[i + 1];
    cost[4] += (partial[4][i] * partial[4][i] + partial[4][14 - i] * partial[4][14 - i]) * div_table[i + 1];
  }
  cost[0] += partial[0][7] * partial[0][7] * div_table[8];
  cost[4] += partial[4][7] * partial[4][7] * div_table[8];
  for (int i = 1; i < 8; i += 2) {
    for (int j = 0; j < 5; j++) cost[i] += partial[i][3 + j] * partial[i][3 + j];
    cost[i] *= div_table[8];
    for (int j = 0; j < 3; j++) cost[i] += (partial[i][j] * partial[i][j] + partial[i][10 - j] * partial[i][10 - j]) * div_table[2 * j + 2];
  }
  int32_t best_cost = 0;
  int best_dir = 0;
  for (int i = 0; i < 8; i++)
    if (cost[i] > best_cost) { best_cost = cost[i]; best_dir = i; }
  *var = (best_cost - cost[(best_dir + 4) & 7]) >> 10;
  return best_dir;
}

/* common/common_frame.c:766-807: (bs+4)^2 uint16 staging tile; 30000 outside the frame */
void FN(orc_cdef_prepare_input)(int sizex, int sizey, int xpos, int ypos, int bt, int padding, uint16_t *src16, int stride16, const S *src, int sstride) {
  for (int i = -padding; i < sizey + padding; i++)
    for (int j = -padding; j < sizex + padding; j++) {
      int out = ((bt & 4) && i < 0) || ((bt & 8) && i >= sizey) || ((bt & 1) && j < 0) || ((bt & 2) && j >= sizex);
      src16[i * stride16 + j] = out ? 30000 : src[(ypos + i) * sstride + xpos + j];
    }
}

/* Whole-plane CDEF, out of place (see orc_clpf_plane).  common/common_frame.c:826-1003.  width,height = LUMA
 * frame dimensions.  fb_pri/fb_sec: per 64x64 filter block `level` and `sec_strength` of this plane class
 * (cdef_strength.level / .sec_strength).  dirs/vars: 64 ints per filter block, written when plane==0 and read by
 * the chroma planes. dst must be pre-filled with src. */
void FN(orc_cdef_plane)(const S *src, S *dst, int stride, int width, int height, const orc_blkinfo_t *bi, int bi_stride, int sub_in, int plane,
                        const int8_t *fb_pri, const int8_t *fb_sec, int pri_damping_f, int sec_damping_f, int *dirs, int *vars, int bitdepth) {
  int sub = plane != 0 && sub_in, bs = sub ? 4 : 8, bslog = sub ? 2 : 3;
  int nh = (width + 63) >> 6, nv = (height + 63) >> 6, coeff_shift = bitdepth - 8;
  uint16_t tile[12 * 16];
  (void)bi_stride;
  for (int k = 0, ci = 0; k < nv; k++)
    for (int l = 0; l < nh; l++, ci++) {
      int xoff = l << 6, yoff = k << 6, allskip = 1;
      for (int m = 0; allskip && m < 8; m++)
        for (int n = 0; allskip && n < 8; n++) {
          int xpos = xoff + n * 8, ypos = yoff + m * 8;
          if (xpos < width && ypos < height) allskip &= bi[(ypos / 4) * (width / 4) + xpos / 4].mode == 0;
        }
      if (allskip) continue;
      int h = (height < ((k + 1) << 6) ? height : ((k + 1) << 6)) & 63, w = (width < ((l + 1) << 6) ? width : ((l + 1) << 6)) & 63;
      h += !h << 6;
      w += !w << 6;
      int pri_strength = fb_pri[ci], sec_strength = fb_sec[ci] + (fb_sec[ci] == 3);
      for (int m = 0; m < ((h + bs - 1) >> (bslog + sub)); m++)
        for (int n = 0; n < ((w + bs - 1) >> (bslog + sub)); n++) {
          int xpos = (xoff >> sub) + n * bs, ypos = (yoff >> sub) + m * bs;
          int sizex = (width >> sub) - xpos < bs ? (width >> sub) - xpos : bs, sizey = (height >> sub) - ypos < bs ? (height >> sub) - ypos : bs;
          int index = ((yoff + m * 8) / 4) * (width / 4) + (xoff + n * 8) / 4;
          if (plane == 0) dirs[ci * 64 + m * 8 + n] = FN(orc_cdef_find_dir)(src + ypos * stride + xpos, stride, &vars[ci * 64 + m * 8 + n], coeff_shift);
          if (bi[index].mode == 0) continue;
          int bt = (xpos == 0 ? 1 : 0) | (ypos == 0 ? 4 : 0) | (xpos == (width >> sub) - sizex ? 2 : 0) | (ypos == (height >> sub) - sizey ? 8 : 0);
          FN(orc_cdef_prepare_input)(sizex, sizey, xpos, ypos, bt, 2, tile + 2 * 16 + 2, 16, src, stride);
          int adj = plane ? pri_strength : orc_adjust_strength(pri_strength, vars[ci * 64 + m * 8 + n]);
          int pd = pri_damping_f - !!plane, sd = sec_damping_f - !!plane;
          if (adj && orc_log2i(adj) > pd) pd = orc_log2i(adj);
          S *o = dst + ypos * stride + xpos;
          orc_cdef_filter_block(sizeof(S) == 1 ? (uint8_t *)o : NULL, sizeof(S) == 1 ? NULL : (uint16_t *)o, stride, tile + 2 * 16 + 2, 16,
                                adj << coeff_shift, sec_strength << coeff_shift, pri_strength ? dirs[ci * 64 + m * 8 + n] : 0, pd + coeff_shift,
                                sd + coeff_shift, sizex, coeff_shift);
        }
    }
}

/* ---- a20: border replication.  common/common_frame.c:657-743 ---- */
void FN(orc_pad_plane)(S *p, int stride, int w, int h, int pad_hor, int pad_ver) {
  for (int i = 0; i < h; i++) {
    S l = p[i * stride], r = p[i * stride + w - 1];
    for (int j = 0; j < pad_hor; j++) { p[i * stride - pad_hor + j] = l; p[i * stride + w + j] = r; }
  }
  for (int i = -pad_ver; i < 0; i++) memcpy(p + i * stride - pad_hor, p - pad_hor, (size_t)(w + 2 * pad_hor) * sizeof(S));
  for (int i = h; i < h + pad_ver; i++) memcpy(p + i * stride - pad_hor, p + (h - 1) * stride - pad_hor, (size_t)(w + 2 * pad_hor) * sizeof(S));
}

/* ---- a21: 2x2 down-scaling.  common/temporal_interp.c:143-175, common/common_kernels.c:1847-1866 ---- */
void FN(orc_scale_down2x2)(const S *in, int si, S *out, int so, int wo, int ho) {
  for (int i = 0; i < ho; i++)
    for (int j = 0; j < wo; j++)
      out[i * so + j] = (S)((ORC_UP(in[2 * i * si + 2 * j], in[(2 * i + 1) * si + 2 * j]) + ORC_UP(in[2 * i * si + 2 * j + 1], in[(2 * i + 1) * si + 2 * j + 1])) >> 1);
}

/* ---- a5: the uni-directional motion search.  enc/encode_block.c:517-711.  orig = compact block (stride=size);
 * ref = reference-frame sample at the block position. ---- */
static unsigned FN(orc_me_cost)(unsigned sad, int bitdepth, double lambda, const orc_mv_t *c, const orc_mv_t *mvp) {
  sad >>= bitdepth - 8;
  return sad + (unsigned)(lambda * (double)orc_quote_mv_bits(c->y - mvp->y, c->x - mvp->x) + 0.5);
}
int FN(orc_motion_estimate)(const S *orig, const S *ref, int size, int stride_r, int width, int height, orc_mv_t *mv, const orc_mv_t *mvc,
                            const orc_mv_t *mvp, double lambda, int speed, int bitdepth, int sign, int fwidth, int fheight, int xpos, int ypos,
                            const orc_mv_t *mvcand, int mvcand_num, int enable_bipred) {
  static S rf[128 * 128];
  int s = sign ? -1 : 1;
  uint32_t min_sad = 1u << 31;
  orc_mv_t cand, opt = {0, 0}, mref;
  unsigned sad;
  mref.y = (int16_t)(((mvc->y + 2) >> 2) << 2);
  mref.x = (int16_t)(((mvc->x + 2) >> 2) << 2);
#define ORC_AT(c) (ref + s * ((c).x >> 2) + s * ((c).y >> 2) * stride_r)
  if ((size == 16 && enable_bipred) || speed == 0) {
    for (int step = 32; step >= 4; step >>= 1) {
      int range = 2 * step;
      for (int k = -range; k <= range; k += step)
        for (int l = -range; l <= range; l += step) {
          if (step < 32 && !k && !l) continue;
          cand.y = (int16_t)(mref.y + k);
          cand.x = (int16_t)(mref.x + l);
          orc_clip_mv(&cand, ypos, xpos, fwidth, fheight, size, size, sign);
          if (step == 32 && size == 16 && speed == 1) {
            int x = 0;
            sad = FN(orc_widesad)(orig, ORC_AT(cand), size, stride_r, width, height, &x);
            cand.x = (int16_t)(cand.x + (s * x << 2));
          } else
            sad = FN(orc_sad)(orig, ORC_AT(cand), size, stride_r, width, height);
          sad = FN(orc_me_cost)(sad, bitdepth, lambda, &cand, mvp);
          if (sad < min_sad) { min_sad = sad; opt = cand; }
        }
      mref = opt;
    }
  }
  for (int idx = 0; idx < mvcand_num; idx++) {
    int x = 0;
    cand.y = (int16_t)(mvcand[idx].y << 2);
    cand.x = (int16_t)(mvcand[idx].x << 2);
    orc_clip_mv(&cand, ypos, xpos, fwidth, fheight, size, size, sign);
    if (size == 16) sad = FN(orc_widesad)(orig, ORC_AT(cand), size, stride_r, width, height, &x);
    else sad = FN(orc_sad)(orig, ORC_AT(cand), size, stride_r, width, height);
    cand.x = (int16_t)(cand.x + (s * x << 2));
    sad = FN(orc_me_cost)(sad, bitdepth, lambda, &cand, mvp);
    if (sad < min_sad) { min_sad = sad; opt = cand; }
  }
  mref = opt;
  int maxsteps = (size <= 16 || speed == 0) ? 6 : 0, start = 0, end = 5;
  for (int step = 1; step < maxsteps; step++) {
    static const int diy[6] = {1, 2, 1, -1, -2, -1}, dix[6] = {-1, 0, 1, 1, 0, -1};
    int dir = start - 1, best_dir = -1;
    do {
      dir++;
      if (dir == 6) dir = 0;
      cand.y = (int16_t)(mref.y + dix[dir] * 4);
      cand.x = (int16_t)(mref.x + diy[dir] * 4);
      orc_clip_mv(&cand, ypos, xpos, fwidth, fheight, size, size, sign);
      sad = FN(orc_me_cost)(FN(orc_sad)(orig, ORC_AT(cand), size, stride_r, width, height), bitdepth, lambda, &cand, mvp);
      if (sad < min_sad) { min_sad = sad; opt = cand; best_dir = dir; }
    } while (dir != end);
    mref = opt;
    start = best_dir ? best_dir - 1 : 5;
    end = start + 2;
    end -= (end >= 6) * 6;
    if (best_dir < 0) break;
  }
  int ydh = 0, xdh = 0, ydq = 0, xdq = 0;
  unsigned cmin = min_sad;
  if (speed == 0) {
    static const int8_t hm[9] = {0, 0, -2, 2, 0, -2, -2, 2, 2}, hn[9] = {0, -2, 0, 0, 2, -2, 2, -2, 2};
    static const int8_t qm[9] = {0, 0, -1, 1, 0, -1, -1, 1, 1}, qn[9] = {0, -1, 0, 0, 1, -1, 1, -1, 1};
    for (int i = 1; i <= 8; i++) {
      cand.y = (int16_t)(mref.y + hm[i]);
      cand.x = (int16_t)(mref.x + hn[i]);
      FN(orc_get_inter_prediction_luma)(rf, ref, width, height, stride_r, width, &cand, sign, enable_bipred, fwidth, fheight, xpos, ypos, bitdepth);
      sad = FN(orc_me_cost)(FN(orc_sad)(orig, rf, size, width, width, height), bitdepth, lambda, &cand, mvp);
      if (sad < cmin) { cmin = sad; ydh = hm[i]; xdh = hn[i]; }
    }
    opt.x = (int16_t)(opt.x + xdh);
    opt.y = (int16_t)(opt.y + ydh);
    for (int i = 1; i <= 8; i++) {
      cand.y = (int16_t)(opt.y + qm[i]);
      cand.x = (int16_t)(opt.x + qn[i]);
      FN(orc_get_inter_prediction_luma)(rf, ref, width, height, stride_r, width, &cand, sign, enable_bipred, fwidth, fheight, xpos, ypos, bitdepth);
      unsigned raw = FN(orc_sad)(orig, rf, size, width, width, height) >> (bitdepth - 8);
      sad = raw + (unsigned)(int)(lambda * (double)orc_quote_mv_bits(cand.y - mvp->y, cand.x - mvp->x) + 0.5);
      if (sad < cmin) { cmin = sad; ydq = qm[i]; xdq = qn[i]; }
    }
  } else {
    int spx, spy;
    mref.x = (int16_t)(mref.x * s);
    mref.y = (int16_t)(mref.y * s);
    sad = FN(orc_sad_fasthalf)(orig, ref + (mref.x >> 2) + (mref.y >> 2) * stride_r, size, stride_r, width, height, &spx, &spy);
    sad >>= bitdepth - 8;
    sad += (unsigned)(lambda * (double)orc_quote_mv_bits(mref.y + s * spy - mvp->y, mref.x + s * spx - mvp->x) + 0.5);
    if (sad < cmin) { cmin = sad; xdh = s * spx; ydh = s * spy; }
    spx = xdh;
    spy = ydh;
    mref.x = (int16_t)(opt.x + s * spx);
    mref.y = (int16_t)(opt.y + s * spy);
    opt.x = (int16_t)(opt.x + xdh);
    opt.y = (int16_t)(opt.y + ydh);
    sad = FN(orc_sad_fastquarter)(orig, ref + s * (mref.x >> 2) + s * (mref.y >> 2) * stride_r, size, stride_r, width, height, &spx, &spy);
    sad >>= bitdepth - 8;
    sad += (unsigned)(int)(lambda * (double)orc_quote_mv_bits(mref.y + s * spy - mvp->y, mref.x + s * spx - mvp->x) + 0.5);
    if (sad < cmin) { cmin = sad; xdq = s * spx; ydq = s * spy; }
  }
#undef ORC_AT
  opt.x = (int16_t)(opt.x + xdq);
  opt.y = (int16_t)(opt.y + ydq);
  *mv = opt;
  return (int)(cmin < min_sad ? cmin : min_sad);
}

/* ---- a21: temporal frame interpolation.  common/temporal_interp.c:36-992.
 * Hierarchical (<= 4 levels, 2x2 down-scaled luma), raster-order bi-directional block matching on 16x16 blocks stored on
 * an 8x8 grid, with skip test, neighbour/guide candidates, cross refinement and a neighbour-smoothness cost; then a merge
 * pass per 8x8 block and integer-pel bi-directional averaging of all three planes.  MVs are in 1/8 sample units and are
 * rounded to integers for every access ((mv + 4) >> 3).  mv[1] refers to the farther picture, mv[0] = scaled mv[1]. ---- */
typedef struct {
  orc_mv_t *mv[2];
  int *bgmap;
  int wt[2], reversed, bw, bh;
  orc_mv_t skip_mv, scaled_skip_mv;
} FN(orc_ti_mvd);

typedef struct { const S *y; int stride, width, height, pad; } FN(orc_ti_pic);

#ifndef ORC_TI_HELPERS
#define ORC_TI_HELPERS
static int orc_ti_scale_val(int v, int numer, int denom) {
  if (denom == 0) return 0;
  int prod = v * numer;
  if (denom < 0) { denom = -denom; prod = -prod; }
  return prod >= 0 ? (prod + denom / 2) / denom : -((-prod + denom / 2) / denom);
}
static orc_mv_t orc_ti_scale_mv(orc_mv_t mv, int numer, int denom) {
  orc_mv_t o;
  if (numer == denom) return mv;
  if (numer == -denom) { o.x = (int16_t)-mv.x; o.y = (int16_t)-mv.y; return o; }
  o.x = (int16_t)orc_ti_scale_val(mv.x, numer, denom);
  o.y = (int16_t)orc_ti_scale_val(mv.y, numer, denom);
  return o;
}
static int orc_ti_add_cand(orc_mv_t *list, int max, int len, orc_mv_t c) { /* temporal_interp.c:205-218 */
  if (len < max) {
    list[len] = c;
    for (int i = 0; i < len; i++)
      if (list[i].x == c.x && list[i].y == c.y) return len;
    return len + 1;
  }
  return len;
}
static orc_mv_t orc_ti_absdist_filter(const orc_mv_t *l, int num) { /* :695-716, ties -> last */
  int best = 0, best_cost = 0x3fffffff;
  for (int j = 0; j < num; j++) {
    int cost = 0;
    for (int i = 0; i < num; i++) cost += abs(l[i].x - l[j].x) + abs(l[i].y - l[j].y);
    if (cost <= best_cost) { best = j; best_cost = cost; }
  }
  return l[best];
}
#endif

/* :375-456 (luma only): SAD between the two displaced size x size blocks; clipped per-sample form outside the padding */
static uint32_t FN(orc_ti_sad_cost)(int xstart, int ystart, const FN(orc_ti_pic) *pic, const orc_mv_t *mv, int size, uint32_t cost_start) {
  int xs[2], ys[2];
  for (int t = 0; t < 2; t++) { xs[t] = xstart + ((mv[t].x + 4) >> 3); ys[t] = ystart + ((mv[t].y + 4) >> 3); }
  const int pad = pic[0].pad, wP = pic[0].width + pad, hP = pic[0].height + pad;
  const int s0 = pic[0].stride, s1 = pic[1].stride;
  uint32_t c = cost_start;
  if (xs[0] >= -pad && xs[0] + size <= wP && ys[0] >= -pad && ys[0] + size <= hP && xs[1] >= -pad && xs[1] + size <= wP && ys[1] >= -pad && ys[1] + size <= hP) {
    c += FN(orc_sad)(pic[0].y + ys[0] * s0 + xs[0], pic[1].y + ys[1] * s1 + xs[1], s0, s1, size, size);
  } else {
    for (int i = 0; i < size; i++)
      for (int j = 0; j < size; j++) {
        int x0 = j + xs[0], x1 = j + xs[1], y0 = i + ys[0], y1 = i + ys[1];
        x0 = x0 < -pad ? -pad : (x0 > wP - 1 ? wP - 1 : x0); x1 = x1 < -pad ? -pad : (x1 > wP - 1 ? wP - 1 : x1);
        y0 = y0 < -pad ? -pad : (y0 > hP - 1 ? hP - 1 : y0); y1 = y1 < -pad ? -pad : (y1 > hP - 1 ? hP - 1 : y1);
        c += (uint32_t)abs((int)pic[1].y[y1 * s1 + x1] - (int)pic[0].y[y0 * s0 + x0]);
      }
  }
  return c;
}

static int FN(orc_ti_mv_cost)(orc_mv_t mv, const FN(orc_ti_mvd) *d, int xp, int yp, int st, int lambda) { /* :299-317, idx = 1 */
  const orc_mv_t *a = d->mv[1];
  int bw = d->bw, diff = 0;
#define ORC_TI_D(p) (abs(mv.x - a[p].x) + abs(mv.y - a[p].y))
  if (xp == 0 && yp == 0) diff = 0;
  else if (yp > 0 && xp > 0 && xp < bw - st)
    diff = ORC_TI_D((yp - st) * bw + xp + st) + ORC_TI_D((yp - st) * bw + xp) + ORC_TI_D((yp - st) * bw + xp - st) + ORC_TI_D(yp * bw + xp - st);
  else if (yp == 0) diff = ORC_TI_D(xp - st);
  else if (xp == 0) diff = ORC_TI_D((yp - st) * bw + xp + st) + ORC_TI_D((yp - st) * bw + xp);
#undef ORC_TI_D
  return (diff * lambda) >> 7;
}

/* :786-875 */
static void FN(orc_ti_motion_estimate_bi)(FN(orc_ti_mvd) *d, const FN(orc_ti_mvd) *guide, const FN(orc_ti_pic) *in0, const FN(orc_ti_pic) *in1) {
  const int bw = d->bw, bh = d->bh, st = 2, n = bw * bh;
  if (!guide) { memset(d->mv[0], 0, sizeof(orc_mv_t) * (size_t)n); memset(d->mv[1], 0, sizeof(orc_mv_t) * (size_t)n); }
  memset(d->bgmap, 0, sizeof(int) * (size_t)n);
  FN(orc_ti_pic) pic[2];
  pic[0] = d->reversed ? *in1 : *in0;
  pic[1] = d->reversed ? *in0 : *in1;
  const int pad = pic[0].pad, wP = pic[0].width + pad, hP = pic[0].height + pad;
  orc_mv_t cand[20];
  for (int i = 0; i < bh; i += st)
    for (int j = 0; j < bw; j += st) {
      const int pos = i * bw + j, xstart = j * 8, ystart = i * 8;
      /* skip vector from the causal neighbours (:758-770) */
      {
        orc_mv_t vl[3];
        int num = 0;
        d->skip_mv.x = d->skip_mv.y = 0;
        if (i > 0 && j < bw - st) vl[num++] = d->mv[1][(i - st) * bw + j + st];
        if (j > 0) vl[num++] = d->mv[1][i * bw + j - st];
        if (i > 0) vl[num++] = d->mv[1][(i - st) * bw + j];
        if (num) d->skip_mv = orc_ti_absdist_filter(vl, num);
        d->scaled_skip_mv = orc_ti_scale_mv(d->skip_mv, -d->wt[1], d->wt[0]);
      }
      /* skip test (:458-580): all four 8x8 quarters inside the padded area with SAD <= 8*64 */
      {
        orc_mv_t m1 = d->skip_mv, m0 = d->scaled_skip_mv;
        int skip = 1;
        for (int p = ystart; p < ystart + 16 && skip; p += 8)
          for (int q = xstart; q < xstart + 16 && skip; q += 8) {
            int x0 = q + ((m0.x + 4) >> 3), x1 = q + ((m1.x + 4) >> 3), y0 = p + ((m0.y + 4) >> 3), y1 = p + ((m1.y + 4) >> 3);
            if (x0 >= -pad && x0 + 8 <= wP && y0 >= -pad && y0 + 8 <= hP && x1 >= -pad && x1 + 8 <= wP && y1 >= -pad && y1 + 8 <= hP) {
              if ((int)FN(orc_sad)(pic[0].y + y0 * pic[0].stride + x0, pic[1].y + y1 * pic[1].stride + x1, pic[0].stride, pic[1].stride, 8, 8) > 8 * 64) skip = 0;
            } else
              skip = 0;
          }
        if (skip) { d->bgmap[pos] = 1; d->mv[1][pos] = d->skip_mv; d->mv[0][pos] = d->scaled_skip_mv; }
      }
      if (!d->bgmap[pos]) {
        /* candidates (:230-283): zero, the guide's vector, up-right, left, up */
        int len = 0;
        orc_mv_t zero = {0, 0};
        len = orc_ti_add_cand(cand, 20, len, zero);
        if (guide) {
          int numer = (d->reversed == guide->reversed) ? d->wt[0] : -d->wt[0];
          len = orc_ti_add_cand(cand, 20, len, orc_ti_scale_mv(guide->mv[1][pos], numer, guide->wt[0]));
        }
        if (i > 0 && j < bw - st) len = orc_ti_add_cand(cand, 20, len, d->mv[1][(i - st) * bw + j + st]);
        if (j > 0) len = orc_ti_add_cand(cand, 20, len, d->mv[1][i * bw + j - st]);
        if (i > 0) len = orc_ti_add_cand(cand, 20, len, d->mv[1][(i - st) * bw + j]);
        /* adaptive search (:584-668) */
        const int guided = guide != NULL, lambda = guided ? 3000 / 4 : 3000;
        orc_mv_t best_mv = cand[0], best_smv = orc_ti_scale_mv(cand[0], -d->wt[1], d->wt[0]);
        uint32_t best_cost = 0x3fffffff;
        for (int c = 0; c < len; c++) {
          orc_mv_t mv[2], rl, rsl;
          mv[1] = cand[c];
          mv[0] = orc_ti_scale_mv(cand[c], -d->wt[1], d->wt[0]);
          uint32_t cc = (uint32_t)FN(orc_ti_mv_cost)(cand[c], d, j, i, st, lambda);
          cc = FN(orc_ti_sad_cost)(xstart, ystart, pic, mv, 16, cc);
          rl = mv[1];
          rsl = mv[0];
          if (((4 + (uint32_t)c) * cc) / 8 < best_cost) {
            int shift = guided ? 3 : 6, count = guided ? 8 : 64;
            while (shift >= 3 && count > 0) {
              int off = 1 << shift, better = 0;
              orc_mv_t centre = rl;
              for (int k = 0; k < 4; k++) {
                orc_mv_t r = centre;
                if (k == 0) r.x = (int16_t)(centre.x - off);
                else if (k == 1) r.x = (int16_t)(centre.x + off);
                else if (k == 2) r.y = (int16_t)(centre.y - off);
                else r.y = (int16_t)(centre.y + off);
                mv[1] = r;
                mv[0] = orc_ti_scale_mv(r, -d->wt[1], d->wt[0]);
                uint32_t bc = (uint32_t)FN(orc_ti_mv_cost)(r, d, j, i, st, lambda);
                bc = FN(orc_ti_sad_cost)(xstart, ystart, pic, mv, 16, bc);
                if (bc < cc) { cc = bc; rl = r; rsl = mv[0]; better = 1; }
              }
              if (!better) shift--;
              count -= 4;
            }
          }
          if (cc < best_cost) { best_mv = rl; best_smv = rsl; best_cost = cc; }
        }
        d->mv[1][pos] = best_mv;
        d->mv[0][pos] = best_smv;
      }
      for (int q = 0; q < st; q++)
        for (int p = 0; p < st; p++) { d->mv[0][pos + q * bw + p] = d->mv[0][pos]; d->mv[1][pos + q * bw + p] = d->mv[1][pos]; d->bgmap[pos + q * bw + p] = d->bgmap[pos]; }
    }
  /* merge pass on the 8x8 grid (:219-229, 670-693, 853-872) */
  orc_mv_t *m0 = (orc_mv_t *)malloc(sizeof(orc_mv_t) * (size_t)n), *m1 = (orc_mv_t *)malloc(sizeof(orc_mv_t) * (size_t)n);
  for (int i = 0; i < bh; i++)
    for (int j = 0; j < bw; j++) {
      int len = 0, off = (i & 1) ? 2 : 1;
      len = orc_ti_add_cand(cand, 20, len, d->mv[1][i * bw + j]);
      if (i - off >= 0) len = orc_ti_add_cand(cand, 20, len, d->mv[1][(i - off) * bw + j]);
      if (i + off < bh) len = orc_ti_add_cand(cand, 20, len, d->mv[1][(i + off) * bw + j]);
      if (j - off >= 0) len = orc_ti_add_cand(cand, 20, len, d->mv[1][i * bw + j - off]);
      if (j + off < bw) len = orc_ti_add_cand(cand, 20, len, d->mv[1][i * bw + j + off]);
      if (len > 1) {
        uint32_t best = 0x3fffffff;
        orc_mv_t bm = {0, 0}, bs = {0, 0};
        for (int c = 0; c < len; c++) {
          orc_mv_t mv[2];
          mv[1] = cand[c];
          mv[0] = orc_ti_scale_mv(cand[c], -d->wt[1], d->wt[0]);
          uint32_t bc = FN(orc_ti_sad_cost)(j * 8, i * 8, pic, mv, 8, 0);
          if (bc < best) { best = bc; bm = cand[c]; bs = mv[0]; }
        }
        m1[i * bw + j] = bm;
        m0[i * bw + j] = bs;
      } else {
        m0[i * bw + j] = d->mv[0][i * bw + j];
        m1[i * bw + j] = d->mv[1][i * bw + j];
      }
    }
  memcpy(d->mv[0], m0, sizeof(orc_mv_t) * (size_t)n);
  memcpy(d->mv[1], m1, sizeof(orc_mv_t) * (size_t)n);
  free(m0);
  free(m1);
}

/* :319-373, 877-935: integer-pel bi-directional average of one plane */
static void FN(orc_ti_interp_plane)(const FN(orc_ti_mvd) *d, const S *p0, int s0, const S *p1, int s1, S *out, int so, int wP, int hP, int pad, int chroma) {
  const int bs = chroma ? 4 : 8;
  for (int yp = 0; yp < d->bh; yp++)
    for (int xp = 0; xp < d->bw; xp++) {
      orc_mv_t mv0 = d->mv[0][yp * d->bw + xp], mv1 = d->mv[1][yp * d->bw + xp];
      if (chroma) { mv1.x >>= 1; mv1.y >>= 1; mv0 = orc_ti_scale_mv(mv1, -d->wt[1], d->wt[0]); }
      const int xstart = xp * bs, ystart = yp * bs;
      int xs[2] = {xstart + ((mv0.x + 4) >> 3), xstart + ((mv1.x + 4) >> 3)}, ys[2] = {ystart + ((mv0.y + 4) >> 3), ystart + ((mv1.y + 4) >> 3)};
      int in0 = xs[0] >= -pad && xs[0] + bs <= wP && ys[0] >= -pad && ys[0] + bs <= hP, in1 = xs[1] >= -pad && xs[1] + bs <= wP && ys[1] >= -pad && ys[1] + bs <= hP;
      S *p = out + ystart * so + xstart;
      for (int i = 0; i < bs; i++)
        for (int j = 0; j < bs; j++) {
          if (in0 && in1) p[i * so + j] = (S)(((int)p0[(ys[0] + i) * s0 + xs[0] + j] + (int)p1[(ys[1] + i) * s1 + xs[1] + j] + 1) >> 1);
          else if (in1) p[i * so + j] = p1[(ys[1] + i) * s1 + xs[1] + j];
          else if (in0) p[i * so + j] = p0[(ys[0] + i) * s1 + xs[0] + j]; /* sic: row pitch s1 (temporal_interp.c:353) */
          else {
            int x0 = j + xs[0], x1 = j + xs[1], y0 = i + ys[0], y1 = i + ys[1];
            x0 = x0 < -pad ? -pad : (x0 > wP - 1 ? wP - 1 : x0); x1 = x1 < -pad ? -pad : (x1 > wP - 1 ? wP - 1 : x1);
            y0 = y0 < -pad ? -pad : (y0 > hP - 1 ? hP - 1 : y0); y1 = y1 < -pad ? -pad : (y1 > hP - 1 ? hP - 1 : y1);
            p[i * so + j] = (S)(((int)p0[y0 * s0 + x0] + (int)p1[y1 * s1 + x1] + 1) / 2);
          }
        }
    }
}

static void FN(orc_ti_alloc)(FN(orc_ti_mvd) *d, int w, int h, int ratio, int k) { /* :84-129, interpolate = 1 */
  d->bw = 2 * ((w + 15) / 16);
  d->bh = 2 * ((h + 15) / 16);
  size_t n = (size_t)d->bw * d->bh;
  d->mv[0] = (orc_mv_t *)calloc(n, sizeof(orc_mv_t));
  d->mv[1] = (orc_mv_t *)calloc(n, sizeof(orc_mv_t));
  d->bgmap = (int *)calloc(n, sizeof(int));
  d->reversed = k > ratio / 2;
  d->wt[0] = d->reversed ? k : ratio - k;
  d->wt[1] = ratio - d->wt[0];
}

/* outY/U/V: planes of the new frame at sample (0,0) (needs >= 8 samples of writable border right/below); r0x, r1x: the two
 * references with `pad` samples of replicated border (luma; pad/2 chroma).  max_levels is computed by the caller exactly as
 * the reference does (:914, double log10).  Level l > 0 pictures are 2x2 down-scaled luma with 32 samples of border. */
void FN(orc_interpolate_frames)(S *outY, S *outU, S *outV, int so_y, int so_c, const S *r0Y, const S *r0U, const S *r0V, const S *r1Y, const S *r1U,
                                const S *r1V, int sy, int sc, int width, int height, int pad, int ratio, int pos, int max_levels) {
  FN(orc_ti_mvd) mvd[4], spat[4];
  S *buf[4][2] = {{0}};
  FN(orc_ti_pic) in[4][2];
  in[0][0].y = r0Y; in[0][1].y = r1Y;
  for (int t = 0; t < 2; t++) { in[0][t].stride = sy; in[0][t].width = width; in[0][t].height = height; in[0][t].pad = pad; }
  for (int l = 0; l < max_levels; l++) { FN(orc_ti_alloc)(&mvd[l], width >> l, height >> l, ratio, pos); FN(orc_ti_alloc)(&spat[l], width >> l, height >> l, ratio, pos); }
  for (int l = 1; l < max_levels; l++) {
    int w = width >> l, h = height >> l, st = (w + 64 + 15) & ~15;
    for (int t = 0; t < 2; t++) {
      buf[l][t] = (S *)calloc((size_t)st * (h + 64) + 64, sizeof(S));
      S *o = buf[l][t] + 32 * st + 32;
      FN(orc_scale_down2x2)(in[l - 1][t].y, in[l - 1][t].stride, o, st, w, h);
      FN(orc_pad_plane)(o, st, w, h, 32, 32);
      in[l][t].y = o; in[l][t].stride = st; in[l][t].width = w; in[l][t].height = h; in[l][t].pad = 32;
    }
  }
  for (int l = max_levels - 1; l >= 0; l--) {
    FN(orc_ti_motion_estimate_bi)(&mvd[l], l != max_levels - 1 ? &spat[l] : NULL, &in[l][0], &in[l][1]);
    if (l > 0) { /* upscale_mv_data_2x2 :176-203 */
      FN(orc_ti_mvd) *o = &spat[l - 1];
      for (int i = 0; i < o->bh; i++)
        for (int j = 0; j < o->bw; j++) {
          orc_mv_t m = mvd[l].mv[1][(i / 2) * mvd[l].bw + j / 2];
          m.x = (int16_t)(m.x << 1);
          m.y = (int16_t)(m.y << 1);
          o->mv[1][i * o->bw + j] = m;
          o->mv[0][i * o->bw + j] = orc_ti_scale_mv(m, -o->wt[1], o->wt[0]);
        }
    }
  }
  {
    const FN(orc_ti_mvd) *d = &mvd[0];
    const int rev = d->reversed, wP = width + 4, hP = height + 4;
    FN(orc_ti_interp_plane)(d, rev ? r1Y : r0Y, sy, rev ? r0Y : r1Y, sy, outY, so_y, wP, hP, 4, 0);
    FN(orc_ti_interp_plane)(d, rev ? r1U : r0U, sc, rev ? r0U : r1U, sc, outU, so_c, wP >> 1, hP >> 1, 2, 1);
    FN(orc_ti_interp_plane)(d, rev ? r1V : r0V, sc, rev ? r0V : r1V, sc, outV, so_c, wP >> 1, hP >> 1, 2, 1);
  }
  for (int l = 0; l < max_levels; l++) {
    free(mvd[l].mv[0]); free(mvd[l].mv[1]); free(mvd[l].bgmap); free(spat[l].mv[0]); free(spat[l].mv[1]); free(spat[l].bgmap);
    if (l) { free(buf[l][0]); free(buf[l][1]); }
  }
}

/* ---- a5: simultaneous bi-directional search with mv0 = -mv1.  enc/encode_block.c:798-914.  3x3 telescope at steps
 * 32..1 quarter-pels (the last step visits only the legal quarter/half positions), then six candidates (four list entries
 * used AS quarter-pel vectors, the predictor, zero).  Each probe averages the two true interpolations, (a+b)>>1.
 * Note the second clip_mv runs on the already clipped vector and its result is the one kept. ---- */
int FN(orc_motion_estimate_bi)(const S *orig, const S *ref0, const S *ref1, int size, int stride_r, int width, int height, orc_mv_t *mv, const orc_mv_t *mvc,
                               const orc_mv_t *mvp, double lambda, int bitdepth, int sign, int fwidth, int fheight, int xpos, int ypos, const orc_mv_t *mvcand,
                               int mvcand_num, int enable_bipred) {
  static S rf0[128 * 128], rf1[128 * 128];
  uint32_t min_sad = 1u << 31, sad;
  orc_mv_t cand, opt = {0, 0}, mref;
  mref.y = (int16_t)(((mvc->y + 2) >> 2) << 2);
  mref.x = (int16_t)(((mvc->x + 2) >> 2) << 2);
  for (int pass = 0; pass < 2; pass++) {
    int nsteps = pass == 0 ? 6 : 1;
    for (int si = 0; si < nsteps; si++) {
      int step = pass == 0 ? (32 >> si) : 0;
      int kmax = pass == 0 ? 3 : 6;  /* 3x3 grid rows, or the six candidates */
      for (int kk = 0; kk < kmax; kk++)
        for (int ll = 0; ll < (pass == 0 ? 3 : 1); ll++) {
          if (pass == 0) {
            int k = (kk - 1) * step, l = (ll - 1) * step;
            if (step < 32 && k == 0 && l == 0) continue;
            if (step == 1) {
              int vf = mref.y & 3, hf = mref.x & 3, skip;
              if (vf == 0 && hf == 0) skip = abs(k) != abs(l);
              else if (vf == 2 && hf == 2) skip = 1;
              else skip = abs(k) == abs(l);
              if (skip) continue;
            }
            cand.y = (int16_t)(mref.y + k);
            cand.x = (int16_t)(mref.x + l);
          } else {
            orc_mv_t z = {0, 0};
            cand = kk < 4 ? (kk < mvcand_num ? mvcand[kk] : z) : (kk == 4 ? *mvp : z);
          }
          orc_clip_mv(&cand, ypos, xpos, fwidth, fheight, size, size, sign);
          FN(orc_get_inter_prediction_luma)(rf0, ref0, width, height, stride_r, width, &cand, sign, enable_bipred, fwidth, fheight, xpos, ypos, bitdepth);
          orc_clip_mv(&cand, ypos, xpos, fwidth, fheight, size, size, 1 - sign);
          FN(orc_get_inter_prediction_luma)(rf1, ref1, width, height, stride_r, width, &cand, 1 - sign, enable_bipred, fwidth, fheight, xpos, ypos, bitdepth);
          sad = 0;
          for (int i = 0; i < height; i++)
            for (int j = 0; j < width; j++) sad += (unsigned)abs((int)orig[i * size + j] - (((int)rf0[i * size + j] + (int)rf1[i * size + j]) >> 1));
          sad >>= bitdepth - 8;
          sad += (unsigned)(lambda * (double)orc_quote_mv_bits((int16_t)(cand.y - mvp->y), (int16_t)(cand.x - mvp->x)) + 0.5);
          if (sad < min_sad) { min_sad = sad; opt = cand; }
        }
      if (pass == 0) mref = opt;
    }
  }
  *mv = opt;
  return (int)min_sad;
}

/* ---- a5: motion_estimate_sync, the search used with -sync 1.  enc/encode_block.c:713-796.  The same 3x3 telescope (steps 32..1 quarter-pels, the legal positions only
 * at step 1) and six candidates as the bi-directional search, on ONE reference with every probe truly interpolated; the candidate list is used AS quarter-pel vectors and
 * entries 4 / 5 are overwritten with the predictor / zero (the caller's list is scribbled on like in motion_estimate_bi: pass a writable copy of >= 6 entries).
 * ORACLE ONLY so far: libthor_b200 has no CUDA form of it (the RD-loop binding leaves -sync 1 to the reference's own loop). ---- */
int FN(orc_motion_estimate_sync)(const S *orig, const S *ref, int size, int stride_r, int width, int height, orc_mv_t *mv, const orc_mv_t *mvc, const orc_mv_t *mvp,
                                 double lambda, int bitdepth, int sign, int fwidth, int fheight, int xpos, int ypos, orc_mv_t *mvcand, int enable_bipred) {
  static S rf[128 * 128];
  uint32_t min_sad = 1u << 31, sad;
  orc_mv_t cand, opt = {0, 0}, mref;
  mref.y = (int16_t)(((mvc->y + 2) >> 2) << 2);
  mref.x = (int16_t)(((mvc->x + 2) >> 2) << 2);
  for (int step = 32; step > 0; step >>= 1) {
    for (int k = -step; k <= step; k += step)
      for (int l = -step; l <= step; l += step) {
        if (step < 32 && k == 0 && l == 0) continue;
        if (step == 1) {
          int vf = mref.y & 3, hf = mref.x & 3, skip;
          if (vf == 0 && hf == 0) skip = abs(k) != abs(l);
          else if (vf == 2 && hf == 2) skip = 1;
          else skip = abs(k) == abs(l);
          if (skip) continue;
        }
        cand.y = (int16_t)(mref.y + k);
        cand.x = (int16_t)(mref.x + l);
        orc_clip_mv(&cand, ypos, xpos, fwidth, fheight, size, size, sign);
        FN(orc_get_inter_prediction_luma)(rf, ref, width, height, stride_r, width, &cand, sign, enable_bipred, fwidth, fheight, xpos, ypos, bitdepth);
        sad = FN(orc_sad)(orig, rf, size, width, width, height) >> (bitdepth - 8);
        sad += (unsigned)(int)(lambda * (double)orc_quote_mv_bits((int16_t)(cand.y - mvp->y), (int16_t)(cand.x - mvp->x)) + 0.5);
        if (sad < min_sad) { min_sad = sad; opt = cand; }
      }
    mref = opt;
  }
  mvcand[4] = *mvp;
  mvcand[5].y = 0; mvcand[5].x = 0;
  for (int idx = 0; idx < 6; idx++) {  /* ME_CANDIDATES */
    cand = mvcand[idx];
    orc_clip_mv(&cand, ypos, xpos, fwidth, fheight, size, size, sign);
    FN(orc_get_inter_prediction_luma)(rf, ref, width, height, stride_r, width, &cand, sign, enable_bipred, fwidth, fheight, xpos, ypos, bitdepth);
    sad = FN(orc_sad)(orig, rf, size, width, width, height) >> (bitdepth - 8);
    sad += (unsigned)(int)(lambda * (double)orc_quote_mv_bits((int16_t)(cand.y - mvp->y), (int16_t)(cand.x - mvp->x)) + 0.5);
    if (sad < min_sad) { min_sad = sad; opt = cand; }
  }
  *mv = opt;
  return (int)min_sad;
}

/* ---- a9/a5 element-wise block combinations: op 0 average_blocks_all (a+b)>>1 (common/inter_prediction.c:228-247),
 * op 1 bipred search target sat(2a - b) (enc/encode_block.c:1780-1782), op 2 block_avg (a+b+1)>>1 ---- */
void FN(orc_block_combine)(S *dst, int ds, const S *a, int as, const S *b, int bs, int w, int h, int op, int bitdepth) {
  int maxv = (1 << bitdepth) - 1;
  for (int i = 0; i < h; i++)
    for (int j = 0; j < w; j++) {
      int x = a[i * as + j], y = b[i * bs + j], v;
      if (op == 0) v = (x + y) >> 1;
      else if (op == 1) v = orc_sat(2 * (int16_t)x - (int16_t)y, maxv);
      else v = (x + y + 1) >> 1;
      dst[i * ds + j] = (S)v;
    }
}

/* enc/encode_frame.c:194-221: perceptual 8x8 distortion; src = original, dst = filtered.  ISO-C double arithmetic
 * (no contraction): ((A * .5) * B) / sqrt(C + svar * dvar), floor(.5 + ...). */
uint64_t FN(orc_dist_8x8)(const S *dst, int dstride, const S *src, int sstride, int coeff_shift) {
  uint64_t sum_s = 0, sum_d = 0, sum_s2 = 0, sum_d2 = 0, sum_sd = 0;
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) {
      uint64_t s = src[i * sstride + j], d = dst[i * dstride + j];
      sum_s += s; sum_d += d; sum_s2 += s * s; sum_d2 += d * d; sum_sd += s * d;
    }
  uint64_t svar = sum_s2 - ((sum_s * sum_s + 32) >> 6), dvar = sum_d2 - ((sum_d * sum_d + 32) >> 6);
  return (uint64_t)floor(.5 + (sum_d2 + sum_s2 - 2 * sum_sd) * .5 * (svar + dvar + (400 << 2 * coeff_shift)) / (sqrt((20000 << 4 * coeff_shift) + svar * (double)dvar)));
}

/* ---- a19 (encoder): the pixel work of cdef_search.  enc/encode_frame.c:228-376.
 * For every 64x64 filter block that is not all-skip, every plane and every strength index gi < total (= pristrengths[speed]),
 * the distortion of the CDEF-filtered blocks against the original: dist_8x8 (double arithmetic, :194-221) for full 8x8 luma
 * blocks, plain SSE otherwise (U and V accumulate into the same slot).  Reference quirks reproduced: the search filters chroma
 * in 8x8 blocks taken from the top-left 32x32 of the filter block's block-info/direction grid, and passes sec_strength
 * unadjusted (0..3) whereas cdef_frame applies 4 for 3.
 *   mse[(plane != 0) * nfb * 64 + fb * 64 + gi], dirs/vars[fb * 64 + m*8+n], allskip[fb]; fb = raster index of the filter block */
void FN(orc_cdef_search_mse)(const S *recY, const S *recU, const S *recV, const S *orgY, const S *orgU, const S *orgV, int sy, int sc, int width, int height,
                             const orc_blkinfo_t *bi, int speed, int pri_damping, int bitdepth, uint64_t *mse, int *dirs, int *vars, uint8_t *allskip_out) {
  static const int priconv[3][16] = {{0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {0, 1, 2, 3, 5, 7, 10, 13}, {0, 1, 3, 6}};
  static const int pristrengths[3] = {64, 32, 16};
  const int total = pristrengths[speed], nh = (width + 63) >> 6, nv = (height + 63) >> 6, nfb = nh * nv, cs = bitdepth - 8;
  static uint16_t tile[(64 + 4) * 80];
  S dst[64];
  for (int k = 0, ci = 0; k < nv; k++)
    for (int l = 0; l < nh; l++, ci++) {
      const int xoff = l << 6, yoff = k << 6;
      int allskip = 1;
      for (int m = 0; allskip && m < 8; m++)
        for (int n = 0; allskip && n < 8; n++) {
          int xp = xoff + n * 8, yp = yoff + m * 8;
          if (xp < width && yp < height) allskip &= bi[(yp / 4) * (width / 4) + xp / 4].mode == 0;
        }
      allskip_out[ci] = (uint8_t)allskip;
      for (int gi = 0; gi < 64; gi++) mse[ci * 64 + gi] = mse[(size_t)nfb * 64 + ci * 64 + gi] = 0;
      if (allskip) continue;
      int h = (height < ((k + 1) << 6) ? height : ((k + 1) << 6)) & 63, w = (width < ((l + 1) << 6) ? width : ((l + 1) << 6)) & 63;
      h += !h << 6;
      w += !w << 6;
      for (int plane = 0; plane < 3; plane++) {
        const int sub = plane != 0, sstride = plane ? sc : sy;
        const S *src = plane ? (plane == 1 ? recU : recV) : recY, *org = plane ? (plane == 1 ? orgU : orgV) : orgY;
        int fsx = (width - xoff < 64 ? width - xoff : 64) >> sub, fsy = (height - yoff < 64 ? height - yoff : 64) >> sub;
        int fx = xoff >> sub, fy = yoff >> sub;
        int bt = (fx == 0 ? 1 : 0) | (fy == 0 ? 4 : 0) | (fx == (width >> sub) - fsx ? 2 : 0) | (fy == (height >> sub) - fsy ? 8 : 0);
        FN(orc_cdef_prepare_input)(fsx, fsy, fx, fy, bt, 2, tile + 2 * 80 + 2, 80, src, sstride);
        for (int gi = 0; gi < total; gi++) {
          const int pri = priconv[speed][gi / 4], sec = gi % 4;
          for (int m = 0; m < ((h + 7) >> (3 + sub)); m++)
            for (int n = 0; n < ((w + 7) >> (3 + sub)); n++) {
              int xpos = fx + n * 8, ypos = fy + m * 8;
              int sizex = (width >> sub) - xpos < 8 ? (width >> sub) - xpos : 8, sizey = (height >> sub) - ypos < 8 ? (height >> sub) - ypos : 8;
              int index = ((yoff + m * 8) / 4) * (width / 4) + (xoff + n * 8) / 4;
              if (plane == 0 && gi == 0) dirs[ci * 64 + m * 8 + n] = FN(orc_cdef_find_dir)(src + ypos * sstride + xpos, sstride, &vars[ci * 64 + m * 8 + n], cs);
              if (bi[index].mode == 0) continue;
              int adj = plane ? pri : orc_adjust_strength(pri, vars[ci * 64 + m * 8 + n]);
              int pd = pri_damping - !!plane, sd = pri_damping - !!plane;
              if (adj && orc_log2i(adj) > pd) pd = orc_log2i(adj);
              orc_cdef_filter_block(sizeof(S) == 1 ? (uint8_t *)dst : NULL, sizeof(S) == 1 ? NULL : (uint16_t *)dst, sizex, tile + 2 * 80 + 2 + n * 8 + m * 8 * 80, 80,
                                    adj << cs, sec << cs, pri ? dirs[ci * 64 + m * 8 + n] : 0, pd + cs, sd + cs, sizex, cs);
              const S *ob = org + ypos * sstride + xpos;
              uint64_t *acc = &mse[(size_t)(plane != 0) * nfb * 64 + ci * 64 + gi];
              if (plane || sizex != 8 || sizey != 8) {
                for (int i = 0; i < sizey; i++)
                  for (int j = 0; j < sizex; j++) { int d = (int)dst[i * sizex + j] - (int)ob[i * sstride + j]; *acc += (uint64_t)(int64_t)(d * d); }
              } else
                *acc += FN(orc_dist_8x8)(dst, sizex, ob, sstride, cs);
            }
        }
      }
    }
}
