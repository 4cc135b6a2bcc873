/* thor_b200.h — C ABI of libthor_b200.so, the H100 (sm_90a) implementation of the cisco/thor per-block hot path.
 *
 * Two faces (DESIGN.md §2):
 *
 *  (A) DROP-IN SYMBOLS.  Exactly the functions the reference's four kernel objects export and its host objects
 *      call (enc/enc_kernels.o, enc/enc_kernels_hbd.o, common/common_kernels.o, common/common_kernels_hbd.o;
 *      list: SURVEY.md §8b).  Same names, argument order, pointer/stride conventions and return values as
 *      /root/reference/enc/enc_kernels.h:32-40 and /root/reference/common/common_kernels.h:33-43, 69-76, so the
 *      reference's encode_block.o / encode_frame.o / transform.o / inter_prediction.o / temporal_interp.o /
 *      common_frame.o link against this library unchanged.  Caller owns every buffer (host memory); each call
 *      stages its operands into HBM, runs the CUDA kernel, and copies the result back before returning.
 *      There is NO CPU fallback: without a usable CUDA device the first call aborts like the reference's
 *      fatalerror() (common/global.h:38-44).
 *
 *  (B) BATCHED ENTRY POINTS (tb_*).  The same kernels over arrays of work items whose operands are already
 *      resident in HBM (frames uploaded once with tb_frame_*), one launch per batch.  This is the form a
 *      batching host RD loop uses; pointers inside items are DEVICE pointers obtained from tb_frame_plane().
 *
 * All functions are extern "C", take plain pointers and sizes, and are safe to call from one host thread
 * (like the reference, which is single-threaded; SURVEY.md §8b "Threading").
 */
#ifndef THOR_B200_H
#define THOR_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------------------
 * (A) drop-in symbols.  `_lbd`: SAMPLE = uint8_t, `_hbd`: SAMPLE = uint16_t (reference TEMPLATE(), types.h:35-38)
 * ---------------------------------------------------------------------------------------------------------- */
struct tb_yuv_frame; /* layout-compatible with the reference's yuv_frame_t (common/types.h:58-80) */

#define TB_DECL_SAMPLE_SYMBOLS(S, SFX)                                                                                                   \
  /* enc/enc_kernels.h:32-38 (definitions enc/enc_kernels.c:36, 119, 257, 296, 330, 516, 84) */                                          \
  int sad_calc_simd_##SFX(S *a, S *b, int astride, int bstride, int width, int height);                                                  \
  uint64_t ssd_calc_simd_##SFX(S *a, S *b, int astride, int bstride, int size);                                                          \
  void detect_clpf_simd_##SFX(const S *rec, const S *org, int x0, int y0, int width, int height, int so, int stride, int *sum0,          \
                              int *sum1, unsigned int strength, unsigned int shift, unsigned int size, unsigned int dmp);                \
  void detect_multi_clpf_simd_##SFX(const S *rec, const S *org, int x0, int y0, int width, int height, int so, int stride, int *sum,     \
                                    unsigned int shift, unsigned int size, unsigned int dmp);                                            \
  unsigned int sad_calc_fasthalf_simd_##SFX(const S *a, const S *b, int astride, int bstride, int width, int height, int *x, int *y);    \
  unsigned int sad_calc_fastquarter_simd_##SFX(const S *o, const S *r, int os, int rs, int width, int height, int *x, int *y);           \
  unsigned int widesad_calc_simd_##SFX(S *a, S *b, int astride, int bstride, int width, int height, int *x);                             \
  /* common/common_kernels.h:33-43 (definitions common/common_kernels.c:38, 68, 2181, 2360, 1623-1845, 1847) */                          \
  void block_avg_simd_##SFX(S *p, S *r0, S *r1, int sp, int s0, int s1, int width, int height);                                          \
  int sad_calc_simd_unaligned_##SFX(S *a, S *b, int astride, int bstride, int width, int height);                                        \
  void get_inter_prediction_luma_simd_##SFX(int width, int height, int xoff, int yoff, S *qp, int qstride, const S *ip, int istride,     \
                                            int bipred, int bitdepth);                                                                   \
  void get_inter_prediction_chroma_simd_##SFX(int width, int height, int xoff, int yoff, S *qp, int qstride, const S *ip, int istride,   \
                                              int bitdepth);                                                                             \
  void clpf_block4_##SFX(const S *src, S *dst, int sstride, int dstride, int x0, int y0, int sizey, int bt, unsigned int strength,       \
                         unsigned int dmp);                                                                                              \
  void clpf_block8_##SFX(const S *src, S *dst, int sstride, int dstride, int x0, int y0, int sizey, int bt, unsigned int strength,       \
                         unsigned int dmp);                                                                                              \
  void clpf_block4_noclip_##SFX(const S *src, S *dst, int sstride, int dstride, int x0, int y0, int sizey, unsigned int strength,        \
                                unsigned int dmp);                                                                                       \
  void clpf_block8_noclip_##SFX(const S *src, S *dst, int sstride, int dstride, int x0, int y0, int sizey, unsigned int strength,        \
                                unsigned int dmp);                                                                                       \
  void scale_frame_down2x2_simd_##SFX(struct tb_yuv_frame *sin, struct tb_yuv_frame *sout);                                              \
  /* common/common_kernels.h:73 (definition common/common_kernels.c:2533) */                                                             \
  int cdef_find_dir_simd_##SFX(const S *img, int stride, int32_t *var, int coeff_shift);

TB_DECL_SAMPLE_SYMBOLS(uint8_t, lbd)
TB_DECL_SAMPLE_SYMBOLS(uint16_t, hbd)

/* bit-depth independent symbols of common/common_kernels.o and enc/enc_kernels.o */
void transform_simd(const int16_t *block, int16_t *coeff, int size, int fast, int bitdepth);    /* common_kernels.h:37, common_kernels.c:1482 */
void inverse_transform_simd(const int16_t *coeff, int16_t *block, int size, int bitdepth);      /* common_kernels.h:38, common_kernels.c:1563 */
int check_nz_area(const int16_t *coeff, int size);                                              /* common_kernels.c:128 */
int calc_cbp_simd(int16_t *block, int size, int threshold);                                     /* enc_kernels.h:40, enc_kernels.c:828 */
void cdef_filter_block_simd(uint8_t *dst8, uint16_t *dst16, int dstride, const uint16_t *in, int sstride, int pri_strength,
                            int sec_strength, int dir, int pri_damping, int sec_damping, int bsize, int cdef_directions[8][2],
                            int coeff_shift);                                                   /* common_kernels.h:69-72, common_kernels.c:3234 */
/* read-only data referenced by common/inter_prediction.c:47-49 from both the lbd and hbd builds */
extern const int16_t coeffs_standard_lbd[4][8], coeffs_bipred_lbd[4][8], coeffs_chroma_lbd[8][4];
extern const int16_t coeffs_standard_hbd[4][8], coeffs_bipred_hbd[4][8], coeffs_chroma_hbd[8][4];

/* ------------------------------------------------------------------------------------------------------------
 * (B) batched entry points
 * ---------------------------------------------------------------------------------------------------------- */
#define TB_OK 0
#define TB_ERR_CUDA (-1)
#define TB_ERR_ARG (-2)

/* Library / device management.  tb_init is optional (every entry point initialises lazily); it returns TB_OK or
 * TB_ERR_CUDA and never falls back to the CPU.  device < 0 selects $LOCAL_RANK or 0. */
int tb_init(int device);
const char *tb_last_error(void);
/* number of kernel launches issued by this library since load (bench.py's gpu_launches) */
uint64_t tb_launch_count(void);
void *tb_stream(void); /* the cudaStream_t every batched call is enqueued on (per-thread default unless tb_set_stream) */
int tb_set_stream(void *cuda_stream);
int tb_sync(void);

/* ---- frames resident in HBM, same geometry as the reference's yuv_frame_t (common/common_frame.c:435-469):
 * 4:2:0, luma pitch = (width + 2*pad + 15) & ~15 samples, chroma pad = pad/2.  sample_bytes = 1 (lbd) or 2 (hbd). */
typedef struct tb_frame tb_frame_t;
tb_frame_t *tb_frame_create(int width, int height, int pad, int sample_bytes);
void tb_frame_destroy(tb_frame_t *f);
/* copies of the visible area to/from caller memory (planes given with their pitches in samples).  The caller's buffers may be host
 * memory (pinned or pageable) or device memory (e.g. a buffer an NCCL scatter just filled): the copy kind is inferred (UVA). */
int tb_frame_upload(tb_frame_t *f, const void *y, int ystride, const void *u, const void *v, int cstride);
int tb_frame_download(const tb_frame_t *f, void *y, int ystride, void *u, void *v, int cstride);
/* same, without waiting: the host buffers (pinned) are valid once the current stream has been synchronised */
int tb_frame_download_async(const tb_frame_t *f, void *y, int ystride, void *u, void *v, int cstride);
/* device pointer to sample (0,0) of plane p (0 Y, 1 U, 2 V) and its pitch in samples */
void *tb_frame_plane(const tb_frame_t *f, int plane, int *stride);

/* ---- a1/a2/a3: SAD / five-position wide SAD / SSD over (a, b) block pairs (device pointers) */
typedef struct {
  const void *a, *b; /* a: original block, b: reference position */
  int32_t astride, bstride;
  uint16_t width, height;
  uint32_t pad;
} tb_sad_item_t;
/* out[i] = SAD; kind 0: sad (enc/encode_block.c:417), 1: widesad -> out2[i] = best x offset (:430), 2: ssd -> out64 (:455) */
int tb_sad_batch(const tb_sad_item_t *items_dev, int n, int sample_bytes, int kind, uint32_t *out_dev, int32_t *out2_dev, uint64_t *out64_dev);

/* ---- a5: complete uni-directional motion search of enc/encode_block.c:517-711, one search per item */
typedef struct {
  const void *orig; /* device ptr: first sample of the prediction block inside the ORIGINAL frame (or a compact block) */
  const void *ref;  /* device ptr: same position inside the padded reference frame */
  int32_t ostride, rstride;
  int16_t xpos, ypos;       /* luma position of the CODING block (clip_mv / interpolation clamp use it) */
  uint8_t size;             /* coding-block size (clip_mv block dimensions) */
  uint8_t width, height;    /* prediction-block dimensions */
  uint8_t sign;             /* 1: reference later than the current frame in display order */
  int16_t mvc_x, mvc_y;     /* search centre  (quarter-pel) */
  int16_t mvp_x, mvp_y;     /* MV predictor   (quarter-pel) */
  int32_t cand_ofs;         /* first candidate in the cand array (integer-pel int16 x,y pairs) */
  int32_t ncand;
  double lambda;            /* the `lambda` argument of motion_estimate (= sqrt(frame lambda) at the call site) */
} tb_me_item_t;
typedef struct { int16_t mvx, mvy; uint32_t cost; } tb_me_result_t;
int tb_motion_estimate_batch(const tb_me_item_t *items_dev, int n, const int16_t *cand_dev, int sample_bytes, int bitdepth,
                             int encoder_speed, int enable_bipred, int fwidth, int fheight, tb_me_result_t *out_dev);

/* ---- a5: simultaneous bi-directional search (mv0 = -mv1) of motion_estimate_bi(), enc/encode_block.c:798-914 (B frames, speed 0).
 * cand: up to four list entries used AS quarter-pel vectors (sic), like frame_info->mvcand at that call site. */
typedef struct {
  const void *orig, *ref0, *ref1; /* device ptrs at the coding block's position */
  int32_t ostride, rstride;
  int16_t xpos, ypos;
  uint8_t size, sign, pad0, pad1;
  int16_t mvc_x, mvc_y, mvp_x, mvp_y;
  int32_t cand_ofs, ncand;
  double lambda;
} tb_me_bi_item_t;
int tb_motion_estimate_bi_batch(const tb_me_bi_item_t *items_dev, int n, const int16_t *cand_dev, int sample_bytes, int bitdepth, int enable_bipred,
                                int fwidth, int fheight, tb_me_result_t *out_dev);

/* ---- a9 / a5 element-wise block combinations: op 0 average_blocks_all (a+b)>>1 (common/inter_prediction.c:228), op 1 the bipred search
 * target sat(2a - b) (enc/encode_block.c:1780), op 2 block_avg (a+b+1)>>1 (common/common_kernels.c:38) */
typedef struct {
  const void *a, *b;
  void *dst;
  int32_t astride, bstride, dstride;
  uint16_t width, height;
} tb_combine_item_t;
int tb_block_combine_batch(const tb_combine_item_t *items_dev, int n, int sample_bytes, int op, int bitdepth);

/* optional work counters for the roofline: 5 uint64 in HBM {searches, integer-position block SADs, sub-pel probes,
 * samples compared at integer positions (incl. one read of the original block), samples read+written by the sub-pel probes};
 * NULL (default) disables counting */
int tb_me_set_stats(uint64_t *stats_dev);

/* ---- a7/a8: sub-pel interpolation, one prediction block per item (common/inter_prediction.c:65-183) */
typedef struct {
  const void *ref; /* device ptr: block position in the padded reference plane */
  void *dst;       /* device ptr: output block */
  int32_t rstride, dstride;
  int16_t xpos, ypos;    /* block position in the plane (for the normative clamp) */
  int16_t mvx, mvy;      /* quarter-pel (luma) or eighth-pel (chroma) MV, already clip_mv'ed */
  uint8_t width, height; /* block dimensions */
  uint8_t sign, chroma;
  int16_t pic_w, pic_h;  /* plane dimensions passed to the reference (pic_width/pic_height) */
  uint32_t pad;
} tb_interp_item_t;
int tb_interp_batch(const tb_interp_item_t *items_dev, int n, int sample_bytes, int bitdepth, int bipred);

/* ---- a10-a13 + a3: residual -> forward DCT -> quantise -> de-quantise -> inverse DCT -> reconstruct -> SSD,
 * one transform block per item (the body of encode_and_reconstruct_block_*, enc/encode_block.c:1100-1338) */
typedef struct {
  const void *orig, *pred; /* device ptrs */
  void *rec;               /* device ptr: reconstruction out (required; may alias nothing) */
  int16_t *coeffq;         /* device ptr: min(size,16)^2 quantised coefficients out (raster order), or NULL */
  int32_t ostride, pstride, rstride;
  uint8_t size, qp, coeff_type, fast; /* coeff_type: COEFF_TYPE_* (common/global.h:103-106); fast: TB_TXFM_* flags */
} tb_txfm_item_t;
#define TB_TXFM_FAST 1 /* encoder_info->params->encoder_speed > 1: 16-point transform for 32x32 (common/transform.c:252) */
#define TB_TXFM_BITS 2 /* also count the bits write_coeff() would emit for the block (enc/write_bits.c:145-242), SURVEY 8f.2 */
typedef struct { uint64_t ssd; int32_t cbp; int32_t bits; } tb_txfm_result_t; /* bits: 0 unless TB_TXFM_BITS and cbp != 0 */
int tb_txfm_chain_batch(const tb_txfm_item_t *items_dev, int n, int sample_bytes, int bitdepth, tb_txfm_result_t *out_dev);

/* ---- a15/a16: intra prediction from gathered neighbours (common/intra_prediction.c:185-428) and CfL */
typedef struct {
  const void *rec; /* device ptr: the coding block's top-left sample in the reconstructed plane */
  void *dst;       /* device ptr: size x size prediction out (pitch = size) */
  int32_t rstride;
  int16_t xpos, ypos;
  uint8_t size, mode, upright, downleft;
} tb_intra_item_t;
int tb_intra_batch(const tb_intra_item_t *items_dev, int n, int sample_bytes, int bitdepth);

/* ---- a17-a20: frame-level in-loop filters on resident frames.  blkinfo: one 16-byte record per 4x4 luma block
 * in raster order ((height/4) x (width/4)), the subset of deblock_data_t the filters read (common/types.h:178-187) */
typedef struct {
  uint8_t mode, cbp_y, size, tb_split, pb_part, pad[3];
  int16_t mv0x, mv0y, mv1x, mv1y;
} tb_blkinfo_t;
int tb_deblock_frame(tb_frame_t *rec, const tb_blkinfo_t *blkinfo_dev, int qp, int bitdepth); /* y + uv, common_frame.c:47, 354 */
/* plane < 0: all three planes.  fb_on_dev: optional per-filter-block flags (luma only) */
int tb_clpf_frame(tb_frame_t *rec, tb_frame_t *scratch, const tb_blkinfo_t *blkinfo_dev, const uint8_t *fb_on_dev, int fb_size_log2,
                  int strength, int bitdepth, int plane, int qp); /* common_frame.c:1005 */
/* per-8x8 block sums of detect_multi_clpf (enc/encode_block.c:2593): out[(by*bw+bx)*4 + k] */
int tb_clpf_detect_frame(const tb_frame_t *rec, const tb_frame_t *org, const tb_blkinfo_t *blkinfo_dev, int plane, int bitdepth, int qp,
                         int32_t *sums_dev);
/* CDEF with per-64x64 strengths (cdef_strength.level / .sec_strength, luma = plane class 0, chroma = 1);
 * dirvar_dev: 2*64 ints per filter block (dir, var), produced by the luma pass and consumed by the chroma passes */
int tb_cdef_frame(tb_frame_t *rec, tb_frame_t *scratch, const tb_blkinfo_t *blkinfo_dev, const int8_t *fb_pri_dev, const int8_t *fb_sec_dev,
                  int pri_damping, int sec_damping, int32_t *dirvar_dev, int bitdepth, int plane); /* common_frame.c:826 */
/* a19 (encoder): the pixel work of cdef_search (enc/encode_frame.c:285-376) — per 64x64 filter block fb (raster), plane class c (0 luma,
 * 1 = U+V) and strength index gi < {64,32,16}[speed]: mse[(c * nfb + fb) * 64 + gi] (dist_8x8 for full luma 8x8 blocks, SSE otherwise),
 * plus allskip[fb] and the dir/var table (layout of tb_cdef_frame).  The greedy preset selection (:58-192, 378-470) stays on the host. */
int tb_cdef_search_mse(const tb_frame_t *rec, const tb_frame_t *org, const tb_blkinfo_t *blkinfo_dev, int speed, int pri_damping, int bitdepth, int32_t *dirvar_dev,
                       uint8_t *allskip_dev, uint64_t *mse_dev);
int tb_pad_frame(tb_frame_t *f);                                         /* common_frame.c:657 */
int tb_create_reference_frame(tb_frame_t *ref, const tb_frame_t *rec);   /* common_frame.c:745 */
int tb_scale_down2x2(const tb_frame_t *in, tb_frame_t *out);             /* temporal_interp.c:143 (luma + pad) */

/* ---- a21: temporal frame interpolation, interpolate_frames() common/temporal_interp.c:909 (encoder enc/mainenc.c:353,409 and decoder
 * dec/decode_frame.c:110): writes the visible area of `out` (>= 16 samples of border required); the caller pads it (tb_pad_frame)
 * as the reference does.  ref0/ref1 must carry their replicated borders. */
int tb_interpolate_frames(tb_frame_t *out, const tb_frame_t *ref0, const tb_frame_t *ref1, int ratio, int pos);


/* ---- SURVEY 8f.1: device-resident RD loop.  tb_rdo_encode_frame() runs the reference's process_block() recursion
 * (enc/encode_block.c:2401-2565: early skip :2231-2399, mode_decision_rdo :1835-2120, encode_block :1340-1514, the bit
 * counting of write_block enc/write_bits.c:255-600, the MV predictors / skip / merge candidates common/inter_prediction.c:413-836 and
 * find_block_contexts common/common_block.c:283-303) for EVERY super block of one frame on the GPU (one CTA works on one super block at a time), super
 * blocks in a wavefront (left, up-left, up, up-right dependencies), and returns the decisions.  The host then only serialises them
 * (write_super_mode / write_block of the reference's own bit writer: thor_b200/csrc/tb_rdo_shim.c is that binding).
 * Supported: 4:2:0 at internal bit depth 8, 10 or 12, sync = 0, qmtx = 0, interp_ref != 2, max_delta_qp = 0, bitrate = 0 (every BASELINE.json configuration),
 * widths and heights that are multiples of 8, and in 16-bit frames (sample_bytes 2) widths that are multiples of 16 (the reference's SIMD chroma
 * interpolation treats 16-bit chroma widths of 4 mod 8 unlike its C code in rectangular frame-edge blocks); anything else returns TB_ERR_ARG and the binding falls back to the reference's host loop over the per-call drop-in kernels. */
typedef struct { int16_t x, y; } tb_mv_t; /* mv_t, common/types.h:132-136 */
typedef struct { /* per 4x4 luma block: the part of deblock_data_t (common/types.h:178-187) the RD loop and the in-loop filters read */
  uint8_t mode, size, tb_split, pb_part;
  uint8_t cbp_y, cbp_u, cbp_v;
  int8_t bipred_flag; /* inter_pred.bipred_flag: 0 uni, 2 bi, -1 intra */
  tb_mv_t mv0, mv1;
  uint8_t ref_idx0, ref_idx1, pad[2];
} tb_rdo_blk_t; /* 20 bytes */
typedef struct { /* one coded block (a leaf of a super block's quad-tree): everything write_block() needs */
  uint16_t xpos, ypos;
  uint8_t size, mode, intra_mode, skip_idx;
  uint8_t pb_part, tb_split, ref_idx0, ref_idx1;
  int8_t dir;
  uint8_t cbp_y, cbp_u, cbp_v; /* as coded (one bit per transform block when tb_split) */
  uint8_t num_skip_vec, num_merge_vec;
  int8_t ctx_index, ctx_cbp; /* block_context_t.index / .cbp */
  tb_mv_t mv_arr0[4], mv_arr1[4], mvp;
  int32_t coeff_ofs; /* first int16 of this block's quantised coefficients inside its super block's coefficient area; -1: none */
  uint32_t cost;     /* RD cost of the block as process_block() returns it */
} tb_rdo_leaf_t;     /* 64 bytes */
#define TB_RDO_MAX_REF 8
#define TB_RDO_MAX_LEAVES 256    /* 8x8 blocks in a 128x128 super block */
#define TB_RDO_SB_COEFFS 24576   /* int16 per super block: quantised coefficients never outnumber the samples (128*128*3/2) */
typedef struct {
  /* sequence / frame parameters (enc_params, frame_info_t: enc/mainenc.h:35-165) */
  int32_t width, height, log2_sb_size, bitdepth, sample_bytes; /* log2_sb_size 6 or 7, as the reference's encoder allows */
  int32_t frame_type; /* 0 I, 1 P, 2 B (frame_type_t) */
  int32_t qp, num_ref, interp_ref, num_intra_modes;
  double lambda;      /* frame_info.lambda = lambda_coeff * squared_lambda_QP[qp] */
  int32_t enable_bipred, enable_tb_split, enable_pb_split, encoder_speed, intra_rdo, use_block_contexts, cfl_intra, cfl_inter;
  float early_skip_thr;
  int32_t ref_sign[TB_RDO_MAX_REF];    /* per ref_idx: ref->frame_num >  rec->frame_num (encode_block.c:1975, 1437) */
  int32_t ref_sign_ge[TB_RDO_MAX_REF]; /* per ref_idx: ref->frame_num >= frame_info.frame_num (early skip, encode_block.c:2282, sic) */
  /* HOST pointers.  orig / rec: sample (0,0) of each plane; ref: sample (0,0) of padded planes with >= 160 (80) samples of border */
  const void *orig[3];
  int32_t orig_stride[2]; /* luma, chroma pitch in samples */
  const void *ref[TB_RDO_MAX_REF][3];
  int32_t ref_stride[2], ref_pad; /* ref_pad: luma border, >= 160 = the reference's PADDING_Y (the whole padded plane is uploaded) */
  void *rec[3];           /* out: reconstruction before the in-loop filters (visible area) */
  int32_t rec_stride[2];
  tb_rdo_blk_t *blk;      /* out: (height/4) x (width/4), raster */
  tb_rdo_leaf_t *leaves;  /* out: TB_RDO_MAX_LEAVES per super block (raster order of super blocks), coding order inside */
  int32_t *leaf_count;    /* out: per super block */
  int16_t *coeffs;        /* out: TB_RDO_SB_COEFFS per super block */
} tb_rdo_frame_t;
int tb_rdo_encode_frame(const tb_rdo_frame_t *f);
/* n INDEPENDENT frames (the B frames of one hierarchy level, frames of several sequences or intra-period segments) in ONE launch: persistent CTAs
 * draw ready super blocks from all of them, so the GPU is filled although one frame's wavefront is only a few super blocks wide.  All frames must
 * have the same sample size; geometry and parameters may differ.  Same outputs per frame as tb_rdo_encode_frame(). */
int tb_rdo_encode_frames(const tb_rdo_frame_t *f, int n);
/* The same in steps, for callers that keep frames resident or overlap the copies: every call only ENQUEUES on the library's stream
 * (tb_stream()); host buffers must stay valid until tb_rdo_batch_sync() (pinned buffers make the copies truly asynchronous).
 * Any sequence of calls may be enqueued before one sync, e.g. upload A, run, download A, upload B into the same slots, run, download B, sync: each
 * launch reads the uploads enqueued before it and each download returns the launch enqueued before it.  The host waits only where it must:
 *   - an upload into a slot whose previous upload's copies have not started yet waits for them (the frame parameters are staged per slot);
 *   - an upload that changes a slot's geometry (size, super-block size, sample size, reference padding or stride, or more than five references)
 *     reallocates it and first waits for the stream to drain; so does a run that needs more rows, super blocks or CTAs than any launch before;
 *   - a run with eight launches of the batch in flight waits for the oldest of them.
 * A run over [0, n_active) leaves slots >= n_active untouched: their downloads return the decisions of the last launch that included them, until
 * an upload changes their geometry. */
typedef struct tb_rdo_batch tb_rdo_batch_t;
tb_rdo_batch_t *tb_rdo_batch_create(int n_slots, int sample_bytes);                         /* NULL: tb_rdo_last_error() */
int tb_rdo_batch_upload(tb_rdo_batch_t *b, int slot, const tb_rdo_frame_t *f);              /* parameters + source + references -> HBM */
int tb_rdo_batch_run(tb_rdo_batch_t *b, int n_active);                                      /* one launch over slots [0, n_active) */
int tb_rdo_batch_download(tb_rdo_batch_t *b, int slot, const tb_rdo_frame_t *f);            /* decisions of a slot -> f's output buffers (rec[] may be NULL) */
int tb_rdo_batch_sync(tb_rdo_batch_t *b);                                                   /* waits; TB_ERR_CUDA if any launch since the previous sync did not
                                                                                               finish every super block */
int tb_rdo_batch_grid(const tb_rdo_batch_t *b);                                             /* CTAs of the last launch */
/* Stats and trace describe the last launch of the batch and are read after tb_rdo_batch_sync().
 * counters of the last synchronised launch, summed over all warps: [0..10] SM cycles per primitive class (interp, search, bipred search, transform
 * chain, coefficient bits, SSD/SAD, intra, copies, early skip, idle, total); [11..22] work actually executed (the RD loop is data dependent):
 * searches, integer block SADs, sub-pel probes, search samples (SURVEY 8d: (n_int+1) w h + n_sub ((w+5)(h+5) + w h)), predictions, prediction samples,
 * transform chains, chain samples (3 N^2), intra predictions, intra samples (4N + N^2), SSD/SAD samples (2 w h), super blocks */
#define TB_RDO_NSTATS 68 /* [23..39]: cycles of searches by coding-block size 8..128 (5), of transform chains by size 4..128 (6), of predictions by size 4..128 (6);
                            [40..48]: wall cycles of a CTA by decision phase (other, early skip, skip/merge candidates, searches, inter candidates, bipred, intra search,
                            intra candidates, commit); [49..53]: cycles of the searches of blocks <= 16 by stage (telescope, candidates, hexagon, half-pel, quarter-pel);
                            [54..59]: search phase of an overlapped decision, warp 0 and the last warp {own searches, -, barrier wait}; [60..65]: its bi-prediction
                            phase, warp 0 {chain, inter candidates, barrier wait} and the last warp {joint search as the helper, inter candidates, barrier wait};
                            [66..67]: overlapped B-frame decisions whose joint bi-prediction search ran on the helper warp, on warp 0 */
int tb_rdo_batch_stats(const tb_rdo_batch_t *b, uint64_t *out, int n);
/* timeline of the last synchronised launch: one entry per super block, in the order they finished.  Times are the GPU's global nanosecond
 * timer (%globaltimer), comparable between SMs.  A super block starts after the super blocks it depends on have ended. */
typedef struct {
  int32_t frame, row, col; /* slot of the batch, super-block row and column */
  int32_t cta;             /* blockIdx.x of the CTA that decided it */
  uint64_t t_start, t_end; /* ns */
} tb_rdo_sb_trace_t;
/* copies min(n, super blocks of the last launch) entries to out and returns how many (TB_ERR_CUDA if the copy fails);
 * out == NULL: returns the super blocks of the last launch */
int tb_rdo_batch_trace(const tb_rdo_batch_t *b, tb_rdo_sb_trace_t *out, int n);
void tb_rdo_batch_destroy(tb_rdo_batch_t *b);
const char *tb_rdo_last_error(void);
uint64_t tb_rdo_launch_count(void);
/* int16 coefficients a leaf stores for one plane: transform blocks packed back to back, each min(tsize,16)^2 in raster order */
static inline int tb_rdo_coeff_count(int size, int tb_split) {
  int t = tb_split ? size / 2 : size, q = t < 16 ? t : 16;
  return (tb_split ? 4 : 1) * q * q;
}

/* ---- single-block, HOST-buffer forms of host-object functions on the path (staged per call like the drop-in symbols) */
/* quantize(), enc/encode_block.c:84; returns cbp.  qp must be 0..51 (MAX_QP); any other qp returns TB_ERR_ARG and writes nothing */
int tb_quantize(const int16_t *coeff, int16_t *coeffq, int qp, int size, int coeff_block_type);
/* dequantize(), common/common_block.c:45.  qp must be 0..51 (MAX_QP); any other qp sets tb_last_error() and writes nothing */
void tb_dequantize(const int16_t *coeffq, int16_t *rcoeff, int qp, int size);
void tb_improve_uv_prediction(int sample_bytes, const void *y, void *u, void *v, const void *ry, int n, int cstride, int stride, int sub,
                              int bitdepth);                                                    /* improve_uv_prediction(), common/common_block.c:347 */

/* raw device memory helpers so that non-CUDA hosts (C, ctypes) can build item arrays */
void *tb_malloc(size_t bytes);
void tb_free(void *p);
int tb_memcpy_h2d(void *dst_dev, const void *src_host, size_t bytes);
int tb_memcpy_d2h(void *dst_host, const void *src_dev, size_t bytes);
/* enqueue only (pinned destination); pair with tb_sync() or an event on the stream given to tb_set_stream() */
int tb_memcpy_d2h_async(void *dst_host, const void *src_dev, size_t bytes);
int tb_memcpy_d2d(void *dst_dev, const void *src_dev, size_t bytes); /* enqueue only, on the library's stream */
void *tb_malloc_host(size_t bytes); /* pinned */
void tb_free_host(void *p);

#ifdef __cplusplus
}
#endif
#endif
