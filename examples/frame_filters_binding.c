/* examples/frame_filters_binding.c — the reference-side binding of INTEGRATION.md §2.1, as compilable C.
 *
 * What a cisco/thor maintainer adds to enc/encode_frame.c (and dec/decode_frame.c) to run the in-loop filters of one frame on the
 * device through the batched C ABI: pack deblock_data_t (common/types.h:178-187) into the 16-byte tb_blkinfo_t grid, upload the
 * reconstruction once, run deblocking / CDEF / CLPF / reference padding on HBM-resident planes, read the frame back only if the
 * host needs the samples (-rf, PSNR).  Compiled against the reference's own headers by tests/test_abi.py (syntax check) — it is
 * documentation that cannot rot, not part of the library.
 *
 * Build (from the reference tree):  gcc -std=c99 -I common -I enc -I $(THOR_B200)/include -c frame_filters_binding.c
 */
#include <stdlib.h>

#include "global.h"
#include "types.h"
#include "thor_b200.h"

typedef struct {
  tb_frame_t *rec, *scratch, *ref_out;
  tb_blkinfo_t *bi_host, *bi_dev;
  int8_t *fb_pri_dev[2], *fb_sec_dev[2];
  uint8_t *clpf_fb_on_dev;
  int32_t *dirvar_dev;
  int width, height, nblk, nfb;
} tb_filter_ctx;

/* once per sequence */
int tb_filter_ctx_create(tb_filter_ctx *c, int width, int height) {
  c->width = width; c->height = height;
  c->nblk = (width / MIN_PB_SIZE) * (height / MIN_PB_SIZE);
  c->nfb = ((width + 63) / 64) * ((height + 63) / 64);
  c->rec = tb_frame_create(width, height, PADDING_Y, (int)sizeof(SAMPLE));
  c->scratch = tb_frame_create(width, height, PADDING_Y, (int)sizeof(SAMPLE));
  c->ref_out = tb_frame_create(width, height, PADDING_Y, (int)sizeof(SAMPLE));
  c->bi_host = (tb_blkinfo_t *)tb_malloc_host((size_t)c->nblk * sizeof(tb_blkinfo_t));
  c->bi_dev = (tb_blkinfo_t *)tb_malloc((size_t)c->nblk * sizeof(tb_blkinfo_t));
  for (int k = 0; k < 2; k++) {
    c->fb_pri_dev[k] = (int8_t *)tb_malloc((size_t)c->nfb);
    c->fb_sec_dev[k] = (int8_t *)tb_malloc((size_t)c->nfb);
  }
  c->clpf_fb_on_dev = (uint8_t *)tb_malloc((size_t)((width + 15) / 16) * ((height + 15) / 16)); /* the smallest signalled CLPF block is 16x16 */
  c->dirvar_dev = (int32_t *)tb_malloc((size_t)c->nfb * 2 * 64 * sizeof(int32_t));
  return c->rec && c->scratch && c->ref_out && c->bi_host && c->bi_dev && c->clpf_fb_on_dev && c->dirvar_dev ? TB_OK : TB_ERR_CUDA;
}

/* per frame: replaces deblock_frame_y/_uv, cdef_frame x3, clpf_frame x3 and create_reference_frame (enc/encode_frame.c:748-835).
 * fb_pri / fb_sec: per 64x64 filter block, [0] luma, [1] chroma — cdef_strength.level / .sec_strength as chosen by cdef_search;
 * clpf_strength[plane] / clpf_log2[plane]: the outcome of clpf_rdo (0 = plane not filtered).
 * clpf_fb_on: the luma per-filter-block decisions, one byte per 2^clpf_log2[0] filter block in raster order (k * blocks per row + l), as the
 * encoder's clpf_decision callback returned them for (k, l) and as they were signalled; NULL when enable_fb_flag is 0 (every block that is not
 * all skip is filtered).  Chroma never carries such flags. */
int tb_filter_frame(tb_filter_ctx *c, yuv_frame_t *rec, const deblock_data_t *deblock_data, int qp, int bitdepth, int cdef_damping, const int8_t *fb_pri[2],
                    const int8_t *fb_sec[2], const int clpf_strength[3], const int clpf_log2[3], const uint8_t *clpf_fb_on, int download) {
  for (int i = 0; i < c->nblk; i++) { /* 364-byte deblock_data_t -> 16 bytes */
    const deblock_data_t *d = &deblock_data[i];
    tb_blkinfo_t *b = &c->bi_host[i];
    b->mode = (uint8_t)d->mode; b->cbp_y = (uint8_t)(d->cbp.y != 0); b->size = d->size; b->tb_split = d->tb_split; b->pb_part = (uint8_t)d->pb_part;
    b->mv0x = d->inter_pred.mv0.x; b->mv0y = d->inter_pred.mv0.y; b->mv1x = d->inter_pred.mv1.x; b->mv1y = d->inter_pred.mv1.y;
  }
  int rc = tb_memcpy_h2d(c->bi_dev, c->bi_host, (size_t)c->nblk * sizeof(tb_blkinfo_t));
  if (rc == TB_OK) rc = tb_frame_upload(c->rec, rec->y, rec->stride_y, rec->u, rec->v, rec->stride_c);
  if (rc == TB_OK) rc = tb_deblock_frame(c->rec, c->bi_dev, qp, bitdepth);
  for (int k = 0; k < 2 && rc == TB_OK; k++) {
    rc = tb_memcpy_h2d(c->fb_pri_dev[k], fb_pri[k], (size_t)c->nfb);
    if (rc == TB_OK) rc = tb_memcpy_h2d(c->fb_sec_dev[k], fb_sec[k], (size_t)c->nfb);
  }
  for (int plane = 0; plane < 3 && rc == TB_OK; plane++)
    rc = tb_cdef_frame(c->rec, c->scratch, c->bi_dev, c->fb_pri_dev[plane != 0], c->fb_sec_dev[plane != 0], cdef_damping, cdef_damping, c->dirvar_dev, bitdepth, plane);
  if (rc == TB_OK && clpf_strength[0] && clpf_fb_on) {
    const int fb = 1 << clpf_log2[0];
    rc = tb_memcpy_h2d(c->clpf_fb_on_dev, clpf_fb_on, (size_t)((c->width + fb - 1) / fb) * ((c->height + fb - 1) / fb));
  }
  for (int plane = 0; plane < 3 && rc == TB_OK; plane++)
    if (clpf_strength[plane])
      rc = tb_clpf_frame(c->rec, c->scratch, c->bi_dev, plane == 0 && clpf_fb_on ? c->clpf_fb_on_dev : NULL, clpf_log2[plane], clpf_strength[plane], bitdepth,
                         plane, qp);
  if (rc == TB_OK) rc = tb_create_reference_frame(c->ref_out, c->rec); /* padded reference stays in HBM for the next frame's searches */
  if (rc == TB_OK && download) rc = tb_frame_download(c->rec, rec->y, rec->stride_y, rec->u, rec->v, rec->stride_c);
  return rc;
}
