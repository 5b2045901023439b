/* oracle/ref_pa_stats.c -- TEST / BASELINE INFRASTRUCTURE, compiled into oracle/_ref/libsvtav1_pa_stats.so (oracle/pa_stats.mk),
 * which takes every reference symbol from oracle/_ref/libsvtav1_ref.so.
 *
 * The picture-analysis statistics through the reference's OWN svt_aom_gathering_picture_statistics
 * (pic_analysis_process.c:1559): block variances, region histograms, average intensities, avg_luma and pic_avg_variance
 * of a padded 8-bit picture and its 1/16 picture, as the picture-analysis process computes them.  What this file does is
 * what the encoder does around that call: allocate the SequenceControlSet / PictureParentControlSet fields it reads and
 * writes and point EbPictureBufferDescs at the caller's planes.  Every output starts from the caller's arrays (pre-filled
 * with a sentinel by the tests), so an entry the reference does not write comes back unchanged.  The same picture also
 * takes the device results through the integration glue (ref_pa_stats_store), and the controls the tests hand to the
 * device call come from the glue (svt_b200_pa_controls_from_scs).  Nothing here is used by the product. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "definitions.h"
#include "pcs.h"
#include "sequence_control_set.h"
#include "pd_process.h"
#include "svt_b200.h"
#include "svt_b200_pa_glue.h"

/* the scs fields svt_aom_gathering_picture_statistics reads */
typedef struct RefPaStatsCfg {
    int32_t calculate_variance, block_mean_calc_prec, enable_adaptive_quantization, variance_octile;
    int32_t calc_hist, scene_change_detection, regions_w, regions_h;
} RefPaStatsCfg;

/* host arrays: variance [n_b64][85], histogram [regions_w][regions_h][256], average_intensity [regions_w][regions_h] (the pcs
 * field is uint64), one pic_avg_variance and one avg_luma; read before the call, written after it */
typedef struct RefPaStatsOut {
    uint16_t* variance;
    uint16_t* pic_avg_variance;
    uint32_t* histogram;
    uint64_t* average_intensity;
    uint64_t* avg_luma;
} RefPaStatsOut;

typedef struct PaJob {
    SequenceControlSet*      scs;
    PictureParentControlSet* pcs;
    EbPictureBufferDesc      full, sixteenth;
    int                      n_b64, rw, rh;
} PaJob;

static void fill_desc(EbPictureBufferDesc* d, const SvtB200MePicture* p, int level) {
    memset(d, 0, sizeof(*d));
    d->buffer_y = (uint8_t*)p->plane[level];
    d->stride_y = (uint16_t)p->stride[level];
    d->org_x    = (uint16_t)p->org_x[level];
    d->org_y    = (uint16_t)p->org_y[level];
    d->width    = (uint16_t)p->width[level];
    d->height   = (uint16_t)p->height[level];
    d->max_width = d->width; d->max_height = d->height;
    d->bit_depth = EB_EIGHT_BIT;
}

static void job_open(PaJob* j, const SvtB200MePicture* pic, const RefPaStatsCfg* cfg, const RefPaStatsOut* out) {
    SequenceControlSet* scs = (SequenceControlSet*)calloc(1, sizeof(SequenceControlSet));
    PictureParentControlSet* pcs = (PictureParentControlSet*)calloc(1, sizeof(PictureParentControlSet));
    scs->calculate_variance = (uint8_t)cfg->calculate_variance;
    scs->block_mean_calc_prec = cfg->block_mean_calc_prec ? BLOCK_MEAN_PREC_SUB : BLOCK_MEAN_PREC_FULL;
    scs->static_config.enable_adaptive_quantization = (uint8_t)cfg->enable_adaptive_quantization;
    scs->static_config.variance_octile = (uint8_t)cfg->variance_octile;
    scs->calc_hist = (uint8_t)cfg->calc_hist;
    scs->static_config.scene_change_detection = (uint32_t)cfg->scene_change_detection;
    scs->picture_analysis_number_of_regions_per_width = (uint32_t)cfg->regions_w;
    scs->picture_analysis_number_of_regions_per_height = (uint32_t)cfg->regions_h;
    fill_desc(&j->full, pic, 2);
    fill_desc(&j->sixteenth, pic, 0);
    const int bw = (pic->width[2] + 63) / 64, bh = (pic->height[2] + 63) / 64;
    j->n_b64 = bw * bh;
    j->rw = cfg->regions_w;
    j->rh = cfg->regions_h;
    pcs->b64_total_count = (uint16_t)j->n_b64;
    pcs->b64_geom = (B64Geom*)calloc((size_t)j->n_b64, sizeof(B64Geom));
    pcs->variance = (uint16_t**)calloc((size_t)j->n_b64, sizeof(uint16_t*));
    for (int b = 0; b < j->n_b64; b++) { /* pcs.c:1504-1512 */
        pcs->b64_geom[b].horizontal_index = (uint8_t)(b % bw);
        pcs->b64_geom[b].vertical_index = (uint8_t)(b / bw);
        pcs->b64_geom[b].org_x = (uint16_t)(64 * (b % bw));
        pcs->b64_geom[b].org_y = (uint16_t)(64 * (b / bw));
        pcs->variance[b] = (uint16_t*)malloc(85 * sizeof(uint16_t));
        memcpy(pcs->variance[b], out->variance + (size_t)b * 85, 85 * sizeof(uint16_t));
    }
    pcs->picture_histogram = (uint32_t***)calloc(MAX_NUMBER_OF_REGIONS_IN_WIDTH, sizeof(uint32_t**));
    for (int w = 0; w < MAX_NUMBER_OF_REGIONS_IN_WIDTH; w++) {
        pcs->picture_histogram[w] = (uint32_t**)calloc(MAX_NUMBER_OF_REGIONS_IN_HEIGHT, sizeof(uint32_t*));
        for (int h = 0; h < MAX_NUMBER_OF_REGIONS_IN_HEIGHT; h++)
            pcs->picture_histogram[w][h] = (uint32_t*)calloc(HISTOGRAM_NUMBER_OF_BINS, sizeof(uint32_t));
    }
    for (int w = 0; w < j->rw; w++)
        for (int h = 0; h < j->rh; h++) {
            memcpy(pcs->picture_histogram[w][h], out->histogram + (size_t)(w * j->rh + h) * HISTOGRAM_NUMBER_OF_BINS,
                   HISTOGRAM_NUMBER_OF_BINS * sizeof(uint32_t));
            pcs->average_intensity_per_region[w][h] = out->average_intensity[w * j->rh + h];
        }
    pcs->pic_avg_variance = *out->pic_avg_variance;
    pcs->avg_luma = *out->avg_luma;
    j->scs = scs;
    j->pcs = pcs;
}

static void job_close(PaJob* j, RefPaStatsOut* out) {
    PictureParentControlSet* pcs = j->pcs;
    for (int b = 0; b < j->n_b64; b++) {
        memcpy(out->variance + (size_t)b * 85, pcs->variance[b], 85 * sizeof(uint16_t));
        free(pcs->variance[b]);
    }
    for (int w = 0; w < MAX_NUMBER_OF_REGIONS_IN_WIDTH; w++) {
        for (int h = 0; h < MAX_NUMBER_OF_REGIONS_IN_HEIGHT; h++) {
            if (w < j->rw && h < j->rh) {
                memcpy(out->histogram + (size_t)(w * j->rh + h) * HISTOGRAM_NUMBER_OF_BINS, pcs->picture_histogram[w][h],
                       HISTOGRAM_NUMBER_OF_BINS * sizeof(uint32_t));
                out->average_intensity[w * j->rh + h] = pcs->average_intensity_per_region[w][h];
            }
            free(pcs->picture_histogram[w][h]);
        }
        free(pcs->picture_histogram[w]);
    }
    *out->pic_avg_variance = pcs->pic_avg_variance;
    *out->avg_luma = pcs->avg_luma;
    free(pcs->picture_histogram);
    free(pcs->variance);
    free(pcs->b64_geom);
    free(pcs);
    free(j->scs);
}

static int cfg_ok(const RefPaStatsCfg* cfg) {
    return cfg->regions_w >= 1 && cfg->regions_w <= MAX_NUMBER_OF_REGIONS_IN_WIDTH && cfg->regions_h >= 1 &&
           cfg->regions_h <= MAX_NUMBER_OF_REGIONS_IN_HEIGHT;
}

/* The reference's statistics of `pic` (levels 2 and 0) into `out`; `ctl` (if not NULL) receives the glue's controls for the
 * same scs. */
int ref_pa_stats(const SvtB200MePicture* pic, const RefPaStatsCfg* cfg, SvtB200PaStatsControls* ctl, RefPaStatsOut* out) {
    if (!cfg_ok(cfg)) return -1;
    PaJob j;
    job_open(&j, pic, cfg, out);
    if (ctl) svt_b200_pa_controls_from_scs(j.scs, ctl);
    svt_aom_gathering_picture_statistics(j.scs, j.pcs, &j.full, &j.sixteenth);
    job_close(&j, out);
    return 0;
}

/* The device results (host copies, SvtB200PaStatsResults layout) stored into the same pcs by the glue, then copied out like
 * ref_pa_stats's: equal outputs = the glue writes what the reference writes. */
int ref_pa_stats_store(const SvtB200MePicture* pic, const RefPaStatsCfg* cfg, const uint16_t* variance, uint16_t pic_avg_variance,
                       const uint32_t* histogram, const uint8_t* average_intensity, uint64_t avg_luma, RefPaStatsOut* out) {
    if (!cfg_ok(cfg)) return -1;
    PaJob j;
    job_open(&j, pic, cfg, out);
    svt_b200_pa_store_results(j.scs, j.pcs, variance, pic_avg_variance, histogram, average_intensity, avg_luma);
    job_close(&j, out);
    return 0;
}
