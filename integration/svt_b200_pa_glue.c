/* svt_b200_pa_glue.c -- see svt_b200_pa_glue.h.  Compiled against the reference's headers (Source/Lib/Codec). */
#include <string.h>
#include "definitions.h"
#include "pcs.h"
#include "sequence_control_set.h"
#include "me_context.h"
#include "svt_b200_pa_glue.h"

void svt_b200_pa_controls_from_scs(const SequenceControlSet* scs, SvtB200PaStatsControls* c) {
    memset(c, 0, sizeof(*c));
    c->calculate_variance = scs->calculate_variance;
    c->block_mean_calc_prec = scs->block_mean_calc_prec == BLOCK_MEAN_PREC_SUB; /* pic_analysis_process.c:331: anything else is FULL */
    c->var_8x8 = scs->static_config.enable_adaptive_quantization == 1 || scs->static_config.variance_octile;
    c->calc_hist = scs->calc_hist;
    c->decim_step = scs->static_config.scene_change_detection ? 1 : 4;
    c->regions_w = (int32_t)scs->picture_analysis_number_of_regions_per_width;
    c->regions_h = (int32_t)scs->picture_analysis_number_of_regions_per_height;
}

void svt_b200_pa_store_results(const SequenceControlSet* scs, PictureParentControlSet* pcs, const uint16_t* variance,
                               uint16_t pic_avg_variance, const uint32_t* histogram, const uint8_t* average_intensity, uint64_t avg_luma) {
    SvtB200PaStatsControls c;
    svt_b200_pa_controls_from_scs(scs, &c);
    pcs->avg_luma = avg_luma;
    if (c.calc_hist)
        for (int w = 0; w < c.regions_w; w++)
            for (int h = 0; h < c.regions_h; h++) {
                const int r = w * c.regions_h + h;
                memcpy(pcs->picture_histogram[w][h], histogram + (size_t)r * HISTOGRAM_NUMBER_OF_BINS, HISTOGRAM_NUMBER_OF_BINS * sizeof(uint32_t));
                pcs->average_intensity_per_region[w][h] = average_intensity[r];
            }
    pcs->pic_avg_variance = pic_avg_variance;
    if (c.calculate_variance)
        for (int b = 0; b < pcs->b64_total_count; b++) {
            if (c.var_8x8)
                memcpy(pcs->variance[b], variance + (size_t)b * 85, 85 * sizeof(uint16_t));
            else
                pcs->variance[b][ME_TIER_ZERO_PU_64x64] = variance[(size_t)b * 85];
        }
}
