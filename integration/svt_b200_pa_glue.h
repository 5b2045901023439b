/* svt_b200_pa_glue.h -- reference-side glue of the T2 picture-analysis statistics call (svt_b200_picture_statistics_dev,
 * include/svt_b200.h).
 *
 * A reference build adds integration/svt_b200_pa_glue.c next to Source/Lib/Codec/pic_analysis_process.c.  In place of
 * svt_aom_gathering_picture_statistics (pic_analysis_process.c:2355) the picture-analysis process then does, once the
 * padded picture and its 1/16 picture are on the device (the ME pyramid, SvtB200MePicture):
 *     svt_b200_pa_controls_from_scs(scs, &ctl);                         // this file
 *     svt_b200_picture_statistics_dev(&pic, &ctl, &dev_out, stream);
 *     (one D2H copy of the results)
 *     svt_b200_pa_store_results(scs, pcs, host arrays...);              // this file
 * Both functions are compiled against the reference's own headers (a renamed or re-typed field is a compile error) and are
 * exercised by the parity tests through oracle/ref_pa_stats.c. */
#ifndef SVT_B200_PA_GLUE_H
#define SVT_B200_PA_GLUE_H
#include <stdint.h>
#include "svt_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
struct SequenceControlSet;
struct PictureParentControlSet;
/* the SequenceControlSet fields svt_aom_gathering_picture_statistics reads -> SvtB200PaStatsControls */
void svt_b200_pa_controls_from_scs(const struct SequenceControlSet* scs, SvtB200PaStatsControls* ctl);
/* host copies of the call's outputs (laid out as SvtB200PaStatsResults documents) -> pcs->variance, pic_avg_variance,
 * picture_histogram, average_intensity_per_region and avg_luma.  Only what the reference writes under these controls is
 * stored: the variances 1..84 when the 8x8 flag is off, the histogram fields when calc_hist is off and the variances when
 * calculate_variance is off are left as they were. */
void svt_b200_pa_store_results(const struct SequenceControlSet* scs, struct PictureParentControlSet* pcs, const uint16_t* variance,
                               uint16_t pic_avg_variance, const uint32_t* histogram, const uint8_t* average_intensity, uint64_t avg_luma);
#ifdef __cplusplus
}
#endif
#endif
