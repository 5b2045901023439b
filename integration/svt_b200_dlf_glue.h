/* svt_b200_dlf_glue.h -- reference-side glue of the T2 deblocking call svt_b200_loop_filter_frame_dev.
 *
 * Compiled INSIDE the reference tree (it reads PictureControlSet, ModeInfo and LoopFilterInfoN).  A maintainer who moves
 * deblocking onto the H100 calls, with the picture's reconstruction on the device:
 *   - picture-level deblocking (sb_based_dlf = 0): instead of svt_av1_loop_filter_frame at dlf_process.c:122, after
 *     svt_av1_loop_filter_init (and with lf_info derived by svt_av1_loop_filter_frame_init);
 *   - SB-based deblocking (sb_based_dlf = 1, coding_loop.c:2278-2298): once after the picture's last superblock instead
 *     of the per-SB svt_aom_loop_filter_sb call at coding_loop.c:2297;
 * svt_b200_dlf_frame_from_pcs to fill the frame description and the mode-info records, copies the records to the device
 * and calls svt_b200_loop_filter_frame_dev.  The plane pointers it writes are the host recon's; the caller replaces
 * them with the device copies.
 */
#ifndef SVT_B200_DLF_GLUE_H
#define SVT_B200_DLF_GLUE_H

#include "svt_b200.h"

struct PictureControlSet;
struct EbPictureBufferDesc;

/* Fills *frame (planes of `recon` at their visible origin, sizes, bit depth, the frame header's levels and the lf_info
 * tables, which svt_av1_loop_filter_frame_init must already have derived) and, when mi is not NULL, the
 * frame->mi_rows x frame->mi_stride records of pcs->mi_grid_base.  Returns SVT_B200_ERR_BAD_ARG for what the device
 * call does not do: superres or resize, delta_lf_present, a mode-info grid without an entry. */
int svt_b200_dlf_frame_from_pcs(const struct PictureControlSet* pcs, const struct EbPictureBufferDesc* recon, SvtB200DlfFrame* frame,
                                SvtB200DlfMi* mi);

#endif /* SVT_B200_DLF_GLUE_H */
