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

/* For the filter-level search (search_filter_level, deblocking_filter.c:886), with svt_av1_loop_filter_init already run and
 * the frame header's sharpness set, as svt_av1_pick_filter_level does before its first try: fills *frame as
 * svt_b200_dlf_frame_from_pcs does (lfthr at the frame header's sharpness), *s with the source planes the search compares
 * with (ppcs->enhanced_pic, or pcs->input_frame16bit in the 16-bit pipeline) at their visible origin, the SSE region
 * (ppcs->aligned_width x aligned_height), plane_mask and the n_levels levels, and lvl[3][n_levels][8][2][8][2] with
 * the table svt_av1_loop_filter_frame_init derives for each level of each plane in the mask (luma: both directions at the
 * level; zeros for level 0).  Works on copies of the frame header and lf_info: the pcs is not changed.  The caller copies
 * lvl to the device and sets s->d_lvl, and replaces the host plane pointers with the device copies.  Returns
 * SVT_B200_ERR_BAD_ARG for what svt_b200_dlf_frame_from_pcs refuses, a bad level list or mask, or a missing source. */
int svt_b200_dlf_level_sse_from_pcs(const struct PictureControlSet* pcs, const struct EbPictureBufferDesc* recon, int plane_mask,
                                    int n_levels, const uint8_t* levels, SvtB200DlfFrame* frame, SvtB200DlfLevelSse* s,
                                    uint8_t* lvl);

#endif /* SVT_B200_DLF_GLUE_H */
