/* svt_b200_rtcd.h -- the H100 tier's binding into SVT-AV1-PSY's run-time dispatch.
 *
 * A reference build adds integration/svt_b200_rtcd.c to Source/Lib/Globals and calls
 *     svt_b200_install_rtcd(device)
 * right after the two stock rtcd calls of svt_av1_enc_init (Source/Lib/Globals/enc_handle.c:1444-1445) when
 * static_config.use_cpu_flags carries EB_CPU_FLAGS_B200 (INTEGRATION.md).  Every pointer assigned here is declared
 * RTCD_EXTERN in Source/Lib/Codec/aom_dsp_rtcd.h / common_dsp_rtcd.h; the file is compiled against those headers, so a
 * signature mismatch is a compile error, not a cast. */
#ifndef SVT_B200_RTCD_H
#define SVT_B200_RTCD_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
/* the flag a maintainer adds next to EB_CPU_FLAGS_AVX512* (Source/API/EbSvtAv1.h:390-429); bit 40 is unused there */
#define EB_CPU_FLAGS_B200 (1ULL << 40)

/* Binds libsvtav1_b200.so to CUDA device `device` (svt_b200_init) and points the dispatched DSP functions of the hot
 * path at it.  Returns 0, or the svt_b200_init error (the caller maps it to EB_ErrorInsufficientResources); on error
 * no pointer is changed. */
int svt_b200_install_rtcd(int device);
/* number of pointers svt_b200_install_rtcd assigns (for logs / tests) */
int svt_b200_rtcd_count(void);
/* stock svt_aom_setup_rtcd_internal(flags) followed by svt_b200_install_rtcd() when the environment variable
 * SVT_B200_DEVICE is set (its value is the device index): the test build of the reference compiles enc_handle.c with
 * -D'svt_aom_setup_rtcd_internal(f)=svt_b200_setup_rtcd_then_install(f)', i.e. the hook sits exactly at
 * enc_handle.c:1445 without touching the source. */
void svt_b200_setup_rtcd_then_install(uint64_t flags);
#ifdef __cplusplus
}
#endif
#endif
