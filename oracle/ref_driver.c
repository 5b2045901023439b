/* oracle/ref_driver.c -- TEST / BASELINE INFRASTRUCTURE, compiled INTO oracle/_ref/libsvtav1_ref.so.
 *
 * Whole-picture drivers that run the UNMODIFIED reference kernels (through the reference's own
 * dispatch pointers) over the same work lists the H100 T2 entry points take, so that
 *   (1) the T2 paths can be checked against the reference at picture scale, and
 *   (2) bench.py --impl reference / cpu_baseline can time the reference's CPU path (C tier, or the
 *       intrinsics-only AVX2 tier) on all host cores (OpenMP) for the same workload.
 * The driver arithmetic restates the reference's process-level loops (cited per function); every
 * pixel-level computation is done by reference code.  Nothing here is used by the product.
 *
 * Not available in this build of the AVX2 tier (needs NASM): the dav1d inverse transforms -- the
 * inverse-transform leg runs the reference's intrinsics-only AVX2 inverse instead (av1_inv_txfm_avx2.c,
 * highbd_inv_txfm_avx2.c; stated in DESIGN.md / bench output). */
#define _GNU_SOURCE
#include <sched.h>
#include <time.h>
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <unistd.h>
#include "definitions.h"
#include "aom_dsp_rtcd.h"
#include "common_dsp_rtcd.h"
#include "cdef.h"
#include "restoration.h"
#include "convolve.h"
#include "inv_transforms.h"


/* ---- persistent, core-pinned worker pool -------------------------------------------------------------
 * T-1 worker threads are created ONCE (ref_set_threads) and parked on a condition variable; the calling
 * thread takes part in every parallel-for.  Worker t is pinned to the t-th CPU of the process affinity mask.
 * A body invoked from inside a worker (whole frames in flight, ref_frames_run) runs nested loops serially. */
typedef void (*ParBody)(void* ctx, int i);
static struct {
    pthread_mutex_t mu; pthread_cond_t cv_work, cv_done;
    pthread_t th[256]; int n_workers; int quit; unsigned gen; int active;
    ParBody body; void* ctx; int n, chunk; volatile int next; int max_workers;
} g_pool = {PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER, PTHREAD_COND_INITIALIZER};
static int g_threads = 0;
static __thread int t_in_worker = 0;
static __thread int t_worker_id = 0;

static void pool_drain(void) {
    for (;;) {
        const int s = __atomic_fetch_add(&g_pool.next, g_pool.chunk, __ATOMIC_RELAXED);
        if (s >= g_pool.n) break;
        const int e = s + g_pool.chunk < g_pool.n ? s + g_pool.chunk : g_pool.n;
        for (int i = s; i < e; i++) g_pool.body(g_pool.ctx, i);
    }
}
static void* pool_worker(void* arg) {
    const int id = (int)(intptr_t)arg;
    t_in_worker = 1;
    t_worker_id = id;
    unsigned seen = 0;
    pthread_mutex_lock(&g_pool.mu);
    for (;;) {
        while (!g_pool.quit && g_pool.gen == seen) pthread_cond_wait(&g_pool.cv_work, &g_pool.mu);
        if (g_pool.quit) break;
        seen = g_pool.gen;
        const int take = id <= g_pool.max_workers;
        pthread_mutex_unlock(&g_pool.mu);
        if (take) pool_drain();
        pthread_mutex_lock(&g_pool.mu);
        if (--g_pool.active == 0) pthread_cond_signal(&g_pool.cv_done);
    }
    pthread_mutex_unlock(&g_pool.mu);
    return NULL;
}
static void pool_stop(void) {
    if (!g_pool.n_workers) return;
    pthread_mutex_lock(&g_pool.mu);
    g_pool.quit = 1;
    pthread_cond_broadcast(&g_pool.cv_work);
    pthread_mutex_unlock(&g_pool.mu);
    for (int t = 0; t < g_pool.n_workers; t++) pthread_join(g_pool.th[t], NULL);
    g_pool.n_workers = 0;
    g_pool.quit = 0;
}
int ref_set_threads(int n) {
    if (n <= 0) n = (int)sysconf(_SC_NPROCESSORS_ONLN);
    if (n > 256) n = 256;
    if (n < 1) n = 1;
    if (n == g_threads && g_pool.n_workers == n - 1) return n;
    pool_stop();
    g_threads = n;
    cpu_set_t mask;
    int cpus[1024], nc = 0;
    if (sched_getaffinity(0, sizeof(mask), &mask) == 0)
        for (int c = 0; c < CPU_SETSIZE && nc < 1024; c++)
            if (CPU_ISSET(c, &mask)) cpus[nc++] = c;
    for (int t = 0; t < n - 1; t++) {
        pthread_create(&g_pool.th[t], NULL, pool_worker, (void*)(intptr_t)(t + 1));
        if (nc > 1) { /* worker t+1 -> CPU (t+1) mod nc; the caller keeps whatever CPU it has */
            cpu_set_t one;
            CPU_ZERO(&one);
            CPU_SET(cpus[(t + 1) % nc], &one);
            pthread_setaffinity_np(g_pool.th[t], sizeof(one), &one);
        }
    }
    g_pool.n_workers = n - 1;
    return n;
}
int ref_num_threads(void) { return g_threads ? g_threads : ref_set_threads(0); }
static void par_for(int n, int chunk, ParBody body, void* ctx);
void ref_par_for(int n, int chunk, ParBody body, void* ctx) { par_for(n, chunk, body, ctx); } /* for oracle/ref_me_b64.c */
void ref_pool_shutdown(void) { pool_stop(); g_threads = 0; }
static void par_for(int n, int chunk, ParBody body, void* ctx) {
    if (t_in_worker || ref_num_threads() == 1 || n <= chunk) {
        for (int i = 0; i < n; i++) body(ctx, i);
        return;
    }
    pthread_mutex_lock(&g_pool.mu);
    g_pool.body = body; g_pool.ctx = ctx; g_pool.n = n; g_pool.chunk = chunk; g_pool.next = 0;
    g_pool.max_workers = g_pool.n_workers;
    g_pool.active = g_pool.n_workers;
    g_pool.gen++;
    pthread_cond_broadcast(&g_pool.cv_work);
    pthread_mutex_unlock(&g_pool.mu);
    t_in_worker = 1; /* nested par_for calls made by the body on this thread run inline too */
    pool_drain();
    t_in_worker = 0;
    pthread_mutex_lock(&g_pool.mu);
    while (g_pool.active) pthread_cond_wait(&g_pool.cv_done, &g_pool.mu);
    pthread_mutex_unlock(&g_pool.mu);
}

/* ---- tier selection ------------------------------------------------------------------------------ */
int ref_set_tier(int avx2) {
    extern void ref_glue_init(void);
    ref_glue_init(); /* everything = *_c */
    if (!avx2) return 0;
    if (!__builtin_cpu_supports("avx2")) return -1;
    svt_sad_loop_kernel                       = svt_sad_loop_kernel_avx2_intrin;
    svt_ext_all_sad_calculation_8x8_16x16     = svt_ext_all_sad_calculation_8x8_16x16_avx2;
    svt_ext_eight_sad_calculation_32x32_64x64 = svt_ext_eight_sad_calculation_32x32_64x64_avx2;
    svt_ext_sad_calculation_8x8_16x16         = svt_ext_sad_calculation_8x8_16x16_avx2_intrin;
    svt_nxm_sad_kernel                        = svt_nxm_sad_kernel_helper_avx2;
    downsample_2d                             = svt_aom_downsample_2d_avx2;
    svt_av1_fwd_txfm2d_8x8                    = svt_av1_fwd_txfm2d_8x8_avx2;
    svt_av1_fwd_txfm2d_16x16                  = svt_av1_fwd_txfm2d_16x16_avx2;
    svt_av1_fwd_txfm2d_32x32                  = svt_av1_fwd_txfm2d_32x32_avx2;
    svt_av1_fwd_txfm2d_64x64                  = svt_av1_fwd_txfm2d_64x64_avx2;
    svt_av1_quantize_fp                       = svt_av1_quantize_fp_avx2;
    svt_av1_quantize_fp_32x32                 = svt_av1_quantize_fp_32x32_avx2;
    svt_av1_quantize_fp_64x64                 = svt_av1_quantize_fp_64x64_avx2;
    svt_av1_quantize_fp_qm                    = svt_av1_quantize_fp_qm_avx2;
    svt_aom_quantize_b                        = svt_aom_quantize_b_avx2;
    svt_av1_quantize_b_qm                     = svt_av1_quantize_b_qm_avx2;
    svt_cdef_filter_block                     = svt_cdef_filter_block_avx2;
    svt_cdef_filter_block_8xn_16              = svt_cdef_filter_block_8xn_16_avx2; /* called BY the AVX2 filter (common_dsp_rtcd.c:819) */
    svt_aom_cdef_find_dir                     = svt_aom_cdef_find_dir_avx2;
    svt_aom_cdef_find_dir_dual                = svt_aom_cdef_find_dir_dual_avx2;
    svt_compute_cdef_dist_8bit                = svt_aom_compute_cdef_dist_8bit_avx2;
    svt_compute_cdef_dist_16bit               = svt_aom_compute_cdef_dist_16bit_avx2;
    svt_aom_copy_rect8_8bit_to_16bit          = svt_aom_copy_rect8_8bit_to_16bit_avx2;
    svt_av1_compute_stats                     = svt_av1_compute_stats_avx2;
    svt_av1_wiener_convolve_add_src           = svt_av1_wiener_convolve_add_src_avx2;
    svt_residual_kernel8bit                   = svt_residual_kernel8bit_avx2;
    svt_residual_kernel16bit                  = svt_residual_kernel16bit_avx2;
    /* 8-bit inverse transform: the intrinsics-only AVX2 implementation the reference itself binds when the
     * dav1d NASM kernels cannot be used (common_dsp_rtcd.c:522-523) */
    svt_av1_inv_txfm_add                      = svt_av1_inv_txfm_add_avx2;
    /* 4-point and rectangular forward transforms (aom_dsp_rtcd.c:421-439) */
    svt_av1_fwd_txfm2d_4x4   = svt_av1_fwd_txfm2d_4x4_sse4_1;
    svt_av1_fwd_txfm2d_4x8   = svt_av1_fwd_txfm2d_4x8_avx2;
    svt_av1_fwd_txfm2d_4x16  = svt_av1_fwd_txfm2d_4x16_avx2;
    svt_av1_fwd_txfm2d_8x4   = svt_av1_fwd_txfm2d_8x4_avx2;
    svt_av1_fwd_txfm2d_8x16  = svt_av1_fwd_txfm2d_8x16_avx2;
    svt_av1_fwd_txfm2d_8x32  = svt_av1_fwd_txfm2d_8x32_avx2;
    svt_av1_fwd_txfm2d_16x4  = svt_av1_fwd_txfm2d_16x4_avx2;
    svt_av1_fwd_txfm2d_16x8  = svt_av1_fwd_txfm2d_16x8_avx2;
    svt_av1_fwd_txfm2d_16x32 = svt_av1_fwd_txfm2d_16x32_avx2;
    svt_av1_fwd_txfm2d_16x64 = svt_av1_fwd_txfm2d_16x64_avx2;
    svt_av1_fwd_txfm2d_32x8  = svt_av1_fwd_txfm2d_32x8_avx2;
    svt_av1_fwd_txfm2d_32x16 = svt_av1_fwd_txfm2d_32x16_avx2;
    svt_av1_fwd_txfm2d_32x64 = svt_av1_fwd_txfm2d_32x64_avx2;
    svt_av1_fwd_txfm2d_64x16 = svt_av1_fwd_txfm2d_64x16_avx2;
    svt_av1_fwd_txfm2d_64x32 = svt_av1_fwd_txfm2d_64x32_avx2;
    /* high bit depth (10-bit configurations) */
    svt_aom_highbd_quantize_b                 = svt_aom_highbd_quantize_b_avx2;
    svt_av1_highbd_quantize_fp                = svt_av1_highbd_quantize_fp_avx2;
    svt_av1_highbd_quantize_fp_qm             = svt_av1_highbd_quantize_fp_qm_avx2;
    svt_av1_compute_stats_highbd              = svt_av1_compute_stats_highbd_avx2;
    svt_av1_highbd_wiener_convolve_add_src    = svt_av1_highbd_wiener_convolve_add_src_avx2;
    /* 16-bit inverse transforms: the intrinsics (non-dav1d) AVX2 functions of highbd_inv_txfm_avx2.c for the
     * square sizes, the SSE4.1 intrinsics the rtcd table lists for the rest (common_dsp_rtcd.c:501-519) */
    svt_av1_inv_txfm2d_add_4x4   = svt_av1_inv_txfm2d_add_4x4_avx2;
    svt_av1_inv_txfm2d_add_8x8   = svt_av1_inv_txfm2d_add_8x8_avx2;
    svt_av1_inv_txfm2d_add_16x16 = svt_av1_inv_txfm2d_add_16x16_avx2;
    svt_av1_inv_txfm2d_add_32x32 = svt_av1_inv_txfm2d_add_32x32_avx2;
    svt_av1_inv_txfm2d_add_64x64 = svt_av1_inv_txfm2d_add_64x64_avx2;
    svt_av1_inv_txfm2d_add_4x8   = svt_av1_inv_txfm2d_add_4x8_sse4_1;
    svt_av1_inv_txfm2d_add_8x4   = svt_av1_inv_txfm2d_add_8x4_sse4_1;
    svt_av1_inv_txfm2d_add_4x16  = svt_av1_inv_txfm2d_add_4x16_sse4_1;
    svt_av1_inv_txfm2d_add_16x4  = svt_av1_inv_txfm2d_add_16x4_sse4_1;
    svt_av1_inv_txfm2d_add_8x16  = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_16x8  = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_8x32  = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_32x8  = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_16x32 = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_32x16 = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_16x64 = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_64x16 = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_32x64 = svt_av1_highbd_inv_txfm_add_avx2;
    svt_av1_inv_txfm2d_add_64x32 = svt_av1_highbd_inv_txfm_add_avx2;
    return 1;
}

/* ---- open-loop ME for one picture ---------------------------------------------------------------
 * restates hme_level_0/1/2 (motion_estimation.c:820-1113), set_final_seach_centre_sb (:2182-2390),
 * check_00_center (:1139-1210), integer_search_b64 (:1249-1520), open_loop_me_fullpel_search_sblock
 * (:781-817) for the controls the H100 T2 path honours (see DESIGN.md). */
#include "ref_me_b64.h" /* RefMePicture + the complete driver (ref_me_b64.c) */
typedef struct { int32_t hme_l0_sa_w, hme_l0_sa_h, hme_l1_sa_w, hme_l1_sa_h, hme_l2_sa_w, hme_l2_sa_h, me_sa_w, me_sa_h, hme_sub_sad, me_sub_sad, check_zero_centre, reserved; } RefMeParams;

static void hme_clip(int16_t org, int16_t* origin, int16_t* sa, int16_t pad, int16_t pic, int round8) {
    if ((int16_t)(org + *origin) < -pad) {
        *origin = (int16_t)(-pad - org);
        *sa     = (int16_t)(*sa - (-pad - (org + *origin)));
    }
    if ((int16_t)(org + *origin) > (int16_t)(pic - 1)) *origin = (int16_t)(*origin - ((org + *origin) - (pic - 1)));
    if ((int16_t)(org + *origin + *sa) > pic) {
        int16_t v = (int16_t)(*sa - ((org + *origin + *sa) - pic));
        *sa = v > 1 ? v : 1;
    }
    if (round8) *sa = (*sa < 8) ? *sa : (int16_t)(*sa & ~7);
}
static int z16(int y16, int x16) { return 4 * (2 * (y16 >> 1) + (x16 >> 1)) + 2 * (y16 & 1) + (x16 & 1); }

static void fullpel_b64(const uint8_t* src, uint32_t ss, const uint8_t* ref, uint32_t rs, int sa_w, int sa_h, int org_x, int org_y, int sub,
                        uint32_t* best_sad, uint32_t* best_mv) {
    uint32_t e16[16][8], e8[64][8], e32[4][8], s16[16], s8[64], s32[4];
    for (int i = 0; i < 85; i++) { best_sad[i] = 128 * 128 * 255; best_mv[i] = 0; }
    uint32_t *b64 = best_sad, *b32 = best_sad + 1, *b16 = best_sad + 5, *b8 = best_sad + 21;
    uint32_t *m64 = best_mv, *m32 = best_mv + 1, *m16 = best_mv + 5, *m8 = best_mv + 21;
    const int w8 = sa_w - (sa_w & 7);
    for (int y = 0; y < sa_h; y++) {
        for (int x = 0; x < w8; x += 8) {
            const uint32_t mv = ((uint32_t)((org_y + y) & 0xffff) << 16) | (uint32_t)((org_x + x) & 0xffff);
            svt_ext_all_sad_calculation_8x8_16x16((uint8_t*)src, ss, (uint8_t*)ref + (size_t)y * rs + x, rs, mv, b8, b16, m8, m16, e16, e8, sub);
            svt_ext_eight_sad_calculation_32x32_64x64(e16, b32, b64, m32, m64, mv, e32);
        }
        for (int x = w8; x < sa_w; x++) {
            const uint32_t mv = ((uint32_t)((org_y + y) & 0xffff) << 16) | (uint32_t)((org_x + x) & 0xffff);
            for (int blk = 0; blk < 16; blk++) {
                const int y16 = blk >> 2, x16 = blk & 3, i16 = z16(y16, x16);
                svt_ext_sad_calculation_8x8_16x16((uint8_t*)src + 16 * y16 * ss + 16 * x16, ss,
                                                  (uint8_t*)ref + (size_t)(y + 16 * y16) * rs + x + 16 * x16, rs, b8 + 4 * i16, b16 + i16,
                                                  m8 + 4 * i16, m16 + i16, mv, &s16[i16], &s8[4 * i16], sub);
            }
            svt_ext_sad_calculation_32x32_64x64(s16, b32, b64, m32, m64, mv, s32);
        }
    }
}

typedef struct { const RefMePicture* cur; const RefMePicture* refs; const RefMeParams* prm; int n_refs; uint32_t* best_sad; uint32_t* best_mv; int16_t* hme_centre; uint64_t* hme_sad; } MeCtx;
static void ref_me_picture_body(void* vctx, int i) {
    const MeCtx* c = (const MeCtx*)vctx;
    const RefMePicture* cur = c->cur;
    const RefMePicture* refs = c->refs;
    const RefMeParams* prm = c->prm;
    uint32_t* best_sad = c->best_sad;
    uint32_t* best_mv = c->best_mv;
    int16_t* hme_centre = c->hme_centre;
    uint64_t* hme_sad = c->hme_sad;
    const int W = cur->width[2], H = cur->height[2], b64_w = (W + 63) >> 6, b64_h = (H + 63) >> 6, nb = b64_w * b64_h;
    {
        const int r = i / nb, b = i % nb, bx = b % b64_w, by = b / b64_w;
        const RefMePicture* rp = &refs[r];
        const RefMeParams*  p  = &prm[r];
        const int sub = p->hme_sub_sad ? 1 : 0;
        int16_t  px[4] = {0, 0, 0, 0}, py[4] = {0, 0, 0, 0};
        uint64_t ls[4] = {0, 0, 0, 0};
        for (int level = 0; level < 3; level++) {
            const int sh = 2 - level;
            const int16_t org_x = (int16_t)((bx * 64) >> sh), org_y = (int16_t)((by * 64) >> sh);
            const int blk_w = (W - bx * 64 < 64 ? W - bx * 64 : 64) >> sh, blk_h = (H - by * 64 < 64 ? H - by * 64 : 64) >> sh;
            int16_t nx[4], ny[4];
            for (int reg = 0; reg < 4; reg++) {
                const int sr_w = reg & 1, sr_h = reg >> 1;
                int16_t sa_w, sa_h, ox, oy, pw, ph;
                if (level == 0) {
                    sa_w = (int16_t)((p->hme_l0_sa_w + 7) & ~7); sa_h = (int16_t)p->hme_l0_sa_h;
                    ox = (int16_t)(-(int16_t)((sa_w * 2) >> 1) + sa_w * sr_w); oy = (int16_t)(-(int16_t)((sa_h * 2) >> 1) + sa_h * sr_h);
                    pw = (int16_t)(rp->org_x[0] - 1); ph = (int16_t)(rp->org_y[0] - 1);
                } else if (level == 1) {
                    sa_w = (int16_t)((p->hme_l1_sa_w + 7) & ~7); sa_h = (int16_t)p->hme_l1_sa_h;
                    ox = (int16_t)(-(sa_w >> 1) + (px[reg] >> 1)); oy = (int16_t)(-(sa_h >> 1) + (py[reg] >> 1));
                    pw = (int16_t)(rp->org_x[1] - 1); ph = (int16_t)(rp->org_y[1] - 1);
                } else {
                    sa_w = (int16_t)((p->hme_l2_sa_w + 7) & ~7); sa_h = (int16_t)p->hme_l2_sa_h;
                    ox = (int16_t)(-(sa_w >> 1) + px[reg]); oy = (int16_t)(-(sa_h >> 1) + py[reg]);
                    pw = ph = 63;
                }
                hme_clip(org_x, &ox, &sa_w, pw, (int16_t)rp->width[level], 1);
                hme_clip(org_y, &oy, &sa_h, ph, (int16_t)rp->height[level], 0);
                const uint8_t* s = cur->plane[level] + (size_t)(cur->org_y[level] + org_y) * cur->stride[level] + cur->org_x[level] + org_x;
                const uint8_t* q = rp->plane[level] + (size_t)(rp->org_y[level] + org_y + oy) * rp->stride[level] + rp->org_x[level] + org_x + ox;
                uint64_t bs = 0;
                int16_t  x = 0, y = 0;
                svt_sad_loop_kernel((uint8_t*)s, (uint32_t)(cur->stride[level] << sub), (uint8_t*)q, (uint32_t)(rp->stride[level] << sub),
                                    (uint32_t)(blk_h >> sub), (uint32_t)blk_w, &bs, &x, &y, (uint32_t)rp->stride[level], 0, sa_w, sa_h);
                if (sub) bs *= 2;
                const int mul = level == 0 ? 4 : (level == 1 ? 2 : 1);
                nx[reg] = (int16_t)((int16_t)(x + ox) * mul);
                ny[reg] = (int16_t)((int16_t)(y + oy) * mul);
                ls[reg] = bs;
            }
            memcpy(px, nx, sizeof(px));
            memcpy(py, ny, sizeof(py));
        }
        int16_t  cx = px[0], cy = py[0];
        uint64_t cs = ls[0];
        for (int reg = 1; reg < 4; reg++)
            if (ls[reg] < cs) { cs = ls[reg]; cx = px[reg]; cy = py[reg]; }
        hme_centre[2 * i] = cx;
        hme_centre[2 * i + 1] = cy;
        hme_sad[i] = cs;
        const int16_t org_x = (int16_t)(bx * 64), org_y = (int16_t)(by * 64);
        const int blk_w = W - org_x < 64 ? W - org_x : 64, blk_h = H - org_y < 64 ? H - org_y : 64;
        const uint8_t* src = cur->plane[2] + (size_t)(cur->org_y[2] + org_y) * cur->stride[2] + cur->org_x[2] + org_x;
        int16_t sx = cx, sy = cy;
        if (p->check_zero_centre && (sx || sy)) {
            const int16_t RW = (int16_t)rp->width[2], RH = (int16_t)rp->height[2];
            if ((int16_t)(org_x + sx) < -63) sx = (int16_t)(-63 - org_x);
            if ((int16_t)(org_x + sx) > RW - 1) sx = (int16_t)(sx - ((org_x + sx) - (RW - 1)));
            if ((int16_t)(org_y + sy) < -63) sy = (int16_t)(-63 - org_y);
            if ((int16_t)(org_y + sy) > RH - 1) sy = (int16_t)(sy - ((org_y + sy) - (RH - 1)));
            const uint8_t* r0 = rp->plane[2] + (size_t)(rp->org_y[2] + org_y) * rp->stride[2] + rp->org_x[2] + org_x;
            uint32_t z  = svt_nxm_sad_kernel(src, (uint32_t)cur->stride[2] << 1, r0, (uint32_t)rp->stride[2] << 1, (uint32_t)blk_h >> 1, (uint32_t)blk_w) << 1;
            uint32_t hs = svt_nxm_sad_kernel(src, (uint32_t)cur->stride[2] << 1, r0 + (ptrdiff_t)sy * rp->stride[2] + sx, (uint32_t)rp->stride[2] << 1,
                                             (uint32_t)blk_h >> 1, (uint32_t)blk_w) << 1;
            if (z <= hs) sx = sy = 0;
        }
        int16_t sa_w = (int16_t)(((p->me_sa_w > 1 ? p->me_sa_w : 1) + 7) & ~7), sa_h = (int16_t)(p->me_sa_h > 3 ? p->me_sa_h : 3);
        int16_t ox = (int16_t)(sx - (sa_w >> 1)), oy = (int16_t)(sy - (sa_h >> 1));
        if ((int16_t)(org_x + ox) < -63) ox = (int16_t)(-63 - org_x);
        if ((int16_t)(org_x + ox) > W - 1) ox = (int16_t)(ox - ((org_x + ox) - (W - 1)));
        if ((int16_t)(org_x + ox + sa_w) > W) { int v = sa_w - ((org_x + ox + sa_w) - W); sa_w = (int16_t)(v > 1 ? v : 1); }
        sa_w = sa_w < 8 ? sa_w : (int16_t)(sa_w & ~7);
        if ((int16_t)(org_y + oy) < -63) oy = (int16_t)(-63 - org_y);
        if ((int16_t)(org_y + oy) > H - 1) oy = (int16_t)(oy - ((org_y + oy) - (H - 1)));
        if ((int16_t)(org_y + oy + sa_h) > H) { int v = sa_h - ((org_y + oy + sa_h) - H); sa_h = (int16_t)(v > 1 ? v : 1); }
        const uint8_t* q = rp->plane[2] + (ptrdiff_t)(rp->org_y[2] + org_y + oy) * rp->stride[2] + rp->org_x[2] + org_x + ox;
        fullpel_b64(src, (uint32_t)cur->stride[2], q, (uint32_t)rp->stride[2], sa_w, sa_h, ox, oy, p->me_sub_sad ? 1 : 0, best_sad + (size_t)i * 85,
                    best_mv + (size_t)i * 85);
        }
}
void ref_me_picture(const RefMePicture* cur, const RefMePicture* refs, const RefMeParams* prm, int n_refs, uint32_t* best_sad,
                    uint32_t* best_mv, int16_t* hme_centre, uint64_t* hme_sad) {
    MeCtx c = {cur, refs, prm, n_refs, best_sad, best_mv, hme_centre, hme_sad};
    const int W = cur->width[2], H = cur->height[2], b64_w = (W + 63) >> 6, b64_h = (H + 63) >> 6, nb = b64_w * b64_h;
    par_for(n_refs * nb, 4, ref_me_picture_body, &c);
}


/* ---- transform / quantize / inverse over a block list ---------------------------------------------
 * the trio of svt_aom_estimate_transform -> svt_aom_quantize_inv_quantize -> inverse (SURVEY 3.4),
 * one call per block; 8-bit or 10-bit pixels (the reference's CONVERT_TO_BYTEPTR disguise for 16-bit
 * planes, full_loop.c:1843-1846), "fp" quantizer with quantisation matrices (PSY default). */
typedef struct { uint64_t src_off, dst_off; uint32_t src_stride; uint8_t tx_size, tx_type; uint16_t reserved; } RefFwdItem;
typedef struct { uint64_t coef_off, pred_off, recon_off; uint32_t pred_stride, recon_stride; uint8_t tx_size, tx_type, bd, reserved; uint32_t reserved2; } RefInvItem;
typedef struct {
    uint64_t coeff_off, q_off, dq_off; uint32_t scan_off, qm_off, iqm_off, n_coeffs;
    int16_t zbin[2], round[2], quant[2], quant_shift[2], dequant[2]; uint8_t mode, log_scale; uint16_t reserved;
} RefQuantItem;
static const int TXW[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
static const int TXH[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};

static void fwd_one(int16_t* in, int32_t* out, uint32_t stride, int ty, int sz, int bd) {
    switch (sz) {
    case 0: svt_av1_fwd_txfm2d_4x4(in, out, stride, ty, bd); break;
    case 1: svt_av1_fwd_txfm2d_8x8(in, out, stride, ty, bd); break;
    case 2: svt_av1_fwd_txfm2d_16x16(in, out, stride, ty, bd); break;
    case 3: svt_av1_fwd_txfm2d_32x32(in, out, stride, ty, bd); break;
    case 4: svt_av1_fwd_txfm2d_64x64(in, out, stride, ty, bd); break;
    case 5: svt_av1_fwd_txfm2d_4x8(in, out, stride, ty, bd); break;
    case 6: svt_av1_fwd_txfm2d_8x4(in, out, stride, ty, bd); break;
    case 7: svt_av1_fwd_txfm2d_8x16(in, out, stride, ty, bd); break;
    case 8: svt_av1_fwd_txfm2d_16x8(in, out, stride, ty, bd); break;
    case 9: svt_av1_fwd_txfm2d_16x32(in, out, stride, ty, bd); break;
    case 10: svt_av1_fwd_txfm2d_32x16(in, out, stride, ty, bd); break;
    case 11: svt_av1_fwd_txfm2d_32x64(in, out, stride, ty, bd); break;
    case 12: svt_av1_fwd_txfm2d_64x32(in, out, stride, ty, bd); break;
    case 13: svt_av1_fwd_txfm2d_4x16(in, out, stride, ty, bd); break;
    case 14: svt_av1_fwd_txfm2d_16x4(in, out, stride, ty, bd); break;
    case 15: svt_av1_fwd_txfm2d_8x32(in, out, stride, ty, bd); break;
    case 16: svt_av1_fwd_txfm2d_32x8(in, out, stride, ty, bd); break;
    case 17: svt_av1_fwd_txfm2d_16x64(in, out, stride, ty, bd); break;
    default: svt_av1_fwd_txfm2d_64x16(in, out, stride, ty, bd); break;
    }
}

typedef struct {
    const int16_t* residual; int32_t *coeff, *q, *dq; const int16_t *scan, *iscan; const uint8_t* qm;
    const RefFwdItem* fwd; const RefQuantItem* qi; const RefInvItem* inv; uint16_t* eobs;
    const void* pred; void* recon; int bd;
    const void* srcpix; int16_t* residual_w; int skip_zero_blocks;
} TxCtx;

/* svt_aom_residual_kernel (coding_loop.c:69, called per transform block at :393,:471,:518): residual = source - prediction */
static void residual_body(void* vctx, int i) {
    const TxCtx* c = (const TxCtx*)vctx;
    const RefFwdItem* it = &c->fwd[i];
    const RefInvItem* iv = &c->inv[i];
    const int W = TXW[it->tx_size], H = TXH[it->tx_size];
    if (c->bd == 8)
        svt_residual_kernel8bit((uint8_t*)c->srcpix + it->src_off, it->src_stride, (uint8_t*)c->pred + iv->pred_off, iv->pred_stride,
                                c->residual_w + it->src_off, it->src_stride, (uint32_t)W, (uint32_t)H);
    else
        svt_residual_kernel16bit((uint16_t*)c->srcpix + it->src_off, it->src_stride, (uint16_t*)c->pred + iv->pred_off, iv->pred_stride,
                                 c->residual_w + it->src_off, it->src_stride, (uint32_t)W, (uint32_t)H);
}

static void fwd_body(void* vctx, int i) {
    const TxCtx* c = (const TxCtx*)vctx;
    const RefFwdItem* it = &c->fwd[i];
    const int W = TXW[it->tx_size], H = TXH[it->tx_size];
    if ((it->reserved & 1) && (W > 32 || H > 32)) {
        /* packed output: the re-pack half of svt_handle_transform64x64 & co (transforms.c:2374-2542) */
        DECLARE_ALIGNED(64, int32_t, tmp[64 * 64]);
        const int Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;
        fwd_one((int16_t*)c->residual + it->src_off, tmp, it->src_stride, it->tx_type, it->tx_size, c->bd);
        for (int r = 0; r < Hp; r++) memcpy(c->coeff + it->dst_off + (size_t)r * Wp, tmp + (size_t)r * W, (size_t)Wp * sizeof(int32_t));
        return;
    }
    fwd_one((int16_t*)c->residual + it->src_off, c->coeff + it->dst_off, it->src_stride, it->tx_type, it->tx_size, c->bd);
}
void ref_fwd_txfm_batch_bd(const int16_t* residual, int32_t* coeff, const RefFwdItem* items, int n, int bd) {
    TxCtx c;
    memset(&c, 0, sizeof(c));
    c.residual = residual; c.coeff = coeff; c.fwd = items; c.bd = bd;
    par_for(n, 64, fwd_body, &c);
}
void ref_fwd_txfm_batch(const int16_t* residual, int32_t* coeff, const RefFwdItem* items, int n) { ref_fwd_txfm_batch_bd(residual, coeff, items, n, 8); }

static void quant_body(void* vctx, int i) {
    const TxCtx* c = (const TxCtx*)vctx;
    const int32_t* coeff = c->coeff;
    int32_t *q = c->q, *dq = c->dq;
    uint16_t* eobs = c->eobs;
    const RefQuantItem* it = &c->qi[i];
    const uint8_t* wm = it->qm_off == 0xffffffffu ? NULL : c->qm + it->qm_off;
    const uint8_t* im = it->iqm_off == 0xffffffffu ? NULL : c->qm + it->iqm_off;
    const int16_t* sc = c->scan + it->scan_off;
    const int16_t* isc = c->iscan + it->scan_off; /* the SIMD tiers derive eob from the inverse scan */
    /* MacroblockPlane tables are int16[8] = {DC, AC x 7}; the SIMD tiers load all eight lanes */
    DECLARE_ALIGNED(16, int16_t, zbin[8]);
    DECLARE_ALIGNED(16, int16_t, round[8]);
    DECLARE_ALIGNED(16, int16_t, quant[8]);
    DECLARE_ALIGNED(16, int16_t, quant_shift[8]);
    DECLARE_ALIGNED(16, int16_t, dequant[8]);
    for (int k = 0; k < 8; k++) {
        zbin[k] = it->zbin[k != 0]; round[k] = it->round[k != 0]; quant[k] = it->quant[k != 0];
        quant_shift[k] = it->quant_shift[k != 0]; dequant[k] = it->dequant[k != 0];
    }
    if (it->mode == 2) { /* SVT_B200_QUANT_FP_LBD */
        if (wm || im)
            svt_av1_quantize_fp_qm(coeff + it->coeff_off, it->n_coeffs, zbin, round, quant, quant_shift, q + it->q_off,
                                   dq + it->dq_off, dequant, &eobs[i], sc, isc, wm, im, it->log_scale);
        else if (it->log_scale == 0)
            svt_av1_quantize_fp(coeff + it->coeff_off, it->n_coeffs, zbin, round, quant, quant_shift, q + it->q_off,
                                dq + it->dq_off, dequant, &eobs[i], sc, isc);
        else if (it->log_scale == 1)
            svt_av1_quantize_fp_32x32(coeff + it->coeff_off, it->n_coeffs, zbin, round, quant, quant_shift, q + it->q_off,
                                      dq + it->dq_off, dequant, &eobs[i], sc, isc);
        else
            svt_av1_quantize_fp_64x64(coeff + it->coeff_off, it->n_coeffs, zbin, round, quant, quant_shift, q + it->q_off,
                                      dq + it->dq_off, dequant, &eobs[i], sc, isc);
    } else if (it->mode == 0)
        svt_aom_quantize_b(coeff + it->coeff_off, it->n_coeffs, zbin, round, quant, quant_shift, q + it->q_off, dq + it->dq_off,
                           dequant, &eobs[i], sc, isc, wm, im, it->log_scale);
    else if (it->mode == 1)
        svt_aom_highbd_quantize_b(coeff + it->coeff_off, it->n_coeffs, zbin, round, quant, quant_shift, q + it->q_off,
                                  dq + it->dq_off, dequant, &eobs[i], sc, isc, wm, im, it->log_scale);
    else if (wm || im)
        svt_av1_highbd_quantize_fp_qm(coeff + it->coeff_off, it->n_coeffs, zbin, round, quant, quant_shift, q + it->q_off,
                                      dq + it->dq_off, dequant, &eobs[i], sc, isc, wm, im, it->log_scale);
    else
        svt_av1_highbd_quantize_fp(coeff + it->coeff_off, it->n_coeffs, zbin, round, quant, quant_shift, q + it->q_off,
                                   dq + it->dq_off, dequant, &eobs[i], sc, isc, it->log_scale);
}
void ref_quant_batch(const int32_t* coeff, int32_t* q, int32_t* dq, const int16_t* scan, const int16_t* iscan, const uint8_t* qm,
                     const RefQuantItem* items, int n, uint16_t* eobs) {
    TxCtx c;
    memset(&c, 0, sizeof(c));
    c.coeff = (int32_t*)coeff; c.q = q; c.dq = dq; c.scan = scan; c.iscan = iscan; c.qm = qm; c.qi = items; c.eobs = eobs;
    par_for(n, 64, quant_body, &c);
}

/* svt_aom_inv_transform_recon8bit / svt_aom_inv_transform_recon (inv_transforms.c:3087,3148): the reference's own
 * wrappers; read and write planes differ, so they pass the maximum eob themselves */
static void inv_body(void* vctx, int i) {
    const TxCtx* c = (const TxCtx*)vctx;
    const RefInvItem* it = &c->inv[i];
    if (c->skip_zero_blocks && c->eobs[i] == 0) {
        /* no coefficient survived: the encode pass does not run the inverse (coding_loop.c:601,632,655), the
         * reconstruction is the prediction */
        const int W = TXW[it->tx_size], H = TXH[it->tx_size], psz = c->bd > 8 ? 2 : 1;
        for (int r = 0; r < H; r++)
            memcpy((uint8_t*)c->recon + (it->recon_off + (size_t)r * it->recon_stride) * psz,
                   (const uint8_t*)c->pred + (it->pred_off + (size_t)r * it->pred_stride) * psz, (size_t)W * psz);
        return;
    }
    if (c->bd == 8)
        svt_aom_inv_transform_recon8bit((int32_t*)c->dq + it->coef_off, (uint8_t*)c->pred + it->pred_off, it->pred_stride,
                                        (uint8_t*)c->recon + it->recon_off, it->recon_stride, (TxSize)it->tx_size, (TxType)it->tx_type,
                                        PLANE_TYPE_Y, 0, 0);
    else
        svt_aom_inv_transform_recon((int32_t*)c->dq + it->coef_off, CONVERT_TO_BYTEPTR((uint16_t*)c->pred + it->pred_off), it->pred_stride,
                                    CONVERT_TO_BYTEPTR((uint16_t*)c->recon + it->recon_off), it->recon_stride, (TxSize)it->tx_size,
                                    (uint32_t)c->bd, (TxType)it->tx_type, PLANE_TYPE_Y, 0, 0);
}
void ref_inv_txfm_batch_bd(const int32_t* coeff, const void* pred, void* recon, const RefInvItem* items, int n, int bd) {
    TxCtx c;
    memset(&c, 0, sizeof(c));
    c.dq = (int32_t*)coeff; c.pred = pred; c.recon = recon; c.inv = items; c.bd = bd;
    par_for(n, 64, inv_body, &c);
}
void ref_inv_txfm_batch_8bit(const int32_t* coeff, const uint8_t* pred, uint8_t* recon, const RefInvItem* items, int n) {
    ref_inv_txfm_batch_bd(coeff, pred, recon, items, n, 8);
}

/* ---- CDEF picture search / apply (cdef_seg_search, cdef_process.c:106-352; svt_av1_cdef_frame) ----- */
typedef struct {
    const void *recon_y, *recon_cb, *recon_cr, *src_y, *src_cb, *src_cr;
    int32_t recon_stride_y, recon_stride_c, src_stride_y, src_stride_c, width, height, bit_depth, damping, subsampling_factor, reserved;
} RefCdefFrame;

static void cdef_tile(uint16_t* inbuf, const void* plane, int stride, int fbr, int fbc, int nvfb, int nhfb, int fbs, int vsz, int hsz, int is16) {
    uint16_t* in = inbuf + CDEF_VBORDER * CDEF_BSTRIDE + CDEF_HBORDER;
    for (int i = 0; i < CDEF_BSTRIDE * (64 + 2 * CDEF_VBORDER); i++) inbuf[i] = CDEF_VERY_LARGE;
    const int yoff = CDEF_VBORDER * (fbr != 0), xoff = CDEF_HBORDER * (fbc != 0);
    const int ysize = vsz + CDEF_VBORDER * (fbr + 1 < nvfb) + yoff, xsize = hsz + CDEF_HBORDER * (fbc + 1 < nhfb) + xoff;
    svt_aom_copy_sb8_16(&in[-yoff * CDEF_BSTRIDE - xoff], CDEF_BSTRIDE, (const uint8_t*)plane, fbr * fbs - yoff, fbc * fbs - xoff, stride, ysize, xsize,
                        is16 ? true : false);
}
static int cdef_list(const RefCdefFrame* f, const uint8_t* skip8x8, int fbr, int fbc, CdefList* dlist) {
    const int w8 = (f->width + 7) >> 3, h8 = (f->height + 7) >> 3;
    int cnt = 0;
    for (int by = 0; by < 8; by++)
        for (int bx = 0; bx < 8; bx++) {
            const int gy = fbr * 8 + by, gx = fbc * 8 + bx;
            if (gy < h8 && gx < w8 && !skip8x8[gy * w8 + gx]) { dlist[cnt].by = (uint8_t)by; dlist[cnt].bx = (uint8_t)bx; cnt++; }
        }
    return cnt;
}

typedef struct { const RefCdefFrame* f; const uint8_t* skip; const int *sy, *su; int ng; uint64_t* mse; uint8_t* dir; int32_t* var; } CdefSearchCtx;
static void cdef_search_body(void* vctx, int fb) {
    const CdefSearchCtx* c = (const CdefSearchCtx*)vctx;
    const RefCdefFrame* f = c->f;
    const int ng = c->ng;
    uint64_t* mse = c->mse;
    const int is16 = f->bit_depth > 8, coeff_shift = f->bit_depth - 8, psz = is16 ? 2 : 1;
    const int nhfb = (f->width + 63) >> 6, nvfb = (f->height + 63) >> 6, nfb = nhfb * nvfb;
    const int fbr = fb / nhfb, fbc = fb % nhfb;
    CdefList dlist[64];
    const int cnt = cdef_list(f, c->skip, fbr, fbc, dlist);
    if (!cnt) {
        for (int g = 0; g < ng; g++) mse[(size_t)fb * ng + g] = mse[(size_t)(nfb + fb) * ng + g] = 0;
        return;
    }
    DECLARE_ALIGNED(32, uint16_t, inbuf[CDEF_INBUF_SIZE]);
    DECLARE_ALIGNED(32, uint16_t, tmp_dst[1 << (MAX_SB_SIZE_LOG2 * 2)]);
    uint8_t dir[CDEF_NBLOCKS][CDEF_NBLOCKS];
    int32_t var[CDEF_NBLOCKS][CDEF_NBLOCKS];
    int32_t dirinit = 0;
    for (int pli = 0; pli < 3; pli++) {
        const int dec = pli ? 1 : 0, fbs = 64 >> dec, pw = f->width >> dec, ph = f->height >> dec;
        const uint8_t* rec = (const uint8_t*)(pli == 0 ? f->recon_y : (pli == 1 ? f->recon_cb : f->recon_cr));
        const uint8_t* src = (const uint8_t*)(pli == 0 ? f->src_y : (pli == 1 ? f->src_cb : f->src_cr));
        const int rs = pli ? f->recon_stride_c : f->recon_stride_y, ss = pli ? f->src_stride_c : f->src_stride_y;
        const int hsz = fbs < pw - fbc * fbs ? fbs : pw - fbc * fbs, vsz = fbs < ph - fbr * fbs ? fbs : ph - fbr * fbs;
        cdef_tile(inbuf, rec, rs, fbr, fbc, nvfb, nhfb, fbs, vsz, hsz, is16);
        uint16_t* in = inbuf + CDEF_VBORDER * CDEF_BSTRIDE + CDEF_HBORDER;
        int subs = f->subsampling_factor;
        if (subs > (dec ? 1 : 4)) subs = dec ? 1 : 4;
        for (int g = 0; g < ng; g++) {
            uint64_t* m = &mse[(size_t)((pli ? 1 : 0) * nfb + fb) * ng + g];
            const int sv = pli ? c->su[g] : c->sy[g];
            if (sv < 0) { *m = (uint64_t)1040400 * 64; continue; }
            const int pri = sv / CDEF_SEC_STRENGTHS, sec = sv % CDEF_SEC_STRENGTHS;
            svt_cdef_filter_fb(is16 ? NULL : (uint8_t*)tmp_dst, is16 ? tmp_dst : NULL, 0, in, dec, dec, dir, &dirinit, var, pli, dlist, cnt, pri,
                               sec + (sec == 3), f->damping, f->damping, coeff_shift, (uint8_t)subs);
            const uint8_t* sp = src + ((size_t)(fbr * fbs) * ss + fbc * fbs) * psz;
            const uint64_t d = is16 ? svt_compute_cdef_dist_16bit((const uint16_t*)sp, ss, tmp_dst, dlist, cnt, dec ? BLOCK_4X4 : BLOCK_8X8, coeff_shift,
                                                                  pli, (uint8_t)subs)
                                    : svt_compute_cdef_dist_8bit(sp, ss, (uint8_t*)tmp_dst, dlist, cnt, dec ? BLOCK_4X4 : BLOCK_8X8, coeff_shift, pli,
                                                                 (uint8_t)subs);
            if (pli == 2) *m += d * subs;
            else *m = d * subs;
        }
    }
    for (int k = 0; k < cnt; k++) {
        c->dir[(size_t)fb * 64 + dlist[k].by * 8 + dlist[k].bx] = dir[dlist[k].by][dlist[k].bx];
        c->var[(size_t)fb * 64 + dlist[k].by * 8 + dlist[k].bx] = var[dlist[k].by][dlist[k].bx];
    }
}
void ref_cdef_search_frame(const RefCdefFrame* f, const uint8_t* skip8x8, const int* str_y, const int* str_uv, int ng, uint64_t* mse, uint8_t* dir_out,
                           int32_t* var_out) {
    CdefSearchCtx c = {f, skip8x8, str_y, str_uv, ng, mse, dir_out, var_out};
    par_for(((f->width + 63) >> 6) * ((f->height + 63) >> 6), 2, cdef_search_body, &c);
}

typedef struct { const RefCdefFrame* f; const uint8_t* skip; const int8_t* idx; const int *ys, *us; void *oy, *ocb, *ocr; int os_y, os_c; } CdefApplyCtx;
static void cdef_apply_body(void* vctx, int fb) {
    const CdefApplyCtx* c = (const CdefApplyCtx*)vctx;
    const RefCdefFrame* f = c->f;
    const int is16 = f->bit_depth > 8, coeff_shift = f->bit_depth - 8;
    const int nhfb = (f->width + 63) >> 6, nvfb = (f->height + 63) >> 6;
    const int fbr = fb / nhfb, fbc = fb % nhfb;
    if (c->idx[fb] < 0) return;
    const int ys = c->ys[c->idx[fb]], us = c->us[c->idx[fb]];
    if (!ys && !us) return;
    CdefList dlist[64];
    const int cnt = cdef_list(f, c->skip, fbr, fbc, dlist);
    if (!cnt) return;
    DECLARE_ALIGNED(32, uint16_t, inbuf[CDEF_INBUF_SIZE]);
    uint8_t dir[CDEF_NBLOCKS][CDEF_NBLOCKS];
    int32_t var[CDEF_NBLOCKS][CDEF_NBLOCKS];
    int32_t dirinit = 0;
    for (int pli = 0; pli < 3; pli++) {
        const int dec = pli ? 1 : 0, fbs = 64 >> dec, pw = f->width >> dec, ph = f->height >> dec;
        const uint8_t* rec = (const uint8_t*)(pli == 0 ? f->recon_y : (pli == 1 ? f->recon_cb : f->recon_cr));
        void* out = pli == 0 ? c->oy : (pli == 1 ? c->ocb : c->ocr);
        const int rs = pli ? f->recon_stride_c : f->recon_stride_y, os = pli ? c->os_c : c->os_y;
        const int hsz = fbs < pw - fbc * fbs ? fbs : pw - fbc * fbs, vsz = fbs < ph - fbr * fbs ? fbs : ph - fbr * fbs;
        cdef_tile(inbuf, rec, rs, fbr, fbc, nvfb, nhfb, fbs, vsz, hsz, is16);
        uint16_t* in = inbuf + CDEF_VBORDER * CDEF_BSTRIDE + CDEF_HBORDER;
        const int sv = pli ? us : ys, pri = sv / CDEF_SEC_STRENGTHS, sec = sv % CDEF_SEC_STRENGTHS;
        const size_t o = (size_t)(fbr * fbs) * os + fbc * fbs;
        if (pli == 0 || pri || sec)
            svt_cdef_filter_fb(is16 ? NULL : (uint8_t*)out + o, is16 ? (uint16_t*)out + o : NULL, os, in, dec, dec, dir, &dirinit, var, pli, dlist, cnt,
                               pri, sec + (sec == 3), f->damping, f->damping, coeff_shift, 1);
    }
}
void ref_cdef_apply_frame(const RefCdefFrame* f, const uint8_t* skip8x8, const int8_t* fb_idx, const int* y_str, const int* uv_str, void* out_y,
                          void* out_cb, void* out_cr, int os_y, int os_c) {
    CdefApplyCtx c = {f, skip8x8, fb_idx, y_str, uv_str, out_y, out_cb, out_cr, os_y, os_c};
    par_for(((f->width + 63) >> 6) * ((f->height + 63) >> 6), 2, cdef_apply_body, &c);
}

/* ---- Wiener statistics / filter over unit lists ------------------------------------------------------ */
typedef struct { uint64_t dgd_off, src_off; int32_t dgd_stride, src_stride, h_start, h_end, v_start, v_end, wiener_win, reserved; } RefStatsItem;
typedef struct { uint64_t src_off, dst_off; int32_t src_stride, dst_stride; uint16_t w, h; uint32_t reserved; int16_t hfilter[8], vfilter[8]; } RefWienerUnit;

typedef struct { const void *dgd, *src; const RefStatsItem* items; int64_t *M, *H; int bd; } StatsCtx;
static void stats_body(void* vctx, int i) {
    const StatsCtx* c = (const StatsCtx*)vctx;
    DECLARE_ALIGNED(64, int64_t, m[WIENER_WIN2 + 7]);
    DECLARE_ALIGNED(64, int64_t, h[WIENER_WIN2 * WIENER_WIN2 + 7]);
    const RefStatsItem* it = &c->items[i];
    if (c->bd == 8)
        svt_av1_compute_stats(it->wiener_win, (const uint8_t*)c->dgd + it->dgd_off, (const uint8_t*)c->src + it->src_off, it->h_start, it->h_end,
                              it->v_start, it->v_end, it->dgd_stride, it->src_stride, m, h);
    else /* restoration_pick.c:1305-1318: 16-bit planes travel as CONVERT_TO_BYTEPTR disguises */
        svt_av1_compute_stats_highbd(it->wiener_win, CONVERT_TO_BYTEPTR((const uint16_t*)c->dgd + it->dgd_off),
                                     CONVERT_TO_BYTEPTR((const uint16_t*)c->src + it->src_off), it->h_start, it->h_end, it->v_start, it->v_end,
                                     it->dgd_stride, it->src_stride, m, h, (EbBitDepth)c->bd);
    const int w2 = it->wiener_win * it->wiener_win;
    memcpy(c->M + (size_t)i * 49, m, sizeof(int64_t) * w2);
    memcpy(c->H + (size_t)i * 2401, h, sizeof(int64_t) * w2 * w2);
}
void ref_compute_stats_batch_bd(const void* dgd, const void* src, const RefStatsItem* items, int n, int64_t* M, int64_t* H, int bd) {
    StatsCtx c = {dgd, src, items, M, H, bd};
    par_for(n, 1, stats_body, &c);
}
void ref_compute_stats_batch(const uint8_t* dgd, const uint8_t* src, const RefStatsItem* items, int n, int64_t* M, int64_t* H) {
    ref_compute_stats_batch_bd(dgd, src, items, n, M, H, 8);
}

typedef struct { const void* src; void* dst; const RefWienerUnit* units; int bd; } WienerCtx;
static void wiener_body(void* vctx, int i) {
    const WienerCtx* c = (const WienerCtx*)vctx;
    const RefWienerUnit* u = &c->units[i];
    /* the reference derives the kernel base by masking the low address bits (convolve.c:48-56) */
    DECLARE_ALIGNED(256, int16_t, fx[128]);
    DECLARE_ALIGNED(256, int16_t, fy[128]);
    memcpy(fx, u->hfilter, 16);
    memcpy(fy, u->vfilter, 16);
    const ConvolveParams cp = get_conv_params_wiener(c->bd);
    if (c->bd == 8)
        svt_av1_wiener_convolve_add_src((const uint8_t*)c->src + u->src_off, u->src_stride, (uint8_t*)c->dst + u->dst_off, u->dst_stride, fx, fy, u->w,
                                        u->h, &cp);
    else /* svt_aom_wiener_filter_stripe_highbd, restoration.c */
        svt_av1_highbd_wiener_convolve_add_src(CONVERT_TO_BYTEPTR((const uint16_t*)c->src + u->src_off), u->src_stride,
                                               CONVERT_TO_BYTEPTR((uint16_t*)c->dst + u->dst_off), u->dst_stride, fx, fy, u->w, u->h, &cp, c->bd);
}
void ref_wiener_units_bd(const void* src, void* dst, const RefWienerUnit* units, int n, int bd) {
    WienerCtx c = {src, dst, units, bd};
    par_for(n, 16, wiener_body, &c);
}
void ref_wiener_units_8bit(const uint8_t* src, uint8_t* dst, const RefWienerUnit* units, int n) { ref_wiener_units_bd(src, dst, units, n, 8); }

/* ---- whole frames --------------------------------------------------------------------------------------
 * One RefFrameJob = every buffer and work list of one frame of hot-path work (bench.py / FrameWorkload).
 * ref_frame_step runs the frame's calls in path order (each call's loop parallel over the pool when called
 * from the main thread); ref_frames_run keeps WHOLE FRAMES IN FLIGHT instead, one frame per pool thread, each
 * worker running its frame's calls serially into its own private output buffers -- how the encoder uses the
 * host cores (picture-level parallelism, enc_handle.c:770-781). */
typedef struct { int32_t restoration_type, sgr_ep, sgr_xqd[2]; int16_t hfilter[8], vfilter[8]; } RefLrUnitInfo;
void ref_lr_save_boundaries(void* plane_px00, int stride, int w, int h, int bit_depth, int plane, int frame_w, int frame_h, int after_cdef,
                            void* above, void* below, int bstride);
void ref_lr_filter_plane(void* data, int stride, void* dst, int dst_stride, int w, int h, int ss_x, int ss_y, int bit_depth, int unit_size,
                         const RefLrUnitInfo* units, void* above, void* below, int bstride, int optimized_lr);
typedef struct RefFrameJob {
    int32_t width, height, bit_depth, n_refs;
    const RefMePicture* cur; const RefMePicture* refs; const RefMeB64Cfg* me_cfg;
    RefMeB64Out me; /* MeSbResults + distortions + per-reference state of svt_aom_motion_estimation_b64 (best_sad / best_mv unused: NULL) */
    int16_t* residual; int32_t *coeff, *q, *dq; const int16_t *scan, *iscan; const uint8_t* qm;
    const RefFwdItem* fwd; const RefQuantItem* qi; const RefInvItem* inv; uint16_t* eobs;
    int64_t n_tx, n_coeffs;
    const void* pred; void* recon; void* cdef_out; void* final; const void* src;
    int64_t padded_elems;          /* pixels of one padded Y|U|V buffer */
    int64_t plane_off[3];          /* first pixel of each padded plane (including its border) */
    int32_t plane_stride[3], plane_w[3], plane_h[3], pad;
    int64_t src_off[3]; int32_t src_stride[3]; int32_t reserved0;
    const uint8_t* skip; const int32_t *str_y, *str_uv; int32_t n_str, damping, subsampling, reserved1;
    uint64_t* mse; uint8_t* dir; int32_t* var;
    const int8_t* fb_idx; const int32_t *apply_y, *apply_uv;
    const RefStatsItem* stats; int64_t *M, *H; const RefWienerUnit* units; int32_t n_stats, n_units;
    const RefLrUnitInfo* lr_units[3]; void* lr_above[3]; void* lr_below[3]; int32_t lr_unit_size[3], lr_bstride[3], lr_stripes[3], reserved2;
} RefFrameJob;

static void job_cdef_frame(const RefFrameJob* j, RefCdefFrame* f) {
    const int psz = j->bit_depth > 8 ? 2 : 1;
    const void** rec[3] = {&f->recon_y, &f->recon_cb, &f->recon_cr};
    const void** src[3] = {&f->src_y, &f->src_cb, &f->src_cr};
    for (int p = 0; p < 3; p++) {
        *rec[p] = (const uint8_t*)j->recon + (size_t)(j->plane_off[p] + (int64_t)j->pad * j->plane_stride[p] + j->pad) * psz;
        *src[p] = (const uint8_t*)j->src + (size_t)j->src_off[p] * psz;
    }
    f->recon_stride_y = j->plane_stride[0]; f->recon_stride_c = j->plane_stride[1];
    f->src_stride_y = j->src_stride[0]; f->src_stride_c = j->src_stride[1];
    f->width = j->width; f->height = j->height; f->bit_depth = j->bit_depth; f->damping = j->damping; f->subsampling_factor = j->subsampling;
    f->reserved = 0;
}
/* svt_extend_frame: replicate the picture edge into the padded border (restoration reads beyond the edge) */
static void job_extend(const RefFrameJob* j, void* buf) {
    const int psz = j->bit_depth > 8 ? 2 : 1, pad = j->pad;
    for (int p = 0; p < 3; p++) {
        const int w = j->plane_w[p], h = j->plane_h[p], st = j->plane_stride[p];
        uint8_t* base = (uint8_t*)buf + (size_t)j->plane_off[p] * psz;
        for (int y = 0; y < h; y++) {
            uint8_t* row = base + ((size_t)(pad + y) * st) * psz;
            if (psz == 1) {
                memset(row, row[pad], pad);
                memset(row + pad + w, row[pad + w - 1], pad);
            } else {
                uint16_t* r16 = (uint16_t*)row;
                for (int x = 0; x < pad; x++) { r16[x] = r16[pad]; r16[pad + w + x] = r16[pad + w - 1]; }
            }
        }
        const size_t rb = (size_t)(w + 2 * pad) * psz;
        for (int y = 0; y < pad; y++) {
            memcpy(base + ((size_t)y * st) * psz, base + ((size_t)pad * st) * psz, rb);
            memcpy(base + ((size_t)(pad + h + y) * st) * psz, base + ((size_t)(pad + h - 1) * st) * psz, rb);
        }
    }
}
static void lr_plane_body(void* vjob, int p) {
    const RefFrameJob* j = (const RefFrameJob*)vjob;
    const int psz = j->bit_depth > 8 ? 2 : 1, ss = p ? 1 : 0;
    const size_t o = (size_t)(j->plane_off[p] + (int64_t)j->pad * j->plane_stride[p] + j->pad) * psz;
    ref_lr_filter_plane((uint8_t*)j->cdef_out + o, j->plane_stride[p], (uint8_t*)j->final + o, j->plane_stride[p], j->plane_w[p], j->plane_h[p], ss, ss,
                        j->bit_depth, j->lr_unit_size[p], j->lr_units[p], j->lr_above[p], j->lr_below[p], j->lr_bstride[p], 0);
}
static void tx_chain_body(void* vctx, int i) { residual_body(vctx, i); fwd_body(vctx, i); quant_body(vctx, i); inv_body(vctx, i); }

static int g_trace = -1;
#define TRACE(x) do { if (g_trace < 0) g_trace = getenv("REF_TRACE") != NULL; if (g_trace) { fprintf(stderr, "[ref] %s\n", x); fflush(stderr); } } while (0)
void ref_frame_step(const RefFrameJob* j) {
    TRACE("me");
    const int nb = ((j->width + 63) >> 6) * ((j->height + 63) >> 6), psz = j->bit_depth > 8 ? 2 : 1;
    {   /* the reference's own open-loop ME driver for every 64x64 block (oracle/ref_me_b64.c) */
        RefMeControls ctrl;
        RefMeB64Out   mo = j->me;
        ref_me_b64_picture(j->cur, j->refs, j->me_cfg, &ctrl, &mo);
    }
    TRACE("tx");
    TxCtx tx = {j->residual, j->coeff, j->q, j->dq, j->scan, j->iscan, j->qm, j->fwd, j->qi, j->inv, j->eobs, j->pred, j->recon, j->bit_depth,
                j->src, j->residual, 1};
    par_for((int)j->n_tx, 64, tx_chain_body, &tx); /* per block: residual -> transform -> quantise -> inverse, as enc-dec does */
    TRACE("cdef search");
    /* svt_av1_loop_restoration_save_boundary_lines(frame, cm, 0) on the deblocked picture, before CDEF (dlf_process.c / cdef_process.c) */
    for (int p = 0; p < 3; p++)
        ref_lr_save_boundaries((uint8_t*)j->recon + (size_t)(j->plane_off[p] + (int64_t)j->pad * j->plane_stride[p] + j->pad) * psz, j->plane_stride[p],
                               j->plane_w[p], j->plane_h[p], j->bit_depth, p, j->width, j->height, 0, j->lr_above[p], j->lr_below[p], j->lr_bstride[p]);
    RefCdefFrame f;
    job_cdef_frame(j, &f);
    CdefSearchCtx cs = {&f, j->skip, j->str_y, j->str_uv, j->n_str, j->mse, j->dir, j->var};
    par_for(nb, 2, cdef_search_body, &cs);
    memcpy(j->cdef_out, j->recon, (size_t)j->padded_elems * psz); /* svt_av1_cdef_frame filters in place; the search input is kept */
    void* outp[3];
    for (int p = 0; p < 3; p++) outp[p] = (uint8_t*)j->cdef_out + (size_t)(j->plane_off[p] + (int64_t)j->pad * j->plane_stride[p] + j->pad) * psz;
    TRACE("cdef apply");
    CdefApplyCtx ca = {&f, j->skip, j->fb_idx, j->apply_y, j->apply_uv, outp[0], outp[1], outp[2], j->plane_stride[0], j->plane_stride[1]};
    par_for(nb, 2, cdef_apply_body, &ca);
    TRACE("extend");
    job_extend(j, j->cdef_out);
    TRACE("stats");
    StatsCtx st = {j->cdef_out, j->src, j->stats, j->M, j->H, j->bit_depth};
    par_for(j->n_stats, 1, stats_body, &st);
    TRACE("restoration");
    /* ... (cm, 1) after CDEF, then svt_av1_loop_restoration_filter_frame: every unit, stripe by stripe (rest_process.c:663-745) */
    for (int p = 0; p < 3; p++)
        ref_lr_save_boundaries(outp[p], j->plane_stride[p], j->plane_w[p], j->plane_h[p], j->bit_depth, p, j->width, j->height, 1, j->lr_above[p],
                               j->lr_below[p], j->lr_bstride[p]);
    par_for(3, 1, lr_plane_body, (void*)j);
}

/* private output buffers of one pool thread (allocated on first use, grown when a larger job arrives) */
typedef struct { size_t cap[32]; void* buf[32]; } WorkerBufs;
static __thread WorkerBufs t_bufs;
static void* wb(int k, size_t bytes) {
    if (t_bufs.cap[k] < bytes) {
        free(t_bufs.buf[k]);
        if (posix_memalign(&t_bufs.buf[k], 64, bytes + 64)) abort();
        memset(t_bufs.buf[k], 0, bytes); /* first touch on the worker's own NUMA node */
        t_bufs.cap[k] = bytes;
    }
    return t_bufs.buf[k];
}
typedef struct { const RefFrameJob* sets; int n_sets; } FramesCtx;
static void frame_body(void* vctx, int i) {
    const FramesCtx* c = (const FramesCtx*)vctx;
    RefFrameJob j = c->sets[i % c->n_sets];
    const size_t nb = (size_t)((j.width + 63) >> 6) * ((j.height + 63) >> 6), psz = j.bit_depth > 8 ? 2 : 1;
    int n_pu, max_cand, max_refs;
    ref_me_b64_sizes(j.me_cfg, j.width, j.height, &n_pu, &max_cand, &max_refs);
    j.me.total_me_candidate_index = wb(0, nb * (size_t)n_pu);
    j.me.me_candidate_array = wb(1, nb * (size_t)n_pu * max_cand);
    j.me.me_mv_array = wb(2, nb * (size_t)n_pu * max_refs * 4);
    j.me.distortion = wb(3, nb * 6 * 4);
    j.me.flags = wb(23, nb * 2);
    j.me.do_ref = wb(24, nb * 8);
    j.me.hme_centre = wb(25, nb * 8 * 2 * 2);
    j.me.zz_sad = wb(26, nb * 8 * 4);
    j.me.best_sad = NULL;
    j.me.best_mv = NULL;
    j.coeff = wb(4, (size_t)j.n_coeffs * 4);
    j.q = wb(5, (size_t)j.n_coeffs * 4);
    j.dq = wb(6, (size_t)j.n_coeffs * 4);
    j.eobs = wb(7, (size_t)j.n_tx * 2);
    j.recon = wb(8, (size_t)j.padded_elems * psz);
    j.cdef_out = wb(9, (size_t)j.padded_elems * psz);
    j.final = wb(10, (size_t)j.padded_elems * psz);
    j.mse = wb(11, 2 * nb * (size_t)j.n_str * 8);
    j.dir = wb(12, nb * 64);
    j.var = wb(13, nb * 64 * 4);
    j.M = wb(14, (size_t)j.n_stats * 49 * 8);
    j.H = wb(15, (size_t)j.n_stats * 2401 * 8);
    int64_t res_elems = 0;
    for (int p = 0; p < 3; p++) res_elems = j.src_off[p] + (int64_t)j.src_stride[p] * j.plane_h[p];
    j.residual = wb(16, (size_t)res_elems * 2);
    for (int p = 0; p < 3; p++) {
        const size_t bb = (size_t)2 * j.lr_stripes[p] * j.lr_bstride[p] * psz;
        j.lr_above[p] = wb(17 + 2 * p, bb);
        j.lr_below[p] = wb(18 + 2 * p, bb);
    }
    ref_frame_step(&j);
}
/* n_frames whole frames, frame i on job set i % n_sets, spread over `n_threads` pool threads (<= 0: all);
 * returns the wall-clock seconds of the batch */
double ref_frames_run(const RefFrameJob* sets, int n_sets, int n_frames, int n_threads) {
    ref_set_threads(n_threads);
    FramesCtx c = {sets, n_sets};
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    if (ref_num_threads() == 1) {
        for (int i = 0; i < n_frames; i++) frame_body(&c, i);
    } else {
        par_for(n_frames, 1, frame_body, &c);
    }
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}

/* ---- a13 groundwork: one restoration unit through the reference's own stripe loop ------------------------
 * svt_av1_loop_restoration_filter_unit (restoration.c:1067-1135) with need_boundaries = 1, RESTORE_WIENER, 8 bit.
 * `data` / `dst` point at pixel (0,0) of the plane; limits = {h_start, h_end, v_start, v_end}; tile = {left, top,
 * right, bottom}; above/below = the saved stripe-boundary lines (RESTORATION_CTX_VERT rows per stripe, `bstride`
 * bytes per row, logical column x at byte x + RESTORATION_EXTRA_HORZ is handled by the caller's pointer). */
static void lr_filter_unit_8bit(const RestorationUnitInfo* ruip, uint8_t* data, int stride, uint8_t* dst, int dst_stride,
                                const int32_t* limits, uint8_t* above, uint8_t* below, int bstride, const int32_t* tile,
                                int tile_stripe0, int ss_x, int ss_y, int optimized_lr);

void ref_lr_filter_unit_wiener_8bit(uint8_t* data, int stride, uint8_t* dst, int dst_stride, const int32_t* limits,
                                    const int16_t* hfilter, const int16_t* vfilter, uint8_t* above, uint8_t* below, int bstride,
                                    const int32_t* tile, int tile_stripe0, int ss_x, int ss_y, int optimized_lr) {
    RestorationUnitInfo rui;
    memset(&rui, 0, sizeof(rui));
    rui.restoration_type = RESTORE_WIENER;
    memcpy(rui.wiener_info.hfilter, hfilter, 8 * sizeof(int16_t));
    memcpy(rui.wiener_info.vfilter, vfilter, 8 * sizeof(int16_t));
    lr_filter_unit_8bit(&rui, data, stride, dst, dst_stride, limits, above, below, bstride, tile, tile_stripe0, ss_x, ss_y, optimized_lr);
}

/* the same with the self-guided filter (svt_aom_sgrproj_filter_stripe, restoration.c:994-1015) */
void ref_lr_filter_unit_sgrproj_8bit(uint8_t* data, int stride, uint8_t* dst, int dst_stride, const int32_t* limits, int ep,
                                     const int32_t* xqd, uint8_t* above, uint8_t* below, int bstride, const int32_t* tile,
                                     int tile_stripe0, int ss_x, int ss_y, int optimized_lr) {
    RestorationUnitInfo rui;
    memset(&rui, 0, sizeof(rui));
    rui.restoration_type    = RESTORE_SGRPROJ;
    rui.sgrproj_info.ep     = ep;
    rui.sgrproj_info.xqd[0] = xqd[0];
    rui.sgrproj_info.xqd[1] = xqd[1];
    lr_filter_unit_8bit(&rui, data, stride, dst, dst_stride, limits, above, below, bstride, tile, tile_stripe0, ss_x, ss_y, optimized_lr);
}

static void lr_filter_unit_8bit(const RestorationUnitInfo* ruip, uint8_t* data, int stride, uint8_t* dst, int dst_stride,
                                const int32_t* limits, uint8_t* above, uint8_t* below, int bstride, const int32_t* tile,
                                int tile_stripe0, int ss_x, int ss_y, int optimized_lr) {
    RestorationTileLimits lim = {limits[0], limits[1], limits[2], limits[3]};
    RestorationUnitInfo   rui = *ruip;
    RestorationStripeBoundaries rsb;
    rsb.stripe_boundary_above  = above;
    rsb.stripe_boundary_below  = below;
    rsb.stripe_boundary_stride = bstride;
    rsb.stripe_boundary_size   = 0;
    RestorationLineBuffers* rlbs = (RestorationLineBuffers*)malloc(sizeof(RestorationLineBuffers));
    Av1PixelRect            tr   = {tile[0], tile[1], tile[2], tile[3]};
    int32_t*                tmp  = (int32_t*)malloc(RESTORATION_TMPBUF_SIZE);
    svt_av1_loop_restoration_filter_unit(1, &lim, &rui, &rsb, rlbs, &tr, tile_stripe0, ss_x, ss_y, 0, 8, data, stride, dst,
                                         dst_stride, tmp, optimized_lr);
    free(tmp);
    free(rlbs);
}

/* ---- a13: whole-plane restoration through the reference's own functions ---------------------------------------------
 * boundary lines: svt_aom_save_tile_row_boundary_lines (restoration.c:1606), which only reads frm_size and the
 * subsampling flags of Av1Common; plane filter: the unit loop of foreach_rest_unit_in_tile (:1247-1294, static there,
 * restated) around the reference's svt_av1_loop_restoration_filter_unit (:1067). */
#include "pcs.h"

void ref_lr_save_boundaries(void* plane_px00, int stride, int w, int h, int bit_depth, int plane, int frame_w, int frame_h, int after_cdef,
                            void* above, void* below, int bstride) {
    Av1Common* cm = (Av1Common*)calloc(1, sizeof(Av1Common));
    cm->frm_size.frame_width = (uint16_t)frame_w;
    cm->frm_size.frame_height = (uint16_t)frame_h;
    cm->frm_size.superres_upscaled_width = (uint16_t)frame_w;
    cm->frm_size.superres_upscaled_height = (uint16_t)frame_h;
    cm->frm_size.superres_denominator = 8;
    cm->subsampling_x = cm->subsampling_y = 1;
    RestorationStripeBoundaries rsb;
    memset(&rsb, 0, sizeof(rsb));
    rsb.stripe_boundary_above = (uint8_t*)above;
    rsb.stripe_boundary_below = (uint8_t*)below;
    rsb.stripe_boundary_stride = bstride;
    svt_aom_save_tile_row_boundary_lines((uint8_t*)plane_px00, stride, w, h, bit_depth > 8, plane, cm, after_cdef, &rsb);
    free(cm);
}

/* data: pixel (0,0) of a plane with >= 3 pixels of writable border (the reference extends it in place, :1223) */
void ref_lr_filter_plane(void* data, int stride, void* dst, int dst_stride, int w, int h, int ss_x, int ss_y, int bit_depth, int unit_size,
                         const RefLrUnitInfo* units, void* above, void* below, int bstride, int optimized_lr) {
    const int highbd = bit_depth > 8;
    uint8_t* data8 = highbd ? CONVERT_TO_BYTEPTR((uint16_t*)data) : (uint8_t*)data;
    uint8_t* dst8 = highbd ? CONVERT_TO_BYTEPTR((uint16_t*)dst) : (uint8_t*)dst;
    svt_extend_frame(data8, w, h, stride, RESTORATION_BORDER, RESTORATION_BORDER, highbd);
    RestorationStripeBoundaries rsb;
    memset(&rsb, 0, sizeof(rsb));
    rsb.stripe_boundary_above = (uint8_t*)above;
    rsb.stripe_boundary_below = (uint8_t*)below;
    rsb.stripe_boundary_stride = bstride;
    RestorationLineBuffers* rlbs = (RestorationLineBuffers*)malloc(sizeof(RestorationLineBuffers));
    int32_t* tmp = (int32_t*)malloc(RESTORATION_TMPBUF_SIZE);
    Av1PixelRect tile = {0, 0, w, h};
    tile.left = 0; tile.top = 0; tile.right = w; tile.bottom = h;
    const int hunits = (w + (unit_size >> 1)) / unit_size > 1 ? (w + (unit_size >> 1)) / unit_size : 1;
    const int ext = unit_size * 3 / 2, voff = RESTORATION_UNIT_OFFSET >> ss_y;
    int y0 = 0, i = 0;
    while (y0 < h) {
        const int rem_h = h - y0, uh = rem_h < ext ? rem_h : unit_size;
        RestorationTileLimits lim;
        lim.v_start = y0; lim.v_end = y0 + uh;
        lim.v_start = lim.v_start - voff > 0 ? lim.v_start - voff : 0;
        if (lim.v_end < h) lim.v_end -= voff;
        int x0 = 0, j = 0;
        while (x0 < w) {
            const int rem_w = w - x0, uw = rem_w < ext ? rem_w : unit_size;
            lim.h_start = x0; lim.h_end = x0 + uw;
            const RefLrUnitInfo* u = &units[i * hunits + j];
            RestorationUnitInfo  rui;
            memset(&rui, 0, sizeof(rui));
            rui.restoration_type = (RestorationType)u->restoration_type;
            memcpy(rui.wiener_info.hfilter, u->hfilter, 16);
            memcpy(rui.wiener_info.vfilter, u->vfilter, 16);
            rui.sgrproj_info.ep = u->sgr_ep;
            rui.sgrproj_info.xqd[0] = u->sgr_xqd[0];
            rui.sgrproj_info.xqd[1] = u->sgr_xqd[1];
            svt_av1_loop_restoration_filter_unit(1, &lim, &rui, &rsb, rlbs, &tile, 0, ss_x, ss_y, highbd, bit_depth, data8, stride, dst8, dst_stride,
                                                 tmp, optimized_lr);
            x0 += uw; j++;
        }
        y0 += uh; i++;
    }
    free(tmp);
    free(rlbs);
}
