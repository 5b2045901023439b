// me_picture.cu -- T2 open-loop motion estimation for a whole picture: HME pyramid construction (K13),
// HME level 0/1/2, final search centre, zero-centre check and the 85-PU full-pel search (sm_90a).
//
// Reference behaviour restated (the "core" open-loop path; see DESIGN.md for the MeContext controls
// that are honoured and those that are not):
//   svt_aom_downsample_2d_c + svt_aom_generate_padding   Source/Lib/Codec/pic_analysis_process.c:130-160, 2138-2190
//   hme_level_0 / hme_level_1 / hme_level_2               Source/Lib/Codec/motion_estimation.c:820-1113
//   hme_level{0,1,2}_b64 region loops                     :1906-2180
//   set_final_seach_centre_sb (HME level-2 branch)        :2182-2390
//   check_00_center                                       :1139-1210
//   integer_search_b64 search-area derivation + clipping  :1249-1520
//   open_loop_me_fullpel_search_sblock                    :781-817   (kernel: me_pyramid.cu)
//
// Pipeline per picture (all references, all 64x64 blocks in every launch):
//   prepare(L0) -> sad_search -> finish(L0) -> prepare(L1) -> sad_search -> finish(L1) ->
//   prepare(L2) -> sad_search -> finish(L2) -> centre (+ optional zero-centre check, builds the
//   full-pel items) -> fullpel_search.
// The search kernels are the ones behind the T1 entry points (sad.cu / me_pyramid.cu); the small
// prepare/finish kernels only do the reference's window arithmetic, one thread per (ref, b64, region).
#include <map>

#include "common.cuh"
#include "sad_small.cuh"
#include "me_hme.cuh"
#include "../../include/svt_b200.h"

namespace b200 {
bool launch_fullpel_tma(const SvtB200MePicture* cur, const SvtB200MePicture* refs, int n_refs, int n_b64, const SvtB200FullpelItem* d_items,
                        int n_items, uint32_t* d_best_sad, uint32_t* d_best_mv, cudaStream_t st, const uint32_t* d_seed_sad = nullptr);  // me_pyramid.cu

void launch_sad_search(const uint8_t* d_src, const uint8_t* d_ref, const SvtB200SadSearchItem* d_items, int n,
                       SvtB200SadSearchResult* d_results, size_t smem, int max_positions, cudaStream_t st);

// ---- K13 ----------------------------------------------------------------------------------------
__global__ void downsample_2d_kernel(const uint8_t* __restrict__ in, int in_stride, int in_w, int in_h, uint8_t* __restrict__ out,
                                     int out_stride, int step) {
    const int half = step >> 1;
    const int ow = (in_w - half + step - 1) / step, oh = (in_h - half + step - 1) / step;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < ow * oh; idx += gridDim.x * blockDim.x) {
        const int oy = idx / ow, ox = idx - oy * ow;
        const int y = half + oy * step, x = half + ox * step;
        const uint32_t s = (uint32_t)in[(size_t)(y - 1) * in_stride + x - 1] + in[(size_t)(y - 1) * in_stride + x] +
                           in[(size_t)y * in_stride + x - 1] + in[(size_t)y * in_stride + x];
        out[(size_t)oy * out_stride + ox] = (uint8_t)((s + 2) >> 2);
    }
}
// replicate the w x h interior (at (org_x, org_y)) into the surrounding padding (svt_aom_generate_padding);
// only the border elements are visited: top band, bottom band, then the left/right strips of the interior rows
template <typename PIX>
__device__ __forceinline__ void pad_border_element(PIX* buf, int stride, int w, int h, int org_x, int org_y, int idx) {
    const int tw = w + 2 * org_x, band = org_y * tw;
    int x, y;
    if (idx < 2 * band) {
        const int j = idx < band ? idx : idx - band;
        y = j / tw + (idx < band ? 0 : org_y + h);
        x = j % tw;
    } else {
        const int j = idx - 2 * band, xx = j % (2 * org_x);
        y = org_y + j / (2 * org_x);
        x = xx < org_x ? xx : w + xx;
    }
    const int sx = min(max(x, org_x), org_x + w - 1), sy = min(max(y, org_y), org_y + h - 1);
    buf[(size_t)y * stride + x] = buf[(size_t)sy * stride + sx];
}
__host__ __device__ __forceinline__ int pad_border_count(int w, int h, int org_x, int org_y) {
    return 2 * org_y * (w + 2 * org_x) + 2 * org_x * h;
}
__global__ void pad_plane_kernel(uint8_t* buf, int stride, int w, int h, int org_x, int org_y) {
    const int n = pad_border_count(w, h, org_x, org_y);
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x)
        pad_border_element(buf, stride, w, h, org_x, org_y, idx);
}

__global__ void hme_prepare_kernel(SvtB200MePicture cur, const SvtB200MePicture* __restrict__ refs, const SvtB200MeParams* __restrict__ prm,
                                   int n_refs, int n_b64, int b64_w, int level, const int16_t* __restrict__ prev_x,
                                   const int16_t* __restrict__ prev_y, SvtB200SadSearchItem* __restrict__ items, HmeSide* __restrict__ side) {
    const int total = n_refs * n_b64 * 4;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        const int reg = idx & 3, b = (idx >> 2) % n_b64, r = (idx >> 2) / n_b64;
        hme_make_item(cur, refs[r], prm[r], level, reg & 1, reg >> 1, b % b64_w, b / b64_w, level ? prev_x[idx] : (int16_t)0,
                      level ? prev_y[idx] : (int16_t)0, items[idx], side[idx]);
    }
}

__global__ void hme_finish_kernel(const SvtB200SadSearchResult* __restrict__ res, const HmeSide* __restrict__ side,
                                  const SvtB200MeParams* __restrict__ prm, int n_refs, int n_b64, int level, int16_t* __restrict__ out_x,
                                  int16_t* __restrict__ out_y, uint64_t* __restrict__ out_sad) {
    const int total = n_refs * n_b64 * 4;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x)
        hme_finish_one(res[idx], side[idx], prm[(idx >> 2) / n_b64], level, out_x[idx], out_y[idx], out_sad[idx]);
}

// One warp per (ref, b64): final HME centre over the four regions' level-2 results (l2x/l2y/l2sad[4]),
// optional zero-centre check, full-pel search item.
__device__ __forceinline__ void me_centre_one(const SvtB200MePicture& cur, const SvtB200MePicture& rp, const SvtB200MeParams& p, int i,
                                              int bx, int by, const int16_t* l2x, const int16_t* l2y, const uint64_t* l2sad,
                                              int16_t* __restrict__ hme_sc, uint64_t* __restrict__ hme_sad,
                                              SvtB200FullpelItem* __restrict__ items, int lane) {
    // region scan order of set_final_seach_centre_sb: [w=0][h=0] first, then w inner / h outer, strict '<'
    int16_t  cx = l2x[0], cy = l2y[0];
    uint64_t cs = l2sad[0];
    for (int reg = 1; reg < 4; reg++)
        if (l2sad[reg] < cs) {
            cs = l2sad[reg];
            cx = l2x[reg];
            cy = l2y[reg];
        }
    const int16_t org_x = (int16_t)(bx * 64), org_y = (int16_t)(by * 64);
    const int blk_w = min(64, cur.width[2] - org_x), blk_h = min(64, cur.height[2] - org_y);
    const uint8_t* src = cur.plane[2] + (size_t)(cur.org_y[2] + org_y) * cur.stride[2] + cur.org_x[2] + org_x;
    int16_t sx = cx, sy = cy;
    if (p.check_zero_centre && (sx != 0 || sy != 0)) {
        // check_00_center: SADs on every other row (x2), zero MV wins ties
        const int16_t pw = 63, ph = 63, W = (int16_t)rp.width[2], H = (int16_t)rp.height[2];
        if ((int16_t)(org_x + sx) < -pw) sx = (int16_t)(-pw - org_x);
        if ((int16_t)(org_x + sx) > (int16_t)(W - 1)) sx = (int16_t)(sx - ((org_x + sx) - (W - 1)));
        if ((int16_t)(org_y + sy) < -ph) sy = (int16_t)(-ph - org_y);
        if ((int16_t)(org_y + sy) > (int16_t)(H - 1)) sy = (int16_t)(sy - ((org_y + sy) - (H - 1)));
        const uint8_t* r0 = rp.plane[2] + (size_t)(rp.org_y[2] + org_y) * rp.stride[2] + rp.org_x[2] + org_x;
        const uint8_t* r1 = r0 + (ptrdiff_t)sy * rp.stride[2] + sx;
        // lane = one of the (up to 32) rows that are summed; each row is walked word by word with
        // funnel-shifted aligned loads, all of them independent (one global round trip per lane)
        uint32_t z = 0, hsad = 0;
        if (lane < (blk_h >> 1)) {
            const int      yy = lane * 2, nw = (blk_w + 3) >> 2, tail = blk_w & 3;
            const uint32_t tailmask = tail ? ((1u << (tail * 8)) - 1u) : 0xffffffffu;
            const ByteRun  S(src + (size_t)yy * cur.stride[2], blk_w), A(r0 + (size_t)yy * rp.stride[2], blk_w),
                B(r1 + (ptrdiff_t)yy * rp.stride[2], blk_w);
            uint32_t slo = S.raw(0), alo = A.raw(0), blo = B.raw(0);
#pragma unroll 4
            for (int j = 0; j < nw; j++) {
                const uint32_t shi = S.raw(j + 1), ahi = A.raw(j + 1), bhi = B.raw(j + 1);
                const uint32_t m = j == nw - 1 ? tailmask : 0xffffffffu;
                const uint32_t sv = __funnelshift_r(slo, shi, S.shift) & m;
                z    = __vsadu4(sv, __funnelshift_r(alo, ahi, A.shift) & m) + z;
                hsad = __vsadu4(sv, __funnelshift_r(blo, bhi, B.shift) & m) + hsad;
                slo = shi;
                alo = ahi;
                blo = bhi;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            z += __shfl_xor_sync(0xffffffffu, z, o);
            hsad += __shfl_xor_sync(0xffffffffu, hsad, o);
        }
        z <<= 1;
        hsad <<= 1;
        if (z <= hsad) sx = sy = 0;  // MIN(zero_cost, hme_cost) == zero_cost
    }
    if (lane == 0) {
        hme_sc[2 * i]     = cx;
        hme_sc[2 * i + 1] = cy;
        hme_sad[i]        = cs;
        // integer_search_b64 (:1296-1320, :1440-1496)
        int16_t sa_w = (int16_t)((max(1, p.me_sa_w) + 7) & ~0x07), sa_h = (int16_t)max(3, p.me_sa_h);
        int16_t ox = (int16_t)(sx - (sa_w >> 1)), oy = (int16_t)(sy - (sa_h >> 1));
        const int16_t pw = 63, ph = 63, W = (int16_t)cur.width[2], H = (int16_t)cur.height[2];
        {
            const bool left = (int16_t)(org_x + ox) < -pw;
            const int16_t nox = left ? (int16_t)(-pw - org_x) : ox;
            // the reference evaluates the width correction with the ALREADY corrected origin
            sa_w = ((int16_t)(org_x + nox) < -pw) ? (int16_t)(sa_w - (-pw - (org_x + nox))) : sa_w;
            ox = nox;
            ox = ((int16_t)(org_x + ox) > (int16_t)(W - 1)) ? (int16_t)(ox - ((org_x + ox) - (W - 1))) : ox;
            sa_w = ((int16_t)(org_x + ox + sa_w) > W) ? (int16_t)max(1, sa_w - ((org_x + ox + sa_w) - W)) : sa_w;
            sa_w = (sa_w < 8) ? sa_w : (int16_t)(sa_w & ~0x07);
            const bool top = (int16_t)(org_y + oy) < -ph;
            const int16_t noy = top ? (int16_t)(-ph - org_y) : oy;
            sa_h = ((int16_t)(org_y + noy) < -ph) ? (int16_t)(sa_h - (-ph - (org_y + noy))) : sa_h;
            oy = noy;
            oy = ((int16_t)(org_y + oy) > (int16_t)(H - 1)) ? (int16_t)(oy - ((org_y + oy) - (H - 1))) : oy;
            sa_h = ((int16_t)(org_y + oy + sa_h) > H) ? (int16_t)max(1, sa_h - ((org_y + oy + sa_h) - H)) : sa_h;
        }
        SvtB200FullpelItem it;
        it.src_off    = (uint64_t)(uintptr_t)src;
        it.ref_off    = (uint64_t)(uintptr_t)(rp.plane[2] + (ptrdiff_t)(rp.org_y[2] + org_y + oy) * rp.stride[2] + rp.org_x[2] + org_x + ox);
        it.src_stride = (uint32_t)cur.stride[2];
        it.ref_stride = (uint32_t)rp.stride[2];
        it.sa_w = sa_w;
        it.sa_h = sa_h;
        it.org_x = ox;
        it.org_y = oy;
        it.sub_sad = (uint8_t)(p.me_sub_sad ? 1 : 0);
        it.seeded = 0;
        it.seed_x = it.seed_y = 0;
        it.reserved[0] = it.reserved[1] = 0;
        items[i] = it;
    }
}

__global__ void me_centre_kernel(SvtB200MePicture cur, const SvtB200MePicture* __restrict__ refs, const SvtB200MeParams* __restrict__ prm,
                                 int n_refs, int n_b64, int b64_w, const int16_t* __restrict__ l2x, const int16_t* __restrict__ l2y,
                                 const uint64_t* __restrict__ l2sad, int16_t* __restrict__ hme_sc /*[n][2]*/, uint64_t* __restrict__ hme_sad,
                                 SvtB200FullpelItem* __restrict__ items) {
    const int lane = threadIdx.x & 31;
    const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int i = wid; i < n_refs * n_b64; i += nw) {
        const int b = i % n_b64, r = i / n_b64;
        me_centre_one(cur, refs[r], prm[r], i, b % b64_w, b / b64_w, l2x + i * 4, l2y + i * 4, l2sad + i * 4, hme_sc, hme_sad, items, lane);
    }
}

// The whole hierarchical search of one (ref, b64) pair in ONE CTA when every level's search area is small:
// warp = search region; a warp runs level 0 -> 1 -> 2 for its region back to back (each level starts from
// the same region's previous result, so nothing leaves the registers), the four level-2 results meet in
// shared memory and warp 0 picks the centre and writes the full-pel item.  Replaces 3 x (prepare, search,
// finish) + centre = 10 launches and their global round trips.
struct MeRefTable {  // passed by value: the descriptors reach the kernel with the launch, no copy to wait for
    SvtB200MePicture pic[16];
    SvtB200MeParams  prm[16];
};
__global__ void __launch_bounds__(128)
hme_fused_kernel(const SvtB200MePicture cur, const __grid_constant__ MeRefTable tab, int n_refs, int n_b64, int b64_w,
                 int16_t* __restrict__ hme_sc, uint64_t* __restrict__ hme_sad, SvtB200FullpelItem* __restrict__ items) {
    __shared__ int16_t  s_x[4], s_y[4];
    __shared__ uint64_t s_sad[4];
    const int i = blockIdx.x, reg = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = i % n_b64, r = i / n_b64, bx = b % b64_w, by = b / b64_w;
    const SvtB200MePicture rp = tab.pic[r];
    const SvtB200MeParams  p  = tab.prm[r];
    int16_t  px = 0, py = 0;
    uint64_t sad = 0;
#pragma unroll 1
    for (int level = 0; level < 3; level++) {
        SvtB200SadSearchItem it;
        HmeSide              sd;
        hme_make_item(cur, rp, p, level, reg & 1, reg >> 1, bx, by, px, py, it, sd);
        const unsigned long long best = sad_search_warp((const uint8_t*)(uintptr_t)it.src_off, (const uint8_t*)(uintptr_t)it.ref_off, it, lane);
        hme_finish_one(sad_key_to_result(best), sd, p, level, px, py, sad);
    }
    if (lane == 0) {
        s_x[reg]   = px;
        s_y[reg]   = py;
        s_sad[reg] = sad;
    }
    __syncthreads();
    if (reg == 0) me_centre_one(cur, rp, p, i, bx, by, s_x, s_y, s_sad, hme_sc, hme_sad, items, lane);
}

struct MeWorkspace {
    size_t cap = 0;  // in (ref, b64) pairs
    SvtB200SadSearchItem* items = nullptr;
    SvtB200SadSearchResult* res = nullptr;
    HmeSide* side = nullptr;
    int16_t *x[3] = {nullptr, nullptr, nullptr}, *y[3] = {nullptr, nullptr, nullptr};
    uint64_t* sad[3] = {nullptr, nullptr, nullptr};
    SvtB200FullpelItem* fp_items = nullptr;
    SvtB200MePicture* refs = nullptr;
    SvtB200MeParams* prm = nullptr;
};
// one workspace per stream: calls enqueued on different streams may execute concurrently
static std::map<cudaStream_t, MeWorkspace> g_me_ws;
static std::mutex  g_me_mu;

static void me_ws_reserve(MeWorkspace& w, size_t pairs) {
    if (pairs <= w.cap) return;
    // a larger picture arrived on this stream: NEW buffers; the old ones stay valid (a captured graph may replay them) until shutdown
    w.cap = pairs * 2;
    const size_t n4 = w.cap * 4;
    w.items = (SvtB200SadSearchItem*)scratch_alloc(n4 * sizeof(SvtB200SadSearchItem));
    w.res = (SvtB200SadSearchResult*)scratch_alloc(n4 * sizeof(SvtB200SadSearchResult));
    w.side = (HmeSide*)scratch_alloc(n4 * sizeof(HmeSide));
    for (int l = 0; l < 3; l++) {
        w.x[l] = (int16_t*)scratch_alloc(n4 * 2);
        w.y[l] = (int16_t*)scratch_alloc(n4 * 2);
        w.sad[l] = (uint64_t*)scratch_alloc(n4 * 8);
    }
    w.fp_items = (SvtB200FullpelItem*)scratch_alloc(w.cap * sizeof(SvtB200FullpelItem));
    w.refs = (SvtB200MePicture*)scratch_alloc(16 * sizeof(SvtB200MePicture));
    w.prm = (SvtB200MeParams*)scratch_alloc(16 * sizeof(SvtB200MeParams));
}
static ResetHook g_me_reset([] { std::lock_guard<std::mutex> lk(g_me_mu); g_me_ws.clear(); });

}  // namespace b200

using namespace b200;

// T1: downsample_2d (aom_dsp_rtcd.h:841)
extern "C" void svt_b200_downsample_2d(uint8_t* input_samples, uint32_t input_stride, uint32_t input_area_width, uint32_t input_area_height,
                                       uint8_t* decim_samples, uint32_t decim_stride, uint32_t decim_step) {
    require_ready();
    const uint32_t half = decim_step >> 1;
    if (input_area_width <= half || input_area_height <= half) return;
    const uint32_t ow = (input_area_width - half + decim_step - 1) / decim_step, oh = (input_area_height - half + decim_step - 1) / decim_step;
    LaneGuard l;
    size_t o_in = l->alloc((size_t)input_area_height * input_area_width);
    size_t in_end = l->used;
    size_t o_out = l->alloc((size_t)ow * oh);
    for (uint32_t r = 0; r < input_area_height; r++) memcpy(l->h<uint8_t>(o_in) + (size_t)r * input_area_width, input_samples + (size_t)r * input_stride, input_area_width);
    l->h2d(0, in_end);
    downsample_2d_kernel<<<grid_for((ow * oh + 255) / 256, 8), 256, 0, l->stream>>>(l->d<uint8_t>(o_in), (int)input_area_width, (int)input_area_width,
                                                                                 (int)input_area_height, l->d<uint8_t>(o_out), (int)ow, (int)decim_step);
    B200_LAUNCH_CHECK();
    l->d2h(o_out, (size_t)ow * oh);
    l->sync();
    for (uint32_t r = 0; r < oh; r++) memcpy(decim_samples + (size_t)r * decim_stride, l->h<uint8_t>(o_out) + (size_t)r * ow, ow);
}

struct PadPlanes {
    SvtB200PlaneExtent p[4];
};
// several planes in one launch: blockIdx.y = plane
__global__ void pad_planes_kernel(const __grid_constant__ PadPlanes pl) {
    const SvtB200PlaneExtent& e = pl.p[blockIdx.y];
    const int n = pad_border_count(e.w, e.h, e.org_x, e.org_y);
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x)
        if (e.pixel_bytes == 2) pad_border_element(reinterpret_cast<uint16_t*>(e.buf), e.stride, e.w, e.h, e.org_x, e.org_y, idx);
        else pad_border_element(e.buf, e.stride, e.w, e.h, e.org_x, e.org_y, idx);
}

extern "C" int svt_b200_extend_planes_dev(const SvtB200PlaneExtent* planes, int n_planes, void* stream) {
    require_ready();
    if (!planes || n_planes <= 0 || n_planes > 4) return SVT_B200_ERR_BAD_ARG;
    PadPlanes pl;
    memset(&pl, 0, sizeof(pl));
    int tn = 0;
    for (int i = 0; i < n_planes; i++) {
        if (!planes[i].buf || planes[i].w <= 0 || planes[i].h <= 0) return SVT_B200_ERR_BAD_ARG;
        pl.p[i] = planes[i];
        const int t = pad_border_count(planes[i].w, planes[i].h, planes[i].org_x, planes[i].org_y);
        tn = t > tn ? t : tn;
    }
    pad_planes_kernel<<<dim3(grid_for((tn + 255) / 256, 4), n_planes), 256, 0, (cudaStream_t)stream>>>(pl);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

extern "C" int svt_b200_extend_plane_dev(uint8_t* d_buf, int stride, int w, int h, int org_x, int org_y, void* stream) {
    require_ready();
    if (!d_buf || w <= 0 || h <= 0) return SVT_B200_ERR_BAD_ARG;
    const int tn = pad_border_count(w, h, org_x, org_y);
    if (tn <= 0) return SVT_B200_OK;
    pad_plane_kernel<<<grid_for((tn + 255) / 256, 8), 256, 0, (cudaStream_t)stream>>>(d_buf, stride, w, h, org_x, org_y);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

// T2: build the padded 1/4 and 1/16 luma planes of one picture on the device
extern "C" int svt_b200_build_hme_pyramid_dev(const SvtB200MePicture* pic, void* stream) {
    require_ready();
    if (!pic) return SVT_B200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    for (int lvl = 1; lvl >= 0; lvl--) {  // quarter from full, sixteenth from quarter
        const int s = lvl + 1;
        const uint8_t* in = pic->plane[s] + (size_t)pic->org_y[s] * pic->stride[s] + pic->org_x[s];
        uint8_t* out = const_cast<uint8_t*>(pic->plane[lvl]) + (size_t)pic->org_y[lvl] * pic->stride[lvl] + pic->org_x[lvl];
        const int n = pic->width[lvl] * pic->height[lvl];
        downsample_2d_kernel<<<grid_for((n + 255) / 256, 8), 256, 0, st>>>(in, pic->stride[s], pic->width[s], pic->height[s], out, pic->stride[lvl], 2);
        B200_LAUNCH_CHECK();
        const int tn = pad_border_count(pic->width[lvl], pic->height[lvl], pic->org_x[lvl], pic->org_y[lvl]);
        pad_plane_kernel<<<grid_for((tn + 255) / 256, 8), 256, 0, st>>>(const_cast<uint8_t*>(pic->plane[lvl]), pic->stride[lvl], pic->width[lvl],
                                                                      pic->height[lvl], pic->org_x[lvl], pic->org_y[lvl]);
        B200_LAUNCH_CHECK();
    }
    return SVT_B200_OK;
}

extern "C" int svt_b200_me_picture_dev(const SvtB200MePicture* cur, const SvtB200MePicture* refs, const SvtB200MeParams* params, int n_refs,
                                       uint32_t* d_best_sad, uint32_t* d_best_mv, int16_t* d_hme_centre, uint64_t* d_hme_sad, void* stream) {
    require_ready();
    if (!cur || !refs || !params || n_refs <= 0 || n_refs > 16) return SVT_B200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int b64_w = (cur->width[2] + 63) >> 6, b64_h = (cur->height[2] + 63) >> 6, n_b64 = b64_w * b64_h;
    const int pairs = n_refs * n_b64, n4 = pairs * 4;
    std::lock_guard<std::mutex> lk(g_me_mu);
    MeWorkspace& w = g_me_ws[st];
    me_ws_reserve(w, (size_t)pairs);
    const int g = grid_for((n4 + 255) / 256, 8);
    int max_l0_w = 8, max_l0_h = 1, max_pos[3] = {1, 1, 1};
    for (int r = 0; r < n_refs; r++) {
        max_l0_w = max_l0_w > ((params[r].hme_l0_sa_w + 7) & ~7) ? max_l0_w : ((params[r].hme_l0_sa_w + 7) & ~7);
        max_l0_h = max_l0_h > params[r].hme_l0_sa_h ? max_l0_h : params[r].hme_l0_sa_h;
        const int pos[3] = {((params[r].hme_l0_sa_w + 7) & ~7) * params[r].hme_l0_sa_h, ((params[r].hme_l1_sa_w + 7) & ~7) * params[r].hme_l1_sa_h,
                            ((params[r].hme_l2_sa_w + 7) & ~7) * params[r].hme_l2_sa_h};
        for (int l = 0; l < 3; l++) max_pos[l] = max_pos[l] > pos[l] ? max_pos[l] : pos[l];
    }
    if (max_pos[0] <= kSmallSearchMaxPos && max_pos[1] <= kSmallSearchMaxPos && max_pos[2] <= kSmallSearchMaxPos) {
        MeRefTable tab;
        memset(&tab, 0, sizeof(tab));
        memcpy(tab.pic, refs, n_refs * sizeof(SvtB200MePicture));
        memcpy(tab.prm, params, n_refs * sizeof(SvtB200MeParams));
        hme_fused_kernel<<<pairs, 128, 0, st>>>(*cur, tab, n_refs, n_b64, b64_w, d_hme_centre, d_hme_sad, w.fp_items);
        B200_LAUNCH_CHECK();
        if (launch_fullpel_tma(cur, refs, n_refs, n_b64, w.fp_items, pairs, d_best_sad, d_best_mv, st)) return SVT_B200_OK;
        return svt_b200_fullpel_search_batch_dev(nullptr, nullptr, w.fp_items, pairs, d_best_sad, d_best_mv, stream);
    }
    B200_CUDA_CHECK(cudaMemcpyAsync(w.refs, refs, n_refs * sizeof(SvtB200MePicture), cudaMemcpyHostToDevice, st));
    B200_CUDA_CHECK(cudaMemcpyAsync(w.prm, params, n_refs * sizeof(SvtB200MeParams), cudaMemcpyHostToDevice, st));
    for (int level = 0; level < 3; level++) {
        hme_prepare_kernel<<<g, 256, 0, st>>>(*cur, w.refs, w.prm, n_refs, n_b64, b64_w, level, level ? w.x[level - 1] : nullptr,
                                              level ? w.y[level - 1] : nullptr, w.items, w.side);
        B200_LAUNCH_CHECK();
        const int bs = 16 << level;
        // shared-memory bound for this level's searches (the kernel adapts its tiling to what it gets)
        const int saw = level == 0 ? max_l0_w : 16, sah = level == 0 ? max_l0_h : 8;
        const size_t lw = ((saw + bs + 3) >> 2) + 10;
        const size_t smem = (size_t)(((bs + 15) >> 4) << 2) * 4 * bs + 2048 * 4 + 64 + (size_t)(sah - 1 + 2 * (bs - 1) + 1) * lw * 4;
        launch_sad_search(nullptr, nullptr, w.items, n4, w.res, smem, max_pos[level], st);
        hme_finish_kernel<<<g, 256, 0, st>>>(w.res, w.side, w.prm, n_refs, n_b64, level, w.x[level], w.y[level], w.sad[level]);
        B200_LAUNCH_CHECK();
    }
    me_centre_kernel<<<grid_for((pairs * 32 + 255) / 256, 8), 256, 0, st>>>(*cur, w.refs, w.prm, n_refs, n_b64, b64_w, w.x[2], w.y[2], w.sad[2],
                                                                          d_hme_centre, d_hme_sad, w.fp_items);
    B200_LAUNCH_CHECK();
    if (launch_fullpel_tma(cur, refs, n_refs, n_b64, w.fp_items, pairs, d_best_sad, d_best_mv, st)) return SVT_B200_OK;
    return svt_b200_fullpel_search_batch_dev(nullptr, nullptr, w.fp_items, pairs, d_best_sad, d_best_mv, stream);
}
