// dlf.cuh -- the AV1 deblocking filters along one line of pixels across an edge (reference: deblocking_common.c:140-866),
// shared by the T1 entry points and the whole-picture passes of dlf.cu.
//
// A "line" is the run of pixels perpendicular to the edge: s[-k * step] is p(k-1), s[k * step] is q(k).  One call
// filters one line; a reference lpf call is four lines.  The 8-bit filters are the high-bit-depth ones at shift 0 (the
// reference's int8 arithmetic with ^0x80 is the same clamp to [-128, 127] around 128), so one body serves both.
#pragma once
#include <cstddef>
#include <cstdint>

namespace b200 {
namespace dlf {

__device__ __forceinline__ int iabs(int v) { return v < 0 ? -v : v; }
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
__device__ __forceinline__ int rnd3(int v) { return (v + 4) >> 3; }
__device__ __forceinline__ int rnd4(int v) { return (v + 8) >> 4; }

// Thresholds of one edge, already scaled to the bit depth: lim / blim / hev compared with pixel differences, flat = 1 << shift.
struct Thr {
    int blim, lim, hev, flat, shift;
};
__device__ __forceinline__ Thr make_thr(int blimit, int limit, int thresh, int shift) {
    Thr t;
    t.blim = blimit << shift;
    t.lim = limit << shift;
    t.hev = thresh << shift;
    t.flat = 1 << shift;
    t.shift = shift;
    return t;
}

// the 4-tap filter (filter4 / highbd_filter4): mask and hev are 0 or -1
template <typename T>
__device__ __forceinline__ void filter4(int mask, int hev, int shift, T& op1, T& op0, T& oq0, T& oq1) {
    const int off = 0x80 << shift, lo = -(128 << shift), hi = (128 << shift) - 1;
    const int ps1 = (int)op1 - off, ps0 = (int)op0 - off, qs0 = (int)oq0 - off, qs1 = (int)oq1 - off;
    int f = clampi(ps1 - qs1, lo, hi) & hev;
    f = clampi(f + 3 * (qs0 - ps0), lo, hi) & mask;
    const int f1 = clampi(f + 4, lo, hi) >> 3;
    const int f2 = clampi(f + 3, lo, hi) >> 3;
    oq0 = (T)(clampi(qs0 - f1, lo, hi) + off);
    op0 = (T)(clampi(ps0 + f2, lo, hi) + off);
    f = ((f1 + 1) >> 1) & ~hev;
    oq1 = (T)(clampi(qs1 - f, lo, hi) + off);
    op1 = (T)(clampi(ps1 + f, lo, hi) + off);
}

__device__ __forceinline__ int hev_of(const Thr& t, int p1, int p0, int q0, int q1) {
    return (iabs(p1 - p0) > t.hev || iabs(q1 - q0) > t.hev) ? -1 : 0;
}
__device__ __forceinline__ bool outer_ok(const Thr& t, int p1, int p0, int q0, int q1) {
    return iabs(p0 - q0) * 2 + iabs(p1 - q1) / 2 <= t.blim;
}

// TAPS = 4, 6, 8 or 14 (lpf_*_4 / _6 / _8 / _14): reads 2 / 3 / 4 / 7 pixels on each side, writes 2 / 2 / 3 / 6.
template <int TAPS, typename T>
__device__ __forceinline__ void filter_line(T* s, ptrdiff_t step, const Thr& t) {
    if (TAPS == 4) {
        T p1 = s[-2 * step], p0 = s[-step], q0 = s[0], q1 = s[step];
        const int mask = (iabs(p1 - p0) <= t.lim && iabs(q1 - q0) <= t.lim && outer_ok(t, p1, p0, q0, q1)) ? -1 : 0;
        filter4(mask, hev_of(t, p1, p0, q0, q1), t.shift, p1, p0, q0, q1);
        s[-2 * step] = p1; s[-step] = p0; s[0] = q0; s[step] = q1;
    } else if (TAPS == 6) {
        const int p2 = s[-3 * step], q2 = s[2 * step];
        T p1 = s[-2 * step], p0 = s[-step], q0 = s[0], q1 = s[step];
        const bool mask = iabs(p2 - p1) <= t.lim && iabs(p1 - p0) <= t.lim && iabs(q1 - q0) <= t.lim && iabs(q2 - q1) <= t.lim &&
                          outer_ok(t, p1, p0, q0, q1);
        const bool flat = iabs(p1 - p0) <= t.flat && iabs(q1 - q0) <= t.flat && iabs(p2 - p0) <= t.flat && iabs(q2 - q0) <= t.flat;
        if (mask && flat) {
            const int a1 = p1, a0 = p0, b0 = q0, b1 = q1;
            p1 = (T)rnd3(p2 * 3 + a1 * 2 + a0 * 2 + b0);
            p0 = (T)rnd3(p2 + a1 * 2 + a0 * 2 + b0 * 2 + b1);
            q0 = (T)rnd3(a1 + a0 * 2 + b0 * 2 + b1 * 2 + q2);
            q1 = (T)rnd3(a0 + b0 * 2 + b1 * 2 + q2 * 3);
        } else {
            filter4(mask ? -1 : 0, hev_of(t, p1, p0, q0, q1), t.shift, p1, p0, q0, q1);
        }
        s[-2 * step] = p1; s[-step] = p0; s[0] = q0; s[step] = q1;
    } else {
        const int p3 = s[-4 * step], q3 = s[3 * step];
        T p2 = s[-3 * step], p1 = s[-2 * step], p0 = s[-step], q0 = s[0], q1 = s[step], q2 = s[2 * step];
        const bool mask = iabs(p3 - p2) <= t.lim && iabs(p2 - p1) <= t.lim && iabs(p1 - p0) <= t.lim && iabs(q1 - q0) <= t.lim &&
                          iabs(q2 - q1) <= t.lim && iabs(q3 - q2) <= t.lim && outer_ok(t, p1, p0, q0, q1);
        const bool flat = iabs(p1 - p0) <= t.flat && iabs(q1 - q0) <= t.flat && iabs(p2 - p0) <= t.flat && iabs(q2 - q0) <= t.flat &&
                          iabs(p3 - p0) <= t.flat && iabs(q3 - q0) <= t.flat;
        if (TAPS == 14) {
            const int p6 = s[-7 * step], p5 = s[-6 * step], p4 = s[-5 * step];
            const int q4 = s[4 * step], q5 = s[5 * step], q6 = s[6 * step];
            const bool flat2 = iabs(p4 - p0) <= t.flat && iabs(q4 - q0) <= t.flat && iabs(p5 - p0) <= t.flat && iabs(q5 - q0) <= t.flat &&
                               iabs(p6 - p0) <= t.flat && iabs(q6 - q0) <= t.flat;
            if (mask && flat && flat2) {
                const int a2 = p2, a1 = p1, a0 = p0, b0 = q0, b1 = q1, b2 = q2;
                s[-6 * step] = (T)rnd4(p6 * 7 + p5 * 2 + p4 * 2 + p3 + a2 + a1 + a0 + b0);
                s[-5 * step] = (T)rnd4(p6 * 5 + p5 * 2 + p4 * 2 + p3 * 2 + a2 + a1 + a0 + b0 + b1);
                s[-4 * step] = (T)rnd4(p6 * 4 + p5 + p4 * 2 + p3 * 2 + a2 * 2 + a1 + a0 + b0 + b1 + b2);
                s[-3 * step] = (T)rnd4(p6 * 3 + p5 + p4 + p3 * 2 + a2 * 2 + a1 * 2 + a0 + b0 + b1 + b2 + q3);
                s[-2 * step] = (T)rnd4(p6 * 2 + p5 + p4 + p3 + a2 * 2 + a1 * 2 + a0 * 2 + b0 + b1 + b2 + q3 + q4);
                s[-step]     = (T)rnd4(p6 + p5 + p4 + p3 + a2 + a1 * 2 + a0 * 2 + b0 * 2 + b1 + b2 + q3 + q4 + q5);
                s[0]         = (T)rnd4(p5 + p4 + p3 + a2 + a1 + a0 * 2 + b0 * 2 + b1 * 2 + b2 + q3 + q4 + q5 + q6);
                s[step]      = (T)rnd4(p4 + p3 + a2 + a1 + a0 + b0 * 2 + b1 * 2 + b2 * 2 + q3 + q4 + q5 + q6 * 2);
                s[2 * step]  = (T)rnd4(p3 + a2 + a1 + a0 + b0 + b1 * 2 + b2 * 2 + q3 * 2 + q4 + q5 + q6 * 3);
                s[3 * step]  = (T)rnd4(a2 + a1 + a0 + b0 + b1 + b2 * 2 + q3 * 2 + q4 * 2 + q5 + q6 * 4);
                s[4 * step]  = (T)rnd4(a1 + a0 + b0 + b1 + b2 + q3 * 2 + q4 * 2 + q5 * 2 + q6 * 5);
                s[5 * step]  = (T)rnd4(a0 + b0 + b1 + b2 + q3 + q4 * 2 + q5 * 2 + q6 * 7);
                return;
            }
        }
        if (mask && flat) {
            const int a2 = p2, a1 = p1, a0 = p0, b0 = q0, b1 = q1, b2 = q2;
            p2 = (T)rnd3(p3 + p3 + p3 + 2 * a2 + a1 + a0 + b0);
            p1 = (T)rnd3(p3 + p3 + a2 + 2 * a1 + a0 + b0 + b1);
            p0 = (T)rnd3(p3 + a2 + a1 + 2 * a0 + b0 + b1 + b2);
            q0 = (T)rnd3(a2 + a1 + a0 + 2 * b0 + b1 + b2 + q3);
            q1 = (T)rnd3(a1 + a0 + b0 + 2 * b1 + b2 + q3 + q3);
            q2 = (T)rnd3(a0 + b0 + b1 + 2 * b2 + q3 + q3 + q3);
        } else {
            filter4(mask ? -1 : 0, hev_of(t, p1, p0, q0, q1), t.shift, p1, p0, q0, q1);
        }
        s[-3 * step] = p2; s[-2 * step] = p1; s[-step] = p0; s[0] = q0; s[step] = q1; s[2 * step] = q2;
    }
}

}  // namespace dlf
}  // namespace b200
