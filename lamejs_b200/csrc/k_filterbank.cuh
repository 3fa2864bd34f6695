/* k_filterbank.cuh -- K1a: 32-band polyphase analysis, K1b: MDCT + alias reduction.
 *
 * Replaces lamejs NewMDCT.mdct_sub48 (reference src/js/NewMDCT.js:1053-1161) with its callees
 * window_subband (:534-914), mdct_long (:981-1051), mdct_short (:927-979).
 *
 * Parallel decomposition (DESIGN.md K1):
 *   k_subband_analysis (needs PCM only; runs beside the psy analysis / under the per-stream scan)
 *     phase 0  stage the block's PCM span in shared memory as double holding the scaled float32 value (coalesced
 *              Int16 loads; the f32->f64 widening each of the 16 taps per sample would need is paid once -- the
 *              first profile showed the conversion (XU) pipe, not FP64, as the busiest unit; one pad word per 32
 *              samples so that the stride-32 window taps hit distinct banks)
 *     phase 1  one thread per (granule slab, time slot): a full window_subband -- 512-tap folded window in
 *              double, 32-point butterfly network in registers -- writes 32 subband samples; slabs go to HBM
 *              (lamejs keeps them in gfc.sb_sample: the MDCT overlaps each granule with its predecessor)
 *   k_mdct (needs the block types)
 *     phase 2  one thread per (granule, subband): block-type windowing + 36->18 / 3x(12->6) MDCT
 *     phase 3  alias-reduction butterflies across subband boundaries, then coalesced store of xr
 * Every arithmetic statement keeps the reference's operand order; doubles with float32 store points.
 */
#ifndef MP3B200_K_FILTERBANK_CUH
#define MP3B200_K_FILTERBANK_CUH
#include "mp3_device.cuh"

#define FB_G 8                                   /* granules per block */
#define FB_SPAN (576 * FB_G + 1055)              /* PCM samples a block touches */
#define FB_PCM_WORDS (FB_SPAN + (FB_SPAN >> 5) + 2)   /* doubles: Int16 -> scaled float32 -> double is converted ONCE */
#define FB_SLAB_STRIDE 33
#define FB_THREADS 192

__constant__ double c_enwindow[285];
__constant__ double c_mdct_win[4 * 36];
__constant__ int c_sb_order[32];

#define EW(i) c_enwindow[(i)]
#define MWIN(t, i) c_mdct_win[(t) * 36 + (i)]
#define WS(i) c_mdct_win[2 * 36 + (i)]
#define SQRT2_D 1.41421356237309504880

__device__ __forceinline__ int fb_pad(int i) { return i + (i >> 5); }

/* x: padded shared PCM; p0 = index (unpadded) of the reference's x1[x1Pos]. a[] = 32 float32 results. */
__device__ __forceinline__ void window_subband_dev(const double* __restrict__ x, int p0, f32s* a) {
#define X1(o) (x[fb_pad(x1p + (o))])
#define X2(o) (x[fb_pad(x2p + (o))])
  int x1p = p0, x2p = p0 + 238 - 14 - 286;
#pragma unroll
  for (int i = -15; i < 0; i++) {
    const int wp = 10 + 18 * (i + 15);
    double w, s, t;
    w = EW(wp + -10); s = X2(-224) * w; t = X1(224) * w;
    w = EW(wp + -9); s += X2(-160) * w; t += X1(160) * w;
    w = EW(wp + -8); s += X2(-96) * w; t += X1(96) * w;
    w = EW(wp + -7); s += X2(-32) * w; t += X1(32) * w;
    w = EW(wp + -6); s += X2(32) * w; t += X1(-32) * w;
    w = EW(wp + -5); s += X2(96) * w; t += X1(-96) * w;
    w = EW(wp + -4); s += X2(160) * w; t += X1(-160) * w;
    w = EW(wp + -3); s += X2(224) * w; t += X1(-224) * w;

    w = EW(wp + -2); s += X1(-256) * w; t -= X2(256) * w;
    w = EW(wp + -1); s += X1(-192) * w; t -= X2(192) * w;
    w = EW(wp + 0); s += X1(-128) * w; t -= X2(128) * w;
    w = EW(wp + 1); s += X1(-64) * w; t -= X2(64) * w;
    w = EW(wp + 2); s += X1(0) * w; t -= X2(0) * w;
    w = EW(wp + 3); s += X1(64) * w; t -= X2(-64) * w;
    w = EW(wp + 4); s += X1(128) * w; t -= X2(-128) * w;
    w = EW(wp + 5); s += X1(192) * w; t -= X2(-192) * w;

    s *= EW(wp + 6);
    w = t - s;
    a[30 + i * 2] = t + s;
    a[31 + i * 2] = EW(wp + 7) * w;
    x1p--;
    x2p++;
  }
  const int wp = 10 + 18 * 15;
  {
    double s, t, u, v;
    t = X1(-16) * EW(wp + -10);
    s = X1(-32) * EW(wp + -2);
    t += (X1(-48) - X1(16)) * EW(wp + -9);
    s += X1(-96) * EW(wp + -1);
    t += (X1(-80) + X1(48)) * EW(wp + -8);
    s += X1(-160) * EW(wp + 0);
    t += (X1(-112) - X1(80)) * EW(wp + -7);
    s += X1(-224) * EW(wp + 1);
    t += (X1(-144) + X1(112)) * EW(wp + -6);
    s -= X1(32) * EW(wp + 2);
    t += (X1(-176) - X1(144)) * EW(wp + -5);
    s -= X1(96) * EW(wp + 3);
    t += (X1(-208) + X1(176)) * EW(wp + -4);
    s -= X1(160) * EW(wp + 4);
    t += (X1(-240) - X1(208)) * EW(wp + -3);
    s -= X1(224);
    u = s - t;
    v = s + t;
    t = a[14];
    s = a[15] - t;
    a[31] = v + t;
    a[30] = u + s;
    a[15] = u - s;
    a[14] = v - t;
  }
#undef X1
#undef X2
  {
    /* Statements of the form a[i] = a[j] +- a[k] (one addition of two float32 values, rounded to float32) are done in
     * float32: rounding the exact sum to 53 and then to 24 bits equals rounding it to 24 bits directly (53 >= 2 * 24 + 2),
     * so the result is the reference's, without two widenings, a double addition and a narrowing.  Everything that chains two
     * operations in double before the store stays in double. */
    double xr;
    float xf;
    xr = a[28] - a[0]; a[0].v = __fadd_rn(a[0].v, a[28].v); a[28] = xr * EW(wp + -2 * 18 + 7);
    xr = a[29] - a[1]; a[1].v = __fadd_rn(a[1].v, a[29].v); a[29] = xr * EW(wp + -2 * 18 + 7);
    xr = a[26] - a[2]; a[2].v = __fadd_rn(a[2].v, a[26].v); a[26] = xr * EW(wp + -4 * 18 + 7);
    xr = a[27] - a[3]; a[3].v = __fadd_rn(a[3].v, a[27].v); a[27] = xr * EW(wp + -4 * 18 + 7);
    xr = a[24] - a[4]; a[4].v = __fadd_rn(a[4].v, a[24].v); a[24] = xr * EW(wp + -6 * 18 + 7);
    xr = a[25] - a[5]; a[5].v = __fadd_rn(a[5].v, a[25].v); a[25] = xr * EW(wp + -6 * 18 + 7);
    xr = a[22] - a[6]; a[6].v = __fadd_rn(a[6].v, a[22].v); a[22] = xr * SQRT2_D;
    xr = a[23] - a[7]; a[7].v = __fadd_rn(a[7].v, a[23].v); a[23] = xr * SQRT2_D - a[7];
    a[7].v = __fsub_rn(a[7].v, a[6].v);
    a[22].v = __fsub_rn(a[22].v, a[7].v);
    a[23].v = __fsub_rn(a[23].v, a[22].v);
    xf = a[6].v; a[6].v = __fsub_rn(a[31].v, xf); a[31].v = __fadd_rn(a[31].v, xf);
    xf = a[7].v; a[7].v = __fsub_rn(a[30].v, xf); a[30].v = __fadd_rn(a[30].v, xf);
    xf = a[22].v; a[22].v = __fsub_rn(a[15].v, xf); a[15].v = __fadd_rn(a[15].v, xf);
    xf = a[23].v; a[23].v = __fsub_rn(a[14].v, xf); a[14].v = __fadd_rn(a[14].v, xf);
    xr = a[20] - a[8]; a[8].v = __fadd_rn(a[8].v, a[20].v); a[20] = xr * EW(wp + -10 * 18 + 7);
    xr = a[21] - a[9]; a[9].v = __fadd_rn(a[9].v, a[21].v); a[21] = xr * EW(wp + -10 * 18 + 7);
    xr = a[18] - a[10]; a[10].v = __fadd_rn(a[10].v, a[18].v); a[18] = xr * EW(wp + -12 * 18 + 7);
    xr = a[19] - a[11]; a[11].v = __fadd_rn(a[11].v, a[19].v); a[19] = xr * EW(wp + -12 * 18 + 7);
    xr = a[16] - a[12]; a[12].v = __fadd_rn(a[12].v, a[16].v); a[16] = xr * EW(wp + -14 * 18 + 7);
    xr = a[17] - a[13]; a[13].v = __fadd_rn(a[13].v, a[17].v); a[17] = xr * EW(wp + -14 * 18 + 7);
    xr = -a[20] + a[24]; a[20].v = __fadd_rn(a[20].v, a[24].v); a[24] = xr * EW(wp + -12 * 18 + 7);
    xr = -a[21] + a[25]; a[21].v = __fadd_rn(a[21].v, a[25].v); a[25] = xr * EW(wp + -12 * 18 + 7);
    xr = a[4] - a[8]; a[4].v = __fadd_rn(a[4].v, a[8].v); a[8] = xr * EW(wp + -12 * 18 + 7);
    xr = a[5] - a[9]; a[5].v = __fadd_rn(a[5].v, a[9].v); a[9] = xr * EW(wp + -12 * 18 + 7);
    xr = a[0] - a[12]; a[0].v = __fadd_rn(a[0].v, a[12].v); a[12] = xr * EW(wp + -4 * 18 + 7);
    xr = a[1] - a[13]; a[1].v = __fadd_rn(a[1].v, a[13].v); a[13] = xr * EW(wp + -4 * 18 + 7);
    xr = a[16] - a[28]; a[16].v = __fadd_rn(a[16].v, a[28].v); a[28] = xr * EW(wp + -4 * 18 + 7);
    xr = -a[17] + a[29]; a[17].v = __fadd_rn(a[17].v, a[29].v); a[29] = xr * EW(wp + -4 * 18 + 7);
    xr = SQRT2_D * (a[2] - a[10]); a[2].v = __fadd_rn(a[2].v, a[10].v); a[10] = xr;
    xr = SQRT2_D * (a[3] - a[11]); a[3].v = __fadd_rn(a[3].v, a[11].v); a[11] = xr;
    xr = SQRT2_D * (-a[18] + a[26]); a[18].v = __fadd_rn(a[18].v, a[26].v); a[26] = xr - a[18];
    xr = SQRT2_D * (-a[19] + a[27]); a[19].v = __fadd_rn(a[19].v, a[27].v); a[27] = xr - a[19];
    xf = a[2].v; a[19].v = __fsub_rn(a[19].v, a[3].v); a[3].v = __fsub_rn(a[3].v, xf); a[2].v = __fsub_rn(a[31].v, xf); a[31].v = __fadd_rn(a[31].v, xf);
    xf = a[3].v; a[11].v = __fsub_rn(a[11].v, a[19].v); a[18].v = __fsub_rn(a[18].v, xf); a[3].v = __fsub_rn(a[30].v, xf); a[30].v = __fadd_rn(a[30].v, xf);
    xf = a[18].v; a[27].v = __fsub_rn(a[27].v, a[11].v); a[19].v = __fsub_rn(a[19].v, xf); a[18].v = __fsub_rn(a[15].v, xf); a[15].v = __fadd_rn(a[15].v, xf);
    xf = a[19].v; a[10].v = __fsub_rn(a[10].v, xf); a[19].v = __fsub_rn(a[14].v, xf); a[14].v = __fadd_rn(a[14].v, xf);
    xf = a[10].v; a[11].v = __fsub_rn(a[11].v, xf); a[10].v = __fsub_rn(a[23].v, xf); a[23].v = __fadd_rn(a[23].v, xf);
    xf = a[11].v; a[26].v = __fsub_rn(a[26].v, xf); a[11].v = __fsub_rn(a[22].v, xf); a[22].v = __fadd_rn(a[22].v, xf);
    xf = a[26].v; a[27].v = __fsub_rn(a[27].v, xf); a[26].v = __fsub_rn(a[7].v, xf); a[7].v = __fadd_rn(a[7].v, xf);
    xf = a[27].v; a[27].v = __fsub_rn(a[6].v, xf); a[6].v = __fadd_rn(a[6].v, xf);
    xr = SQRT2_D * (a[0] - a[4]); a[0].v = __fadd_rn(a[0].v, a[4].v); a[4] = xr;
    xr = SQRT2_D * (a[1] - a[5]); a[1].v = __fadd_rn(a[1].v, a[5].v); a[5] = xr;
    xr = SQRT2_D * (a[16] - a[20]); a[16].v = __fadd_rn(a[16].v, a[20].v); a[20] = xr;
    xr = SQRT2_D * (a[17] - a[21]); a[17].v = __fadd_rn(a[17].v, a[21].v); a[21] = xr;
    xr = -SQRT2_D * (a[8] - a[12]); a[8].v = __fadd_rn(a[8].v, a[12].v); a[12] = xr - a[8];
    xr = -SQRT2_D * (a[9] - a[13]); a[9].v = __fadd_rn(a[9].v, a[13].v); a[13] = xr - a[9];
    xr = -SQRT2_D * (a[25] - a[29]); a[25].v = __fadd_rn(a[25].v, a[29].v); a[29] = xr - a[25];
    xr = -SQRT2_D * (a[24] + a[28]); a[24].v = __fsub_rn(a[24].v, a[28].v); a[28] = xr - a[24];
    xr = a[24] - a[16]; a[24] = xr;
    xr = a[20] - xr; a[20] = xr;
    xr = a[28] - xr; a[28] = xr;
    xr = a[25] - a[17]; a[25] = xr;
    xr = a[21] - xr; a[21] = xr;
    xr = a[29] - xr; a[29] = xr;
    xr = a[17] - a[1]; a[17] = xr;
    xr = a[9] - xr; a[9] = xr;
    xr = a[25] - xr; a[25] = xr;
    xr = a[5] - xr; a[5] = xr;
    xr = a[21] - xr; a[21] = xr;
    xr = a[13] - xr; a[13] = xr;
    xr = a[29] - xr; a[29] = xr;
    xr = a[1] - a[0]; a[1] = xr;
    xr = a[16] - xr; a[16] = xr;
    xr = a[17] - xr; a[17] = xr;
    xr = a[8] - xr; a[8] = xr;
    xr = a[9] - xr; a[9] = xr;
    xr = a[24] - xr; a[24] = xr;
    xr = a[25] - xr; a[25] = xr;
    xr = a[4] - xr; a[4] = xr;
    xr = a[5] - xr; a[5] = xr;
    xr = a[20] - xr; a[20] = xr;
    xr = a[21] - xr; a[21] = xr;
    xr = a[12] - xr; a[12] = xr;
    xr = a[13] - xr; a[13] = xr;
    xr = a[28] - xr; a[28] = xr;
    xr = a[29] - xr; a[29] = xr;
    xf = a[0].v; a[0].v = __fadd_rn(a[0].v, a[31].v); a[31].v = __fsub_rn(a[31].v, xf);
    xf = a[1].v; a[1].v = __fadd_rn(a[1].v, a[30].v); a[30].v = __fsub_rn(a[30].v, xf);
    xf = a[16].v; a[16].v = __fadd_rn(a[16].v, a[15].v); a[15].v = __fsub_rn(a[15].v, xf);
    xf = a[17].v; a[17].v = __fadd_rn(a[17].v, a[14].v); a[14].v = __fsub_rn(a[14].v, xf);
    xf = a[8].v; a[8].v = __fadd_rn(a[8].v, a[23].v); a[23].v = __fsub_rn(a[23].v, xf);
    xf = a[9].v; a[9].v = __fadd_rn(a[9].v, a[22].v); a[22].v = __fsub_rn(a[22].v, xf);
    xf = a[24].v; a[24].v = __fadd_rn(a[24].v, a[7].v); a[7].v = __fsub_rn(a[7].v, xf);
    xf = a[25].v; a[25].v = __fadd_rn(a[25].v, a[6].v); a[6].v = __fsub_rn(a[6].v, xf);
    xf = a[4].v; a[4].v = __fadd_rn(a[4].v, a[27].v); a[27].v = __fsub_rn(a[27].v, xf);
    xf = a[5].v; a[5].v = __fadd_rn(a[5].v, a[26].v); a[26].v = __fsub_rn(a[26].v, xf);
    xf = a[20].v; a[20].v = __fadd_rn(a[20].v, a[11].v); a[11].v = __fsub_rn(a[11].v, xf);
    xf = a[21].v; a[21].v = __fadd_rn(a[21].v, a[10].v); a[10].v = __fsub_rn(a[10].v, xf);
    xf = a[12].v; a[12].v = __fadd_rn(a[12].v, a[19].v); a[19].v = __fsub_rn(a[19].v, xf);
    xf = a[13].v; a[13].v = __fadd_rn(a[13].v, a[18].v); a[18].v = __fsub_rn(a[18].v, xf);
    xf = a[28].v; a[28].v = __fadd_rn(a[28].v, a[3].v); a[3].v = __fsub_rn(a[3].v, xf);
    xf = a[29].v; a[29].v = __fadd_rn(a[29].v, a[2].v); a[2].v = __fsub_rn(a[2].v, xf);
  }
}

/* 36 -> 18 MDCT (NewMDCT.js:981-1051). in: 18 float32 (work[]), out: xr row (stride 1). */
__device__ __forceinline__ void mdct_long_dev(f32s* out, const f32s* in) {
#define CX(i) WS(12 + (i))
  double ct, st;
  {
    double tc1, tc2, tc3, tc4, ts5, ts6, ts7, ts8;
    tc1 = in[17] - in[9];
    tc3 = in[15] - in[11];
    tc4 = in[14] - in[12];
    ts5 = in[0] + in[8];
    ts6 = in[1] + in[7];
    ts7 = in[2] + in[6];
    ts8 = in[3] + in[5];
    out[17] = (ts5 + ts7 - ts8) - (ts6 - in[4]);
    st = (ts5 + ts7 - ts8) * CX(7) + (ts6 - in[4]);
    ct = (tc1 - tc3 - tc4) * CX(6);
    out[5] = ct + st;
    out[6] = ct - st;
    tc2 = (in[16] - in[10]) * CX(6);
    ts6 = ts6 * CX(7) + in[4];
    ct = tc1 * CX(0) + tc2 + tc3 * CX(1) + tc4 * CX(2);
    st = -ts5 * CX(4) + ts6 - ts7 * CX(5) + ts8 * CX(3);
    out[1] = ct + st;
    out[2] = ct - st;
    ct = tc1 * CX(1) - tc2 - tc3 * CX(2) + tc4 * CX(0);
    st = -ts5 * CX(5) + ts6 - ts7 * CX(3) + ts8 * CX(4);
    out[9] = ct + st;
    out[10] = ct - st;
    ct = tc1 * CX(2) - tc2 + tc3 * CX(0) - tc4 * CX(1);
    st = ts5 * CX(3) - ts6 + ts7 * CX(4) - ts8 * CX(5);
    out[13] = ct + st;
    out[14] = ct - st;
  }
  {
    double ts1, ts2, ts3, ts4, tc5, tc6, tc7, tc8;
    ts1 = in[8] - in[0];
    ts3 = in[6] - in[2];
    ts4 = in[5] - in[3];
    tc5 = in[17] + in[9];
    tc6 = in[16] + in[10];
    tc7 = in[15] + in[11];
    tc8 = in[14] + in[12];
    out[0] = (tc5 + tc7 + tc8) + (tc6 + in[13]);
    ct = (tc5 + tc7 + tc8) * CX(7) - (tc6 + in[13]);
    st = (ts1 - ts3 + ts4) * CX(6);
    out[11] = ct + st;
    out[12] = ct - st;
    ts2 = (in[7] - in[1]) * CX(6);
    tc6 = in[13] - tc6 * CX(7);
    ct = tc5 * CX(3) - tc6 + tc7 * CX(4) + tc8 * CX(5);
    st = ts1 * CX(2) + ts2 + ts3 * CX(0) + ts4 * CX(1);
    out[3] = ct + st;
    out[4] = ct - st;
    ct = -tc5 * CX(5) + tc6 - tc7 * CX(3) - tc8 * CX(4);
    st = ts1 * CX(1) + ts2 - ts3 * CX(2) - ts4 * CX(0);
    out[7] = ct + st;
    out[8] = ct - st;
    ct = -tc5 * CX(4) + tc6 - tc7 * CX(5) - tc8 * CX(3);
    st = ts1 * CX(0) - ts2 + ts3 * CX(1) - ts4 * CX(2);
    out[15] = ct + st;
    out[16] = ct - st;
  }
#undef CX
}

/* 3 x (12 -> 6) MDCT in place on 18 float32 (NewMDCT.js:927-979) */
__device__ __forceinline__ void mdct_short_dev(f32s* io) {
#pragma unroll
  for (int l = 0; l < 3; l++) {
    double tc0, tc1, tc2, ts0, ts1, ts2;
    ts0 = io[l + 2 * 3] * WS(0) - io[l + 5 * 3];
    tc0 = io[l + 0 * 3] * WS(2) - io[l + 3 * 3];
    tc1 = ts0 + tc0;
    tc2 = ts0 - tc0;
    ts0 = io[l + 5 * 3] * WS(0) + io[l + 2 * 3];
    tc0 = io[l + 3 * 3] * WS(2) + io[l + 0 * 3];
    ts1 = ts0 + tc0;
    ts2 = -ts0 + tc0;
    tc0 = (io[l + 1 * 3] * WS(1) - io[l + 4 * 3]) * 2.069978111953089e-11;
    ts0 = (io[l + 4 * 3] * WS(1) + io[l + 1 * 3]) * 2.069978111953089e-11;
    io[l + 3 * 0] = tc1 * 1.907525191737280e-11 + tc0;
    io[l + 3 * 5] = -ts1 * 1.907525191737280e-11 + ts0;
    tc2 = tc2 * 0.86602540378443870761 * 1.907525191737281e-11;
    ts1 = ts1 * 0.5 * 1.907525191737281e-11 + ts0;
    io[l + 3 * 1] = tc2 - ts1;
    io[l + 3 * 2] = tc2 + ts1;
    tc1 = tc1 * 0.5 * 1.907525191737281e-11 - tc0;
    ts2 = ts2 * 0.86602540378443870761 * 1.907525191737281e-11;
    io[l + 3 * 3] = tc1 + ts2;
    io[l + 3 * 4] = tc1 - ts2;
  }
}

/* ---- K1a: polyphase analysis of FB_SLABS granules per block -> subband slabs in HBM ----
 * A slab (18 time slots x 32 subbands, float32: lamejs gfc.sb_sample) depends on PCM only, so this kernel is launched at
 * the start of the pipeline on a side stream: its blocks fill the SMs the psy analysis has left and the whole machine while the
 * per-stream scan (one block per stream) decides the block types.  Slab rows use the psy row numbering (one leading row per
 * stream for granule -1, the MDCT overlap of the first granule): row = unit_base + z + u + 1.
 * grid: (ceil((max_granules + 1) / FB_SLABS), nch, nstreams); block: FB_THREADS. */
#ifndef FB_MIN_BLOCKS
#define FB_MIN_BLOCKS 3
#endif
#define FB_SLABS (FB_G + 1)
template <bool F32_PCM>     /* as k_psy_analysis: Float32 samples of the resampler instead of Int16 input */
__global__ void __launch_bounds__(FB_THREADS, FB_MIN_BLOCKS)
k_subband_analysis(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, float* __restrict__ slab_out) {
  const int z = blockIdx.z;
  const StreamDesc& sd = streams[z];
  const int ch = blockIdx.y;
  const int ngr = sd.nframes * T->mode_gr;
  const int u0 = (int)blockIdx.x * FB_SLABS - 1;    /* first granule (relative to frame0) of this block, -1 = overlap row */
  if (u0 >= ngr) return;
  const int scount = min(FB_SLABS, ngr - u0);
  const long long cs = (long long)T->mode_gr * sd.frame0 + u0;   /* absolute granule index of slab 0 */
  const int nch = T->nch;

  extern __shared__ double smem_d[];
  double* pcm = smem_d;                             /* FB_PCM_WORDS doubles */
  f32s* slab = reinterpret_cast<f32s*>(smem_d + FB_PCM_WORDS);   /* [FB_SLABS][18][33] */
  __shared__ float s_amp[32];                       /* amp_filter by subband-array position */

  const int tid = threadIdx.x;
  /* ---- phase 0: stage PCM.  sample j of the span is stream sample lo + j; slab s, time slot j has its window origin
   * (reference wkPos) at stream sample 576 (cs + s) - 242 + 32 j = span index 576 s + 286 + 32 j ---- */
  const long long lo = 576 * (cs + 1) - 1104;
  const int scale_applied = T->scale_applied;
  const double scale = T->scale;
  const int span = 576 * (scount - 1) + 1055;
  {
    /* 8 independent loads per thread in flight (one dependent load per iteration left this phase, a third of the
     * kernel's samples in the round-2 profile, waiting for HBM latency) */
    using Sample = pcm_sample_t<F32_PCM>;
    const Sample* __restrict__ pbuf = static_cast<const Sample*>(sd.pcm[ch]);
    const long long pbase = sd.pcm_base, pend = sd.pcm_end;
#pragma unroll 1
    for (int j0 = tid; j0 < span; j0 += FB_THREADS * 8) {
      Sample v[8];
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int j = j0 + k * FB_THREADS;
        const long long i = lo + j;
        v[k] = (j < span && i >= 0 && i < pend) ? __ldg(&pbuf[i - pbase]) : (Sample)0;
      }
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int j = j0 + k * FB_THREADS;
        if (j < span) pcm[fb_pad(j)] = pcm_value(v[k], scale_applied, scale);
      }
    }
  }
  if (tid < 32) s_amp[c_sb_order[tid]] = T->amp_filter[tid];
  __syncthreads();

  /* ---- phase 1: subband analysis, thread = (slab, time slot) ---- */
  for (int w = tid; w < scount * 18; w += FB_THREADS) {
    const int s = w / 18, j = w - s * 18;
    f32s a[32];
    window_subband_dev(pcm, 576 * s + 286 + 32 * j, a);
    f32s* row = slab + (s * 18 + j) * FB_SLAB_STRIDE;
#pragma unroll
    for (int p = 0; p < 32; p++) {
      double v = a[p];
      if ((j & 1) && (p & 1)) v = v * -1;            /* NewMDCT.js:1074-1076 */
      const float amp = s_amp[p];
      f32s r; r = v;
      if ((double)amp < 1.0 && !((double)amp < 1e-12)) r *= (double)amp;   /* NewMDCT.js:1093-1096 (applied once per slab) */
      row[p] = r;
    }
  }
  __syncthreads();
  /* coalesced store: slab rows are 576 consecutive floats [slot][subband] */
  float* const dst = slab_out + (((size_t)sd.unit_base + z + u0 + 1) * nch + ch) * 576;
  for (int w = tid; w < scount * 576; w += FB_THREADS) {
    const int s = w / 576, r = w - s * 576;
    dst[(size_t)s * nch * 576 + r] = slab[(s * 18 + (r >> 5)) * FB_SLAB_STRIDE + (r & 31)].v;
  }
}

/* ---- K1b: block-type windowing + MDCT + alias reduction from the slabs (needs the block types, i.e. the scan) ----
 * thread = (granule, subband); a warp reads one 128-byte line of the previous and of the current slab per time slot.
 * grid: (ceil(max_granules / FB_G), nch, nstreams); block: FB_G * 32.
 * blocktype: int8 [granule row][2]; xr_out: float [granule row][nch][576]. */
__global__ void __launch_bounds__(FB_G * 32)
k_mdct(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, const float* __restrict__ slab_in,
       const signed char* __restrict__ blocktype, float* __restrict__ xr_out) {
  const int z = blockIdx.z;
  const StreamDesc& sd = streams[z];
  const int ch = blockIdx.y;
  const int ngr = sd.nframes * T->mode_gr;
  const int g0 = blockIdx.x * FB_G;                 /* first granule (relative to frame0) of this block */
  if (g0 >= ngr) return;
  const int gcount = min(FB_G, ngr - g0);
  const int nch = T->nch;
  __shared__ f32s xr[FB_G * 576];
  __shared__ float s_amp[32];
  __shared__ int s_bt[FB_G];
  const int tid = threadIdx.x;
  if (tid < 32) s_amp[c_sb_order[tid]] = T->amp_filter[tid];
  if (tid < gcount) s_bt[tid] = blocktype[(size_t)(sd.unit_base + g0 + tid) * 2 + ch];
  __syncthreads();

  /* ---- windowing + MDCT ---- */
  {
    const int g = tid >> 5, band = tid & 31;
    if (g < gcount) {
      const int type = s_bt[g];
      const int ob = c_sb_order[band];
      f32s* o = xr + g * 576 + band * 18;
      if ((double)s_amp[ob] < 1e-12) {
#pragma unroll
        for (int k = 0; k < 18; k++) o[k] = 0.0;
      } else {
        /* slab row of granule g0 + g - 1 (previous) and g0 + g (current): rows unit_base + z + (g0 + g), + 1 */
        const float* p0 = slab_in + (((size_t)sd.unit_base + z + g0 + g) * nch + ch) * 576 + ob;
        const float* p1 = p0 + (size_t)nch * 576;
        float b0[18], b1[18];
#pragma unroll
        for (int k = 0; k < 18; k++) { b0[k] = __ldg(p0 + 32 * k); b1[k] = __ldg(p1 + 32 * k); }   /* 36 loads in flight */
#define B0(k) ((double)b0[(k)])
#define B1(k) ((double)b1[(k)])
        if (type == BT_SHORT) {
          f32s io[18];
#pragma unroll
          for (int k = -3; k < 0; k++) {                 /* NewMDCT.js:1098-1112, static indices after unrolling */
            const double wv = WS(k + 3);
            io[k * 3 + 9] = B0(9 + k) * wv - B0(8 - k);
            io[k * 3 + 18] = B0(14 - k) * wv + B0(15 + k);
            io[k * 3 + 10] = B0(15 + k) * wv - B0(14 - k);
            io[k * 3 + 19] = B1(2 - k) * wv + B1(3 + k);
            io[k * 3 + 11] = B1(3 + k) * wv - B1(2 - k);
            io[k * 3 + 20] = B1(8 - k) * wv + B1(9 + k);
          }
          mdct_short_dev(io);
#pragma unroll
          for (int k = 0; k < 18; k++) o[k] = (double)io[k];
        } else {
          f32s work[18];
#pragma unroll
          for (int k = -9; k < 0; k++) {
            double a, b;
            a = MWIN(type, k + 27) * B1(k + 9) + MWIN(type, k + 36) * B1(8 - k);
            b = MWIN(type, k + 9) * B0(k + 9) - MWIN(type, k + 18) * B0(8 - k);
            work[k + 9] = a - b * WS(3 + k + 9);
            work[k + 18] = a * WS(3 + k + 9) + b;
          }
          mdct_long_dev(o, work);
        }
#undef B0
#undef B1
      }
    }
  }
  __syncthreads();

  /* ---- alias reduction (NewMDCT.js:1133-1154): boundary `band` couples lines 18*band-1-k, 18*band+k ---- */
  for (int w = tid; w < gcount * 31 * 8; w += FB_G * 32) {
    const int g = w / 248, r = w - g * 248;
    const int band = 1 + (r >> 3), k = r & 7;
    if (s_bt[g] == BT_SHORT) continue;
    f32s* e = xr + g * 576 + band * 18;
    const double lo_v = e[-1 - k], hi_v = e[k];
    const double bu = hi_v * WS(20 + k) + lo_v * WS(28 + k);
    const double bd = hi_v * WS(28 + k) - lo_v * WS(20 + k);
    e[-1 - k] = bu;
    e[k] = bd;
  }
  __syncthreads();
  for (int w = tid; w < gcount * 576; w += FB_G * 32) {
    const int g = w / 576, i = w - g * 576;
    xr_out[((size_t)(sd.unit_base + g0 + g) * nch + ch) * 576 + i] = xr[w].v;
  }
}

#endif
