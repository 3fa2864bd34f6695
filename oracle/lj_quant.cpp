/* lj_quant.cpp -- bit allocation, noise shaping, quantizer and Huffman bit counting of the
 * oracle.  TEST INFRASTRUCTURE.  Follows, statement by statement:
 *   src/js/CBRNewIterationLoop.js:25-90   iteration_loop
 *   src/js/Reservoir.js:77-294            ResvFrameBegin / ResvMaxBits / ResvAdjust / ResvFrameEnd
 *   src/js/QuantizePVT.js:229-414         ATHmdct, compute_ath, iteration_init
 *   src/js/QuantizePVT.js:421-484         on_pe
 *   src/js/QuantizePVT.js:541-878         athAdjust, calc_xmin, calc_noise_core, calc_noise
 *   src/js/Quantize.js:92-381             init_xrpow, psfb21_analogsilence, init_outer_loop, bin_search_StepSize
 *   src/js/Quantize.js:447-1078           loop_break, quant_compare, amp_scalefac_bands, inc_scalefac_scale,
 *                                         inc_subblock_gain, balance_noise, outer_loop, iteration_finish_one
 *   src/js/Takehiro.js:102-1172           quantize_*, ix_max, count_bit_*, choose_table, noquant_count_bits,
 *                                         count_bits, best_huffman_divide, scfsi_calc, best_scalefac_store,
 *                                         scale_bitcount, huffman_init
 */
#include <stdlib.h>
#include "lj_encoder.h"
#include "lj_tables.h"

static const int pretab[SBMAX_l] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 3, 2, 0};
static const double DBL_EPS = 2.2204460492503131e-016;

#define HLEN(t, i) LJ_HUFF_LEN[LJ_HUFF_OFF[(t)] + (i)]

/* ---------------------------------------------------------------- init */
static double ATHmdct(const LjEnc* e, double f) {
  double ath = lj_ATHformula(f, e);
  ath -= 100; /* NSATHSCALE */
  ath = js_pow(10.0, ath / 10.0 + e->ATHlower);
  return ath;
}

static void compute_ath(LjEnc* e) {
  double samp_freq = e->out_samplerate;
  for (int sfb = 0; sfb < SBMAX_l; sfb++) {
    int start = e->sfb_l[sfb], end = e->sfb_l[sfb + 1];
    e->ath_l[sfb] = 3.4028235e+38;
    for (int i = start; i < end; i++) {
      double freq = i * samp_freq / (2 * 576);
      double ATH_f = ATHmdct(e, freq);
      e->ath_l[sfb] = js_min(e->ath_l[sfb], ATH_f);
    }
  }
  for (int sfb = 0; sfb < PSFB21; sfb++) {
    int start = e->psfb21[sfb], end = e->psfb21[sfb + 1];
    e->ath_psfb21[sfb] = 3.4028235e+38;
    for (int i = start; i < end; i++) {
      double freq = i * samp_freq / (2 * 576);
      double ATH_f = ATHmdct(e, freq);
      e->ath_psfb21[sfb] = js_min(e->ath_psfb21[sfb], ATH_f);
    }
  }
  for (int sfb = 0; sfb < SBMAX_s; sfb++) {
    int start = e->sfb_s[sfb], end = e->sfb_s[sfb + 1];
    e->ath_s[sfb] = 3.4028235e+38;
    for (int i = start; i < end; i++) {
      double freq = i * samp_freq / (2 * 192);
      double ATH_f = ATHmdct(e, freq);
      e->ath_s[sfb] = js_min(e->ath_s[sfb], ATH_f);
    }
    e->ath_s[sfb] *= (e->sfb_s[sfb + 1] - e->sfb_s[sfb]);
  }
  for (int sfb = 0; sfb < PSFB12; sfb++) {
    int start = e->psfb12[sfb], end = e->psfb12[sfb + 1];
    e->ath_psfb12[sfb] = 3.4028235e+38;
    for (int i = start; i < end; i++) {
      double freq = i * samp_freq / (2 * 192);
      double ATH_f = ATHmdct(e, freq);
      e->ath_psfb12[sfb] = js_min(e->ath_psfb12[sfb], ATH_f);
    }
    e->ath_psfb12[sfb] *= (e->sfb_s[13] - e->sfb_s[12]);
  }
  e->ath_floor = 10. * js_log10(ATHmdct(e, -1.));
}

static void huffman_init(LjEnc* e) {
  static const int subdv_table[23][2] = {{0, 0}, {0, 0}, {0, 0}, {0, 0}, {0, 0}, {0, 1}, {1, 1}, {1, 1}, {1, 2}, {2, 2},
    {2, 3}, {2, 3}, {3, 4}, {3, 4}, {3, 4}, {4, 5}, {4, 5}, {4, 6}, {5, 6}, {5, 6}, {5, 7}, {6, 7}, {6, 7}};
  for (int i = 2; i <= 576; i += 2) {
    int scfb_anz = 0, bv_index;
    while (e->sfb_l[++scfb_anz] < i)
      ;
    bv_index = subdv_table[scfb_anz][0];
    while (e->sfb_l[bv_index + 1] > i) bv_index--;
    if (bv_index < 0) bv_index = subdv_table[scfb_anz][0];
    e->bv_scf[i - 2] = bv_index;
    bv_index = subdv_table[scfb_anz][1];
    while (e->sfb_l[bv_index + e->bv_scf[i - 2] + 2] > i) bv_index--;
    if (bv_index < 0) bv_index = subdv_table[scfb_anz][1];
    e->bv_scf[i - 1] = bv_index;
  }
}

void lj_iteration_init(LjEnc* e) {
  int i;
  e->main_data_begin = 0;
  compute_ath(e);
  e->pow43[0] = 0.0;
  for (i = 1; i < PRECALC_SIZE; i++) e->pow43[i] = js_pow(i, 4.0 / 3.0);
  for (i = 0; i < PRECALC_SIZE - 1; i++) e->adj43[i] = ((i + 1) - js_pow(0.5 * (e->pow43[i] + e->pow43[i + 1]), 0.75));
  e->adj43[i] = 0.5;
  for (i = 0; i < Q_MAX; i++) e->ipow20[i] = js_pow(2.0, (i - 210) * -0.1875);
  for (i = 0; i <= Q_MAX + Q_MAX2; i++) e->pow20[i] = js_pow(2.0, (i - 210 - Q_MAX2) * 0.25);
  huffman_init(e);
  {
    double bass, alto, treble, sfb21;
    i = (e->exp_nspsytune >> 2) & 63; if (i >= 32) i -= 64;
    bass = js_pow(10, i / 4.0 / 10.0);
    i = (e->exp_nspsytune >> 8) & 63; if (i >= 32) i -= 64;
    alto = js_pow(10, i / 4.0 / 10.0);
    i = (e->exp_nspsytune >> 14) & 63; if (i >= 32) i -= 64;
    treble = js_pow(10, i / 4.0 / 10.0);
    i = (e->exp_nspsytune >> 20) & 63; if (i >= 32) i -= 64;
    sfb21 = treble * js_pow(10, i / 4.0 / 10.0);
    for (i = 0; i < SBMAX_l; i++) {
      double f;
      if (i <= 6) f = bass; else if (i <= 13) f = alto; else if (i <= 20) f = treble; else f = sfb21;
      e->longfact[i] = f;
    }
    for (i = 0; i < SBMAX_s; i++) {
      double f;
      if (i <= 5) f = bass; else if (i <= 10) f = alto; else if (i <= 11) f = treble; else f = sfb21;
      e->shortfact[i] = f;
    }
  }
}

/* ---------------------------------------------------------------- reservoir */
static double ResvFrameBegin(LjEnc* e) {
  int frameLength = lj_getframebits(e);
  double mean_bits = (frameLength - e->sideinfo_len * 8) / (double)e->mode_gr;
  const int resvLimit = (8 * 256) * e->mode_gr - 8;        /* main_data_begin has 9 bits in MPEG-1, 8 in MPEG-2 */
  const int maxmp3buf = 8 * 1440;                          /* brate <= 320, !strict_ISO (Reservoir.js:129-152) */
  e->ResvMax = maxmp3buf - frameLength;
  if (e->ResvMax > resvLimit) e->ResvMax = resvLimit;
  if (e->ResvMax < 0 || e->disable_reservoir) e->ResvMax = 0;
  e->resvDrain_pre = 0;
  return mean_bits;
}

/* returns extra_bits; *targ = targ_bits.bits */
static double ResvMaxBits(LjEnc* e, double mean_bits, double* targ, int cbr) {
  double add_bits;
  double ResvSize = e->ResvSize, ResvMax = e->ResvMax;
  if (cbr != 0) ResvSize += mean_bits;
  if ((e->substep_shaping & 1) != 0) ResvMax *= 0.9;
  *targ = mean_bits;
  if (ResvSize * 10 > ResvMax * 9) {
    add_bits = ResvSize - (ResvMax * 9) / 10;
    *targ += add_bits;
    e->substep_shaping |= 0x80;
  } else {
    add_bits = 0;
    e->substep_shaping &= 0x7f;
    if (!e->disable_reservoir && 0 == (e->substep_shaping & 1)) *targ -= .1 * mean_bits;   /* build the reservoir up */
  }
  double extra_bits = (ResvSize < (e->ResvMax * 6) / 10.0 ? ResvSize : (e->ResvMax * 6) / 10.0);
  extra_bits -= add_bits;
  if (extra_bits < 0) extra_bits = 0;
  return extra_bits;
}

static void ResvFrameEnd(LjEnc* e, double mean_bits) {
  double over_bits;
  e->ResvSize += mean_bits * e->mode_gr;
  double stuffingBits = 0;
  e->resvDrain_post = 0;
  e->resvDrain_pre = 0;
  if ((over_bits = fmod(e->ResvSize, 8)) != 0) stuffingBits += over_bits;
  over_bits = (e->ResvSize - stuffingBits) - e->ResvMax;
  if (over_bits > 0) stuffingBits += over_bits;
  {
    /* Math.min(...) / 8 on JS numbers: not an integer division (Java's is), so main_data_begin can hold eighths */
    double mdb_bytes = js_min(e->main_data_begin * 8, stuffingBits) / 8;
    if (e->java_int_div) mdb_bytes = floor(mdb_bytes);     /* Reservoir.java: `int mdb_bytes = Math.min(...) / 8` */
    e->resvDrain_pre += 8 * mdb_bytes;
    stuffingBits -= 8 * mdb_bytes;
    e->ResvSize -= 8 * mdb_bytes;
    e->main_data_begin -= mdb_bytes;
  }
  e->resvDrain_post += stuffingBits;
  e->ResvSize -= stuffingBits;
}

/* QuantizePVT.js:421-484.  targ_bits / add_bits are Int32Arrays: every store truncates. */
static double on_pe(LjEnc* e, double pe[2][2], int* targ_bits, double mean_bits, int gr, int cbr) {
  double tbits = 0, bits;
  int add_bits[2] = {0, 0};
  int ch;
  double extra_bits = ResvMaxBits(e, mean_bits, &tbits, cbr);
  double max_bits = tbits + extra_bits;
  if (max_bits > MAX_BITS_PER_GRANULE) max_bits = MAX_BITS_PER_GRANULE;
  for (bits = 0, ch = 0; ch < e->channels_out; ++ch) {
    targ_bits[ch] = js_toint32(js_min(MAX_BITS_PER_CHANNEL, tbits / e->channels_out));
    add_bits[ch] = js_toint32(targ_bits[ch] * pe[gr][ch] / 700.0 - targ_bits[ch]);
    if (add_bits[ch] > mean_bits * 3 / 4) add_bits[ch] = js_toint32(mean_bits * 3 / 4);
    if (add_bits[ch] < 0) add_bits[ch] = 0;
    if (add_bits[ch] + targ_bits[ch] > MAX_BITS_PER_CHANNEL)
      add_bits[ch] = js_toint32(js_max(0, MAX_BITS_PER_CHANNEL - targ_bits[ch]));
    bits += add_bits[ch];
  }
  if (bits > extra_bits) {
    for (ch = 0; ch < e->channels_out; ++ch) add_bits[ch] = js_toint32(extra_bits * add_bits[ch] / bits);
  }
  for (ch = 0; ch < e->channels_out; ++ch) {
    targ_bits[ch] += add_bits[ch];
    extra_bits -= add_bits[ch];
  }
  for (bits = 0, ch = 0; ch < e->channels_out; ++ch) bits += targ_bits[ch];
  if (bits > MAX_BITS_PER_GRANULE) {
    for (ch = 0; ch < e->channels_out; ++ch) {
      targ_bits[ch] = js_toint32((double)targ_bits[ch] * MAX_BITS_PER_GRANULE); /* *= stores (Int32) */
      targ_bits[ch] = js_toint32((double)targ_bits[ch] / bits);
    }
  }
  return max_bits;                 /* a JS number: fractional when the reservoir build-up rule took a tenth of mean_bits */
}

/* ---------------------------------------------------------------- xmin / noise */
static double athAdjust(double a, double x, double athFloor) {
  double o = 90.30873362;
  double p = 94.82444863;
  double u = js_log10(x) * 10.0;
  double v = a * a;
  double w = 0.0;
  u -= athFloor;
  if (v > 1E-20) w = 1. + js_log10(v) * (10.0 / o);
  if (w < 0) w = 0.;
  u *= w;
  u += athFloor + o - p;
  return js_pow(10., 0.1 * u);
}

static int calc_xmin(LjEnc* e, const PsyRatio* ratio, GrInfo* cod_info, F32* pxmin) {
  int pxminPos = 0;
  int gsfb, j = 0, ath_over = 0;
  const F32* xr = cod_info->xr;
  double masking_lower = e->masking_lower;

  for (gsfb = 0; gsfb < cod_info->psy_lmax; gsfb++) {
    double en0, xmin, rh1, rh2;
    int width, l;
    xmin = e->ath_adjust * e->ath_l[gsfb];
    width = cod_info->width[gsfb];
    rh1 = xmin / width;
    rh2 = DBL_EPS;
    l = width >> 1;
    en0 = 0.0;
    do {
      double xa, xb;
      xa = xr[j] * xr[j]; en0 += xa; rh2 += (xa < rh1) ? xa : rh1; j++;
      xb = xr[j] * xr[j]; en0 += xb; rh2 += (xb < rh1) ? xb : rh1; j++;
    } while (--l > 0);
    if (en0 > xmin) ath_over++;
    if (gsfb == SBPSY_l) {
      double x = xmin * e->longfact[gsfb];
      if (rh2 < x) rh2 = x;
    }
    {
      double en = ratio->en.l[gsfb];
      if (en > 0.0) {
        double x = en0 * ratio->thm.l[gsfb] * masking_lower / en;
        if (xmin < x) xmin = x;
      }
    }
    pxmin[pxminPos++] = xmin * e->longfact[gsfb];
  }
  int max_nonzero = 575;
  if (cod_info->block_type != SHORT_TYPE) {
    int k = 576;
    while (k-- != 0 && bs_EQ(xr[k], 0)) max_nonzero = k;
  }
  cod_info->max_nonzero_coeff = max_nonzero;

  for (int sfb = cod_info->sfb_smin; gsfb < cod_info->psymax; sfb++, gsfb += 3) {
    int width, b;
    double tmpATH = e->ath_adjust * e->ath_s[sfb];
    width = cod_info->width[gsfb];
    for (b = 0; b < 3; b++) {
      double en0 = 0.0, xmin, rh1, rh2;
      int l = width >> 1;
      rh1 = tmpATH / width;
      rh2 = DBL_EPS;
      do {
        double xa, xb;
        xa = xr[j] * xr[j]; en0 += xa; rh2 += (xa < rh1) ? xa : rh1; j++;
        xb = xr[j] * xr[j]; en0 += xb; rh2 += (xb < rh1) ? xb : rh1; j++;
      } while (--l > 0);
      if (en0 > tmpATH) ath_over++;
      if (sfb == SBPSY_s) {
        double x = tmpATH * e->shortfact[sfb];
        if (rh2 < x) rh2 = x;
      }
      xmin = tmpATH;
      {
        double en = ratio->en.s[sfb][b];
        if (en > 0.0) {
          double x = en0 * ratio->thm.s[sfb][b] * masking_lower / en;
          if (xmin < x) xmin = x;
        }
      }
      pxmin[pxminPos++] = xmin * e->shortfact[sfb];
    }
    if (e->useTemporal) {
      if (pxmin[pxminPos - 3] > pxmin[pxminPos - 3 + 1])
        pxmin[pxminPos - 3 + 1] += (pxmin[pxminPos - 3] - pxmin[pxminPos - 3 + 1]) * e->decay;
      if (pxmin[pxminPos - 3 + 1] > pxmin[pxminPos - 3 + 2])
        pxmin[pxminPos - 3 + 2] += (pxmin[pxminPos - 3 + 1] - pxmin[pxminPos - 3 + 2]) * e->decay;
    }
  }
  return ath_over;
}

static double calc_noise_core(const LjEnc* e, const GrInfo* cod_info, int* startline, int l, double step) {
  double noise = 0;
  int j = *startline;
  const int* ix = cod_info->l3_enc;
  if (j > cod_info->count1) {
    while ((l--) != 0) {
      double temp;
      temp = cod_info->xr[j]; j++; noise += temp * temp;
      temp = cod_info->xr[j]; j++; noise += temp * temp;
    }
  } else if (j > cod_info->big_values) {
    F32 ix01[2];
    ix01[0] = 0;
    ix01[1] = step;
    while ((l--) != 0) {
      double temp;
      temp = fabs(cod_info->xr[j]) - ix01[ix[j]]; j++; noise += temp * temp;
      temp = fabs(cod_info->xr[j]) - ix01[ix[j]]; j++; noise += temp * temp;
    }
  } else {
    while ((l--) != 0) {
      double temp;
      temp = fabs(cod_info->xr[j]) - e->pow43[ix[j]] * step; j++; noise += temp * temp;
      temp = fabs(cod_info->xr[j]) - e->pow43[ix[j]] * step; j++; noise += temp * temp;
    }
  }
  *startline = j;
  return noise;
}

static int calc_noise(const LjEnc* e, const GrInfo* cod_info, const F32* l3_xmin, F32* distort, CalcNoiseResult* res,
                      CalcNoiseData* prev_noise) {
  int distortPos = 0, l3_xminPos = 0;
  int sfb, l, over = 0;
  double over_noise_db = 0, tot_noise_db = 0, max_noise = -20.0;
  int j = 0;
  const int* scalefac = cod_info->scalefac;
  int scalefacPos = 0;
  res->over_SSD = 0;
  for (sfb = 0; sfb < cod_info->psymax; sfb++) {
    int s = cod_info->global_gain -
            (((scalefac[scalefacPos++]) + (cod_info->preflag != 0 ? pretab[sfb] : 0)) << (cod_info->scalefac_scale + 1)) -
            cod_info->subblock_gain[cod_info->window[sfb]] * 8;
    double noise = 0.0;
    if (prev_noise != NULL && (prev_noise->step[sfb] == s)) {
      noise = prev_noise->noise[sfb];
      j += cod_info->width[sfb];
      distort[distortPos++] = noise / l3_xmin[l3_xminPos++];
      noise = prev_noise->noise_log[sfb];
    } else {
      double step = e->pow20[s + Q_MAX2];
      l = cod_info->width[sfb] >> 1;
      if ((j + cod_info->width[sfb]) > cod_info->max_nonzero_coeff) {
        int usefullsize = cod_info->max_nonzero_coeff - j + 1;
        if (usefullsize > 0) l = usefullsize >> 1;
        else l = 0;
      }
      int sl = j;
      noise = calc_noise_core(e, cod_info, &sl, l, step);
      j = sl;
      if (prev_noise != NULL) {
        prev_noise->step[sfb] = s;
        prev_noise->noise[sfb] = noise;
      }
      /* `noise = distort[..] = expr`: noise takes the UNROUNDED value of expr */
      noise = noise / l3_xmin[l3_xminPos++];
      distort[distortPos++] = noise;
      noise = js_log10(js_max(noise, 1E-20));
      if (prev_noise != NULL) prev_noise->noise_log[sfb] = noise;
    }
    if (prev_noise != NULL) prev_noise->global_gain = cod_info->global_gain;
    tot_noise_db += noise;
    if (noise > 0.0) {
      double tmp = js_max(js_toint32(noise * 10 + .5), 1);
      res->over_SSD += tmp * tmp;
      over++;
      over_noise_db += noise;
    }
    max_noise = js_max(max_noise, noise);
  }
  res->over_count = over;
  res->tot_noise = tot_noise_db;
  res->over_noise = over_noise_db;
  res->max_noise = max_noise;
  return over;
}

/* ---------------------------------------------------------------- Takehiro: quantize + count */
static void quantize_lines_xrpow_01(int l, double istep, const F32* xr, int xrPos, int* ix, int ixPos) {
  double compareval0 = (1.0 - 0.4054) / istep;
  l = l >> 1;
  while ((l--) != 0) {
    ix[ixPos++] = (compareval0 > xr[xrPos++]) ? 0 : 1;
    ix[ixPos++] = (compareval0 > xr[xrPos++]) ? 0 : 1;
  }
}

static void quantize_lines_xrpow(const LjEnc* e, int l, double istep, const F32* xr, int xrPos, int* ix, int ixPos) {
  const F32* adj43 = e->adj43;
  l = l >> 1;
  int remaining = l % 2;
  l = l >> 1;
  while (l-- != 0) {
    double x0, x1, x2, x3;
    int rx0, rx1, rx2, rx3;
    x0 = xr[xrPos++] * istep;
    x1 = xr[xrPos++] * istep;
    rx0 = js_toint32(x0);
    x2 = xr[xrPos++] * istep;
    rx1 = js_toint32(x1);
    x3 = xr[xrPos++] * istep;
    rx2 = js_toint32(x2);
    x0 += adj43[rx0];
    rx3 = js_toint32(x3);
    x1 += adj43[rx1];
    ix[ixPos++] = js_toint32(x0);
    x2 += adj43[rx2];
    ix[ixPos++] = js_toint32(x1);
    x3 += adj43[rx3];
    ix[ixPos++] = js_toint32(x2);
    ix[ixPos++] = js_toint32(x3);
  }
  if (remaining != 0) {
    double x0, x1;
    int rx0, rx1;
    x0 = xr[xrPos++] * istep;
    x1 = xr[xrPos++] * istep;
    rx0 = js_toint32(x0);
    rx1 = js_toint32(x1);
    x0 += adj43[rx0];
    x1 += adj43[rx1];
    ix[ixPos++] = js_toint32(x0);
    ix[ixPos++] = js_toint32(x1);
  }
}

static void quantize_xrpow(const LjEnc* e, const F32* xp, int* pi, double istep, const GrInfo* codInfo,
                           const CalcNoiseData* prevNoise) {
  int sfb, sfbmax, j = 0;
  bool prev_data_use;
  int accumulate = 0, accumulate01 = 0;
  int xpPos = 0, iDataPos = 0, acc_iDataPos = 0, acc_xpPos = 0;
  prev_data_use = (prevNoise != NULL && (codInfo->global_gain == prevNoise->global_gain));
  if (codInfo->block_type == SHORT_TYPE) sfbmax = 38;
  else sfbmax = 21;
  for (sfb = 0; sfb <= sfbmax; sfb++) {
    int step = -1;
    if (prev_data_use || codInfo->block_type == NORM_TYPE) {
      step = codInfo->global_gain -
             ((codInfo->scalefac[sfb] + (codInfo->preflag != 0 ? pretab[sfb] : 0)) << (codInfo->scalefac_scale + 1)) -
             codInfo->subblock_gain[codInfo->window[sfb]] * 8;
    }
    if (prev_data_use && (prevNoise->step[sfb] == step)) {
      if (accumulate != 0) { quantize_lines_xrpow(e, accumulate, istep, xp, acc_xpPos, pi, acc_iDataPos); accumulate = 0; }
      if (accumulate01 != 0) { quantize_lines_xrpow_01(accumulate01, istep, xp, acc_xpPos, pi, acc_iDataPos); accumulate01 = 0; }
    } else {
      int l = codInfo->width[sfb];
      if ((j + codInfo->width[sfb]) > codInfo->max_nonzero_coeff) {
        int usefullsize = codInfo->max_nonzero_coeff - j + 1;
        for (int z = codInfo->max_nonzero_coeff; z < 576; z++) pi[z] = 0;
        l = usefullsize;
        if (l < 0) l = 0;
        sfb = sfbmax + 1;
      }
      if (0 == accumulate && 0 == accumulate01) { acc_iDataPos = iDataPos; acc_xpPos = xpPos; }
      /* NOTE: `sfb` may already be sfbmax+1 here; prevNoise.step[sfb] then reads step[22] (long) or
       * step[39] (short -> `undefined` in JS: comparisons with undefined are false). */
      bool use01 = false;
      if (prevNoise != NULL && prevNoise->sfb_count1 > 0 && sfb >= prevNoise->sfb_count1) {
        if (sfb < SFBMAX) use01 = (prevNoise->step[sfb] > 0 && step >= prevNoise->step[sfb]);
      }
      if (use01) {
        if (accumulate != 0) {
          quantize_lines_xrpow(e, accumulate, istep, xp, acc_xpPos, pi, acc_iDataPos);
          accumulate = 0;
          acc_iDataPos = iDataPos; acc_xpPos = xpPos;
        }
        accumulate01 += l;
      } else {
        if (accumulate01 != 0) {
          quantize_lines_xrpow_01(accumulate01, istep, xp, acc_xpPos, pi, acc_iDataPos);
          accumulate01 = 0;
          acc_iDataPos = iDataPos; acc_xpPos = xpPos;
        }
        accumulate += l;
      }
      if (l <= 0) {
        if (accumulate01 != 0) { quantize_lines_xrpow_01(accumulate01, istep, xp, acc_xpPos, pi, acc_iDataPos); accumulate01 = 0; }
        if (accumulate != 0) { quantize_lines_xrpow(e, accumulate, istep, xp, acc_xpPos, pi, acc_iDataPos); accumulate = 0; }
        break;
      }
    }
    if (sfb <= sfbmax) {
      iDataPos += codInfo->width[sfb];
      xpPos += codInfo->width[sfb];
      j += codInfo->width[sfb];
    }
  }
  if (accumulate != 0) { quantize_lines_xrpow(e, accumulate, istep, xp, acc_xpPos, pi, acc_iDataPos); accumulate = 0; }
  if (accumulate01 != 0) { quantize_lines_xrpow_01(accumulate01, istep, xp, acc_xpPos, pi, acc_iDataPos); accumulate01 = 0; }
}

static int ix_max(const int* ix, int ixPos, int endPos) {
  int max1 = 0, max2 = 0;
  do {
    int x1 = ix[ixPos++];
    int x2 = ix[ixPos++];
    if (max1 < x1) max1 = x1;
    if (max2 < x2) max2 = x2;
  } while (ixPos < endPos);
  if (max1 < max2) max1 = max2;
  return max1;
}

static int count_bit_ESC(const int* ix, int ixPos, int end, int t1, int t2, int* s) {
  int linbits = LJ_HUFF_XLEN[t1] * 65536 + LJ_HUFF_XLEN[t2];
  int sum = 0, sum2;
  do {
    int x = ix[ixPos++];
    int y = ix[ixPos++];
    if (x != 0) {
      if (x > 14) { x = 15; sum += linbits; }
      x *= 16;
    }
    if (y != 0) {
      if (y > 14) { y = 15; sum += linbits; }
      x += y;
    }
    sum += LJ_HUFF_LARGETBL[x];
  } while (ixPos < end);
  sum2 = sum & 0xffff;
  sum >>= 16;
  if (sum > sum2) { sum = sum2; t1 = t2; }
  *s += sum;
  return t1;
}
static int count_bit_noESC(const int* ix, int ixPos, int end, int* s) {
  int sum1 = 0;
  do {
    int x = ix[ixPos + 0] * 2 + ix[ixPos + 1];
    ixPos += 2;
    sum1 += HLEN(1, x);
  } while (ixPos < end);
  *s += sum1;
  return 1;
}
static int count_bit_noESC_from2(const int* ix, int ixPos, int end, int t1, int* s) {
  int sum = 0, sum2;
  int xlen = LJ_HUFF_XLEN[t1];
  const unsigned int* hlen = (t1 == 2) ? LJ_HUFF_TABLE23 : LJ_HUFF_TABLE56;
  do {
    int x = ix[ixPos + 0] * xlen + ix[ixPos + 1];
    ixPos += 2;
    sum += hlen[x];
  } while (ixPos < end);
  sum2 = sum & 0xffff;
  sum >>= 16;
  if (sum > sum2) { sum = sum2; t1++; }
  *s += sum;
  return t1;
}
static int count_bit_noESC_from3(const int* ix, int ixPos, int end, int t1, int* s) {
  int sum1 = 0, sum2 = 0, sum3 = 0;
  int xlen = LJ_HUFF_XLEN[t1];
  do {
    int x = ix[ixPos + 0] * xlen + ix[ixPos + 1];
    ixPos += 2;
    sum1 += HLEN(t1, x);
    sum2 += HLEN(t1 + 1, x);
    sum3 += HLEN(t1 + 2, x);
  } while (ixPos < end);
  int t = t1;
  if (sum1 > sum2) { sum1 = sum2; t++; }
  if (sum1 > sum3) { sum1 = sum3; t = t1 + 2; }
  *s += sum1;
  return t;
}

static const int huf_tbl_noESC[15] = {1, 2, 5, 7, 7, 10, 10, 13, 13, 13, 13, 13, 13, 13, 13};

static int choose_table(const int* ix, int ixPos, int endPos, int* s) {
  int max = ix_max(ix, ixPos, endPos);
  switch (max) {
    case 0: return max;
    case 1: return count_bit_noESC(ix, ixPos, endPos, s);
    case 2: case 3: return count_bit_noESC_from2(ix, ixPos, endPos, huf_tbl_noESC[max - 1], s);
    case 4: case 5: case 6: case 7: case 8: case 9: case 10: case 11: case 12: case 13: case 14: case 15:
      return count_bit_noESC_from3(ix, ixPos, endPos, huf_tbl_noESC[max - 1], s);
    default: {
      if (max > IXMAX_VAL) { *s = LARGE_BITS; return -1; }
      max -= 15;
      int choice2;
      for (choice2 = 24; choice2 < 32; choice2++) if (LJ_HUFF_LINMAX[choice2] >= max) break;
      int choice;
      for (choice = choice2 - 8; choice < 24; choice++) if (LJ_HUFF_LINMAX[choice] >= max) break;
      return count_bit_ESC(ix, ixPos, endPos, choice, choice2, s);
    }
  }
}

static const int t32l[16] = {1 + 0, 4 + 1, 4 + 1, 5 + 2, 4 + 1, 6 + 2, 5 + 2, 6 + 3, 4 + 1, 5 + 2, 5 + 2, 6 + 3, 5 + 2, 6 + 3, 6 + 3, 6 + 4};
static const int t33l[16] = {4 + 0, 4 + 1, 4 + 1, 4 + 2, 4 + 1, 4 + 2, 4 + 2, 4 + 3, 4 + 1, 4 + 2, 4 + 2, 4 + 3, 4 + 2, 4 + 3, 4 + 3, 4 + 4};

static void best_huffman_divide(const LjEnc* e, GrInfo* gi);

static int noquant_count_bits(const LjEnc* e, GrInfo* gi, CalcNoiseData* prev_noise) {
  int* ix = gi->l3_enc;
  int i = ((gi->max_nonzero_coeff + 2) >> 1) << 1;
  if (i > 576) i = 576;
  if (prev_noise != NULL) prev_noise->sfb_count1 = 0;
  for (; i > 1; i -= 2)
    if ((ix[i - 1] | ix[i - 2]) != 0) break;
  gi->count1 = i;
  int a1 = 0, a2 = 0;
  for (; i > 3; i -= 4) {
    int p;
    if (((ix[i - 1] | ix[i - 2] | ix[i - 3] | ix[i - 4]) & 0x7fffffff) > 1) break;
    p = ((ix[i - 4] * 2 + ix[i - 3]) * 2 + ix[i - 2]) * 2 + ix[i - 1];
    a1 += t32l[p];
    a2 += t33l[p];
  }
  int bits = a1;
  gi->count1table_select = 0;
  if (a1 > a2) { bits = a2; gi->count1table_select = 1; }
  gi->count1bits = bits;
  gi->big_values = i;
  if (i == 0) return bits;
  if (gi->block_type == SHORT_TYPE) {
    a1 = 3 * e->sfb_s[3];
    if (a1 > gi->big_values) a1 = gi->big_values;
    a2 = gi->big_values;
  } else if (gi->block_type == NORM_TYPE) {
    a1 = gi->region0_count = e->bv_scf[i - 2];
    a2 = gi->region1_count = e->bv_scf[i - 1];
    a2 = e->sfb_l[a1 + a2 + 2];
    a1 = e->sfb_l[a1 + 1];
    if (a2 < i) gi->table_select[2] = choose_table(ix, a2, i, &bits);
  } else {
    gi->region0_count = 7;
    gi->region1_count = SBMAX_l - 1 - 7 - 1;
    a1 = e->sfb_l[7 + 1];
    a2 = i;
    if (a1 > a2) a1 = a2;
  }
  a1 = a1 < i ? a1 : i;
  a2 = a2 < i ? a2 : i;
  if (0 < a1) gi->table_select[0] = choose_table(ix, 0, a1, &bits);
  if (a1 < a2) gi->table_select[1] = choose_table(ix, a1, a2, &bits);
  if (e->use_best_huffman == 2) {
    gi->part2_3_length = bits;
    best_huffman_divide(e, gi);
    bits = gi->part2_3_length;
  }
  if (prev_noise != NULL) {
    if (gi->block_type == NORM_TYPE) {
      int sfb = 0;
      while (e->sfb_l[sfb] < gi->big_values) sfb++;
      prev_noise->sfb_count1 = sfb;
    }
  }
  return bits;
}

static int count_bits(const LjEnc* e, const F32* xr, GrInfo* gi, CalcNoiseData* prev_noise) {
  int* ix = gi->l3_enc;
  double w = (IXMAX_VAL) / (double)e->ipow20[gi->global_gain];
  if (gi->xrpow_max > w) return LARGE_BITS;
  quantize_xrpow(e, xr, ix, e->ipow20[gi->global_gain], gi, prev_noise);
  /* substep_shaping & 2 == 0 at quality 3 */
  return noquant_count_bits(e, gi, prev_noise);
}

static void recalc_divide_init(const LjEnc* e, const GrInfo* cod_info, const int* ix, int* r01_bits, int* r01_div,
                               int* r0_tbl, int* r1_tbl) {
  int bigv = cod_info->big_values;
  for (int r0 = 0; r0 <= 7 + 15; r0++) r01_bits[r0] = LARGE_BITS;
  for (int r0 = 0; r0 < 16; r0++) {
    int a1 = e->sfb_l[r0 + 1];
    if (a1 >= bigv) break;
    int r0bits = 0;
    int r0t = choose_table(ix, 0, a1, &r0bits);
    for (int r1 = 0; r1 < 8; r1++) {
      int a2 = e->sfb_l[r0 + r1 + 2];
      if (a2 >= bigv) break;
      int bits = r0bits;
      int r1t = choose_table(ix, a1, a2, &bits);
      if (r01_bits[r0 + r1] > bits) {
        r01_bits[r0 + r1] = bits;
        r01_div[r0 + r1] = r0;
        r0_tbl[r0 + r1] = r0t;
        r1_tbl[r0 + r1] = r1t;
      }
    }
  }
}

static void recalc_divide_sub(const LjEnc* e, const GrInfo* cod_info2, GrInfo* gi, const int* ix, const int* r01_bits,
                              const int* r01_div, const int* r0_tbl, const int* r1_tbl) {
  int bigv = cod_info2->big_values;
  for (int r2 = 2; r2 < SBMAX_l + 1; r2++) {
    int a2 = e->sfb_l[r2];
    if (a2 >= bigv) break;
    int bits = r01_bits[r2 - 2] + cod_info2->count1bits;
    if (gi->part2_3_length <= bits) break;
    int r2t = choose_table(ix, a2, bigv, &bits);
    if (gi->part2_3_length <= bits) continue;
    *gi = *cod_info2;   /* NOTE: `ix` aliases gi.l3_enc in the caller; assign() clones identical contents */
    gi->part2_3_length = bits;
    gi->region0_count = r01_div[r2 - 2];
    gi->region1_count = r2 - 2 - r01_div[r2 - 2];
    gi->table_select[0] = r0_tbl[r2 - 2];
    gi->table_select[1] = r1_tbl[r2 - 2];
    gi->table_select[2] = r2t;
  }
}

static void best_huffman_divide(const LjEnc* e, GrInfo* gi) {
  GrInfo cod_info2;
  /* In lamejs `ix = gi.l3_enc` keeps pointing at the ORIGINAL array even after gi.assign() swaps
   * gi.l3_enc for a clone; contents are identical (nothing writes l3_enc here), so one array suffices. */
  int r01_bits[7 + 15 + 1], r01_div[7 + 15 + 1], r0_tbl[7 + 15 + 1], r1_tbl[7 + 15 + 1];
  memset(r01_div, 0, sizeof r01_div); memset(r0_tbl, 0, sizeof r0_tbl); memset(r1_tbl, 0, sizeof r1_tbl);
  const int* ix = gi->l3_enc;
  if (gi->block_type == SHORT_TYPE && e->mode_gr == 1) return;   /* "SHORT BLOCK stuff fails for MPEG2" (Takehiro.js:735-737) */
  cod_info2 = *gi;
  if (gi->block_type == NORM_TYPE) {
    recalc_divide_init(e, gi, ix, r01_bits, r01_div, r0_tbl, r1_tbl);
    recalc_divide_sub(e, &cod_info2, gi, ix, r01_bits, r01_div, r0_tbl, r1_tbl);
  }
  int i = cod_info2.big_values;
  if (i == 0 || (ix[i - 2] | ix[i - 1]) > 1) return;
  i = gi->count1 + 2;
  if (i > 576) return;
  cod_info2 = *gi;
  cod_info2.count1 = i;
  int a1 = 0, a2 = 0;
  for (; i > cod_info2.big_values; i -= 4) {
    int p = ((ix[i - 4] * 2 + ix[i - 3]) * 2 + ix[i - 2]) * 2 + ix[i - 1];
    a1 += t32l[p];
    a2 += t33l[p];
  }
  cod_info2.big_values = i;
  cod_info2.count1table_select = 0;
  if (a1 > a2) { a1 = a2; cod_info2.count1table_select = 1; }
  cod_info2.count1bits = a1;
  if (cod_info2.block_type == NORM_TYPE)
    recalc_divide_sub(e, &cod_info2, gi, ix, r01_bits, r01_div, r0_tbl, r1_tbl);
  else {
    cod_info2.part2_3_length = a1;
    a1 = e->sfb_l[7 + 1];
    if (a1 > i) a1 = i;
    if (a1 > 0) cod_info2.table_select[0] = choose_table(ix, 0, a1, &cod_info2.part2_3_length);
    if (i > a1) cod_info2.table_select[1] = choose_table(ix, a1, i, &cod_info2.part2_3_length);
    if (gi->part2_3_length > cod_info2.part2_3_length) *gi = cod_info2;
  }
}

static const int slen1_n[16] = {1, 1, 1, 1, 8, 2, 2, 2, 4, 4, 4, 8, 8, 8, 16, 16};
static const int slen2_n[16] = {1, 2, 4, 8, 1, 2, 4, 8, 2, 4, 8, 2, 4, 8, 4, 8};
extern const int lj_slen1_tab[16]; extern const int lj_slen2_tab[16];
const int lj_slen1_tab[16] = {0, 0, 0, 0, 3, 1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4};
const int lj_slen2_tab[16] = {0, 1, 2, 3, 0, 1, 2, 3, 1, 2, 3, 1, 2, 3, 2, 3};
static const int scfsi_band[5] = {0, 6, 11, 16, 21};

static void scfsi_calc(LjEnc* e, int ch) {
  int sfb;
  GrInfo* gi = &e->tt[1][ch];
  const GrInfo* g0 = &e->tt[0][ch];
  for (int i = 0; i < 4; i++) {
    for (sfb = scfsi_band[i]; sfb < scfsi_band[i + 1]; sfb++)
      if (g0->scalefac[sfb] != gi->scalefac[sfb] && gi->scalefac[sfb] >= 0) break;
    if (sfb == scfsi_band[i + 1]) {
      for (sfb = scfsi_band[i]; sfb < scfsi_band[i + 1]; sfb++) gi->scalefac[sfb] = -1;
      e->scfsi[ch][i] = 1;
    }
  }
  int s1 = 0, c1 = 0;
  for (sfb = 0; sfb < 11; sfb++) {
    if (gi->scalefac[sfb] == -1) continue;
    c1++;
    if (s1 < gi->scalefac[sfb]) s1 = gi->scalefac[sfb];
  }
  int s2 = 0, c2 = 0;
  for (; sfb < SBPSY_l; sfb++) {
    if (gi->scalefac[sfb] == -1) continue;
    c2++;
    if (s2 < gi->scalefac[sfb]) s2 = gi->scalefac[sfb];
  }
  for (int i = 0; i < 16; i++) {
    if (s1 < slen1_n[i] && s2 < slen2_n[i]) {
      int c = lj_slen1_tab[i] * c1 + lj_slen2_tab[i] * c2;
      if (gi->part2_length > c) { gi->part2_length = c; gi->scalefac_compress = i; }
    }
  }
}

static const int scale_short[16] = {0, 18, 36, 54, 54, 36, 54, 72, 54, 72, 90, 72, 90, 108, 108, 126};
static const int scale_mixed[16] = {0, 18, 36, 54, 51, 35, 53, 71, 52, 70, 88, 69, 87, 105, 104, 122};
static const int scale_long[16] = {0, 10, 20, 30, 33, 21, 31, 41, 32, 42, 52, 43, 53, 63, 64, 74};

static bool scale_bitcount(GrInfo* cod_info) {
  int k, sfb, max_slen1 = 0, max_slen2 = 0;
  const int* tab;
  int* scalefac = cod_info->scalefac;
  if (cod_info->block_type == SHORT_TYPE) {
    tab = scale_short;
    if (cod_info->mixed_block_flag != 0) tab = scale_mixed;
  } else {
    tab = scale_long;
    if (0 == cod_info->preflag) {
      for (sfb = 11; sfb < SBPSY_l; sfb++) if (scalefac[sfb] < pretab[sfb]) break;
      if (sfb == SBPSY_l) {
        cod_info->preflag = 1;
        for (sfb = 11; sfb < SBPSY_l; sfb++) scalefac[sfb] -= pretab[sfb];
      }
    }
  }
  for (sfb = 0; sfb < cod_info->sfbdivide; sfb++) if (max_slen1 < scalefac[sfb]) max_slen1 = scalefac[sfb];
  for (; sfb < cod_info->sfbmax; sfb++) if (max_slen2 < scalefac[sfb]) max_slen2 = scalefac[sfb];
  cod_info->part2_length = LARGE_BITS;
  for (k = 0; k < 16; k++) {
    if (max_slen1 < slen1_n[k] && max_slen2 < slen2_n[k] && cod_info->part2_length > tab[k]) {
      cod_info->part2_length = tab[k];
      cod_info->scalefac_compress = k;
    }
  }
  return cod_info->part2_length == LARGE_BITS;
}

/* QuantizePVT.js:116-122 */
static const int nr_of_sfb_block[6][3][4] = {
  {{6, 5, 5, 5}, {9, 9, 9, 9}, {6, 9, 9, 9}}, {{6, 5, 7, 3}, {9, 9, 12, 6}, {6, 9, 12, 6}}, {{11, 10, 0, 0}, {18, 18, 0, 0}, {15, 18, 0, 0}},
  {{7, 7, 7, 0}, {12, 12, 12, 0}, {6, 15, 12, 0}}, {{6, 6, 6, 3}, {12, 9, 9, 6}, {6, 12, 9, 6}}, {{8, 8, 5, 0}, {15, 12, 9, 0}, {6, 18, 9, 0}}};

/* scale_bitcount_lsf (Takehiro.js:1036-1132): MPEG-2 / 2.5 scalefactor coding */
static bool scale_bitcount_lsf(GrInfo* cod_info) {
  static const int max_range_sfac_tab[6][4] = {{15, 15, 7, 7}, {15, 15, 7, 0}, {7, 3, 0, 0}, {15, 31, 31, 0}, {7, 7, 7, 0}, {3, 3, 0, 0}};
  static const int log2tab[16] = {0, 1, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 4, 4, 4, 4};
  int table_number, row_in_table, partition, nr_sfb, window, i, sfb;
  bool over;
  int max_sfac[4] = {0, 0, 0, 0};
  const int* scalefac = cod_info->scalefac;
  table_number = cod_info->preflag != 0 ? 2 : 0;
  if (cod_info->block_type == SHORT_TYPE) {
    row_in_table = 1;
    const int* partition_table = nr_of_sfb_block[table_number][row_in_table];
    for (sfb = 0, partition = 0; partition < 4; partition++) {
      nr_sfb = partition_table[partition] / 3;
      for (i = 0; i < nr_sfb; i++, sfb++)
        for (window = 0; window < 3; window++)
          if (scalefac[sfb * 3 + window] > max_sfac[partition]) max_sfac[partition] = scalefac[sfb * 3 + window];
    }
  } else {
    row_in_table = 0;
    const int* partition_table = nr_of_sfb_block[table_number][row_in_table];
    for (sfb = 0, partition = 0; partition < 4; partition++) {
      nr_sfb = partition_table[partition];
      for (i = 0; i < nr_sfb; i++, sfb++)
        if (scalefac[sfb] > max_sfac[partition]) max_sfac[partition] = scalefac[sfb];
    }
  }
  for (over = false, partition = 0; partition < 4; partition++)
    if (max_sfac[partition] > max_range_sfac_tab[table_number][partition]) over = true;
  if (!over) {
    cod_info->sfb_partition_table = nr_of_sfb_block[table_number][row_in_table];
    for (partition = 0; partition < 4; partition++) cod_info->slen[partition] = log2tab[max_sfac[partition]];
    const int slen1 = cod_info->slen[0], slen2 = cod_info->slen[1], slen3 = cod_info->slen[2], slen4 = cod_info->slen[3];
    switch (table_number) {
      case 0: cod_info->scalefac_compress = (((slen1 * 5) + slen2) << 4) + (slen3 << 2) + slen4; break;
      case 1: cod_info->scalefac_compress = 400 + (((slen1 * 5) + slen2) << 2) + slen3; break;
      case 2: cod_info->scalefac_compress = 500 + (slen1 * 3) + slen2; break;
    }
    cod_info->part2_length = 0;
    for (partition = 0; partition < 4; partition++) cod_info->part2_length += cod_info->slen[partition] * cod_info->sfb_partition_table[partition];
  }
  return over;
}

static void best_scalefac_store(LjEnc* e, int gr, int ch) {
  GrInfo* gi = &e->tt[gr][ch];
  int sfb, i, j, l;
  int recalc = 0;
  j = 0;
  for (sfb = 0; sfb < gi->sfbmax; sfb++) {
    int width = gi->width[sfb];
    j += width;
    for (l = -width; l < 0; l++) if (gi->l3_enc[l + j] != 0) break;
    if (l == 0) gi->scalefac[sfb] = recalc = -2;
  }
  if (0 == gi->scalefac_scale && 0 == gi->preflag) {
    int s = 0;
    for (sfb = 0; sfb < gi->sfbmax; sfb++) if (gi->scalefac[sfb] > 0) s |= gi->scalefac[sfb];
    if (0 == (s & 1) && s != 0) {
      for (sfb = 0; sfb < gi->sfbmax; sfb++) if (gi->scalefac[sfb] > 0) gi->scalefac[sfb] >>= 1;
      gi->scalefac_scale = recalc = 1;
    }
  }
  if (0 == gi->preflag && gi->block_type != SHORT_TYPE && e->mode_gr == 2) {
    for (sfb = 11; sfb < SBPSY_l; sfb++) if (gi->scalefac[sfb] < pretab[sfb] && gi->scalefac[sfb] != -2) break;
    if (sfb == SBPSY_l) {
      for (sfb = 11; sfb < SBPSY_l; sfb++) if (gi->scalefac[sfb] > 0) gi->scalefac[sfb] -= pretab[sfb];
      gi->preflag = recalc = 1;
    }
  }
  for (i = 0; i < 4; i++) e->scfsi[ch][i] = 0;
  if (e->mode_gr == 2 && gr == 1 && e->tt[0][ch].block_type != SHORT_TYPE && e->tt[1][ch].block_type != SHORT_TYPE) {
    scfsi_calc(e, ch);
    recalc = 0;
  }
  for (sfb = 0; sfb < gi->sfbmax; sfb++) if (gi->scalefac[sfb] == -2) gi->scalefac[sfb] = 0;
  if (recalc != 0) { if (e->mode_gr == 2) scale_bitcount(gi); else scale_bitcount_lsf(gi); }
}

/* ---------------------------------------------------------------- Quantize.js */
static double init_xrpow_core(GrInfo* cod_info, F32* xrpow, int upper) {
  double sum = 0;
  for (int i = 0; i <= upper; ++i) {
    double tmp = fabs(cod_info->xr[i]);
    sum += tmp;
    xrpow[i] = sqrt(tmp * sqrt(tmp));
    if (xrpow[i] > cod_info->xrpow_max) cod_info->xrpow_max = xrpow[i];
  }
  return sum;
}

static bool init_xrpow(LjEnc* e, GrInfo* cod_info, F32* xrpow) {
  double sum = 0;
  int upper = cod_info->max_nonzero_coeff;
  cod_info->xrpow_max = 0;
  for (int i = upper; i < 576; i++) xrpow[i] = 0;
  sum = init_xrpow_core(cod_info, xrpow, upper);
  if (sum > 1E-20) {
    int j = 0;
    if ((e->substep_shaping & 2) != 0) j = 1;
    for (int i = 0; i < cod_info->psymax; i++) e->pseudohalf[i] = j;
    return true;
  }
  for (int i = 0; i < 576; i++) cod_info->l3_enc[i] = 0;
  return false;
}

static void psfb21_analogsilence(LjEnc* e, GrInfo* cod_info) {
  F32* xr = cod_info->xr;
  if (cod_info->block_type != SHORT_TYPE) {
    bool stop = false;
    for (int gsfb = PSFB21 - 1; gsfb >= 0 && !stop; gsfb--) {
      int start = e->psfb21[gsfb], end = e->psfb21[gsfb + 1];
      double ath21 = athAdjust(e->ath_adjust, e->ath_psfb21[gsfb], e->ath_floor);
      if (e->longfact[21] > 1e-12) ath21 *= e->longfact[21];
      for (int j = end - 1; j >= start; j--) {
        if (fabs(xr[j]) < ath21) xr[j] = 0;
        else { stop = true; break; }
      }
    }
  } else {
    for (int block = 0; block < 3; block++) {
      bool stop = false;
      for (int gsfb = PSFB12 - 1; gsfb >= 0 && !stop; gsfb--) {
        int start = e->sfb_s[12] * 3 + (e->sfb_s[13] - e->sfb_s[12]) * block + (e->psfb12[gsfb] - e->psfb12[0]);
        int end = start + (e->psfb12[gsfb + 1] - e->psfb12[gsfb]);
        double ath12 = athAdjust(e->ath_adjust, e->ath_psfb12[gsfb], e->ath_floor);
        if (e->shortfact[12] > 1e-12) ath12 *= e->shortfact[12];
        for (int j = end - 1; j >= start; j--) {
          if (fabs(xr[j]) < ath12) xr[j] = 0;
          else { stop = true; break; }
        }
      }
    }
  }
}

static void init_outer_loop(LjEnc* e, GrInfo* cod_info) {
  cod_info->part2_3_length = 0;
  cod_info->big_values = 0;
  cod_info->count1 = 0;
  cod_info->global_gain = 210;
  cod_info->scalefac_compress = 0;
  cod_info->table_select[0] = cod_info->table_select[1] = cod_info->table_select[2] = 0;
  cod_info->subblock_gain[0] = cod_info->subblock_gain[1] = cod_info->subblock_gain[2] = cod_info->subblock_gain[3] = 0;
  cod_info->region0_count = 0;
  cod_info->region1_count = 0;
  cod_info->preflag = 0;
  cod_info->scalefac_scale = 0;
  cod_info->count1table_select = 0;
  cod_info->part2_length = 0;
  cod_info->sfb_lmax = SBPSY_l;
  cod_info->sfb_smin = SBPSY_s;
  cod_info->psy_lmax = e->sfb21_extra ? SBMAX_l : SBPSY_l;
  cod_info->psymax = cod_info->psy_lmax;
  cod_info->sfbmax = cod_info->sfb_lmax;
  cod_info->sfbdivide = 11;
  for (int sfb = 0; sfb < SBMAX_l; sfb++) {
    cod_info->width[sfb] = e->sfb_l[sfb + 1] - e->sfb_l[sfb];
    cod_info->window[sfb] = 3;
  }
  if (cod_info->block_type == SHORT_TYPE) {
    F32 ixwork[576];
    cod_info->sfb_smin = 0;
    cod_info->sfb_lmax = 0;
    /* mixed_block_flag == 0 always */
    cod_info->psymax = cod_info->sfb_lmax + 3 * ((e->sfb21_extra ? SBMAX_s : SBPSY_s) - cod_info->sfb_smin);
    cod_info->sfbmax = cod_info->sfb_lmax + 3 * (SBPSY_s - cod_info->sfb_smin);
    cod_info->sfbdivide = cod_info->sfbmax - 18;
    cod_info->psy_lmax = cod_info->sfb_lmax;
    int ix = e->sfb_l[cod_info->sfb_lmax];
    memcpy(ixwork, cod_info->xr, sizeof ixwork);
    for (int sfb = cod_info->sfb_smin; sfb < SBMAX_s; sfb++) {
      int start = e->sfb_s[sfb], end = e->sfb_s[sfb + 1];
      for (int window = 0; window < 3; window++)
        for (int l = start; l < end; l++) cod_info->xr[ix++] = ixwork[3 * l + window];
    }
    int j = cod_info->sfb_lmax;
    for (int sfb = cod_info->sfb_smin; sfb < SBMAX_s; sfb++) {
      cod_info->width[j] = cod_info->width[j + 1] = cod_info->width[j + 2] = e->sfb_s[sfb + 1] - e->sfb_s[sfb];
      cod_info->window[j] = 0;
      cod_info->window[j + 1] = 1;
      cod_info->window[j + 2] = 2;
      j += 3;
    }
  }
  cod_info->count1bits = 0;
  cod_info->sfb_partition_table = nr_of_sfb_block[0][0];
  cod_info->slen[0] = cod_info->slen[1] = cod_info->slen[2] = cod_info->slen[3] = 0;
  cod_info->max_nonzero_coeff = 575;
  for (int i = 0; i < SFBMAX; i++) cod_info->scalefac[i] = 0;
  psfb21_analogsilence(e, cod_info);
}

static int bin_search_StepSize(LjEnc* e, GrInfo* cod_info, int desired_rate, int ch, const F32* xrpow) {
  int nBits;
  int CurrentStep = e->CurrentStep[ch];
  bool flagGoneOver = false;
  int start = e->OldValue[ch];
  int Direction = 0; /* NONE=0 UP=1 DOWN=2 */
  cod_info->global_gain = start;
  desired_rate -= cod_info->part2_length;
  for (;;) {
    int step;
    nBits = count_bits(e, xrpow, cod_info, NULL);
    if (CurrentStep == 1 || nBits == desired_rate) break;
    if (nBits > desired_rate) {
      if (Direction == 2) flagGoneOver = true;
      if (flagGoneOver) CurrentStep /= 2;
      Direction = 1;
      step = CurrentStep;
    } else {
      if (Direction == 1) flagGoneOver = true;
      if (flagGoneOver) CurrentStep /= 2;
      Direction = 2;
      step = -CurrentStep;
    }
    cod_info->global_gain += step;
    if (cod_info->global_gain < 0) { cod_info->global_gain = 0; flagGoneOver = true; }
    if (cod_info->global_gain > 255) { cod_info->global_gain = 255; flagGoneOver = true; e->gain_clamps++; }
  }
  while (nBits > desired_rate && cod_info->global_gain < 255) {
    cod_info->global_gain++;
    nBits = count_bits(e, xrpow, cod_info, NULL);
  }
  e->CurrentStep[ch] = (start - cod_info->global_gain >= 4) ? 4 : 2;
  e->OldValue[ch] = cod_info->global_gain;
  cod_info->part2_3_length = nBits;
  return nBits;
}

static bool loop_break(const GrInfo* cod_info) {
  for (int sfb = 0; sfb < cod_info->sfbmax; sfb++)
    if (cod_info->scalefac[sfb] + cod_info->subblock_gain[cod_info->window[sfb]] == 0) return false;
  return true;
}

static bool quant_compare(int quant_comp, const CalcNoiseResult* best, CalcNoiseResult* calc) {
  bool better;
  switch (quant_comp) {
    default:
    case 9:
      if (best->over_count > 0) {
        better = calc->over_SSD <= best->over_SSD;
        if (calc->over_SSD == best->over_SSD) better = calc->bits < best->bits;
      } else {
        better = ((calc->max_noise < 0) && ((calc->max_noise * 10 + calc->bits) <= (best->max_noise * 10 + best->bits)));
      }
      break;
    case 0:
      better = calc->over_count < best->over_count ||
               (calc->over_count == best->over_count && calc->over_noise < best->over_noise) ||
               (calc->over_count == best->over_count && bs_EQ(calc->over_noise, best->over_noise) && calc->tot_noise < best->tot_noise);
      break;
    case 1: better = calc->max_noise < best->max_noise; break;
  }
  if (best->over_count == 0) better = better && calc->bits < best->bits;
  return better;
}

static void amp_scalefac_bands(LjEnc* e, GrInfo* cod_info, const F32* distort, F32* xrpow, bool bRefine) {
  double ifqstep34;
  if (cod_info->scalefac_scale == 0) ifqstep34 = 1.29683955465100964055;
  else ifqstep34 = 1.68179283050742922612;
  double trigger = 0;
  for (int sfb = 0; sfb < cod_info->sfbmax; sfb++) if (trigger < distort[sfb]) trigger = distort[sfb];
  int noise_shaping_amp = e->noise_shaping_amp;
  if (noise_shaping_amp == 3) noise_shaping_amp = bRefine ? 2 : 1;
  switch (noise_shaping_amp) {
    case 2: break;
    case 1:
      if (trigger > 1.0) trigger = js_pow(trigger, .5);
      else trigger *= .95;
      break;
    case 0:
    default:
      if (trigger > 1.0) trigger = 1.0;
      else trigger *= .95;
      break;
  }
  int j = 0;
  for (int sfb = 0; sfb < cod_info->sfbmax; sfb++) {
    int width = cod_info->width[sfb];
    j += width;
    if (distort[sfb] < trigger) continue;
    /* substep_shaping & 2 == 0 */
    cod_info->scalefac[sfb]++;
    for (int l = -width; l < 0; l++) {
      xrpow[j + l] *= ifqstep34;
      if (xrpow[j + l] > cod_info->xrpow_max) cod_info->xrpow_max = xrpow[j + l];
    }
    if (e->noise_shaping_amp == 2) return;
  }
}

static void inc_scalefac_scale(GrInfo* cod_info, F32* xrpow) {
  double ifqstep34 = 1.29683955465100964055;
  int j = 0;
  for (int sfb = 0; sfb < cod_info->sfbmax; sfb++) {
    int width = cod_info->width[sfb];
    int s = cod_info->scalefac[sfb];
    if (cod_info->preflag != 0) s += pretab[sfb];
    j += width;
    if ((s & 1) != 0) {
      s++;
      for (int l = -width; l < 0; l++) {
        xrpow[j + l] *= ifqstep34;
        if (xrpow[j + l] > cod_info->xrpow_max) cod_info->xrpow_max = xrpow[j + l];
      }
    }
    cod_info->scalefac[sfb] = s >> 1;
  }
  cod_info->preflag = 0;
  cod_info->scalefac_scale = 1;
}

static bool inc_subblock_gain(const LjEnc* e, GrInfo* cod_info, F32* xrpow) {
  int sfb;
  int* scalefac = cod_info->scalefac;
  for (sfb = 0; sfb < cod_info->sfb_lmax; sfb++) if (scalefac[sfb] >= 16) return true;
  for (int window = 0; window < 3; window++) {
    int s1 = 0, s2 = 0;
    for (sfb = cod_info->sfb_lmax + window; sfb < cod_info->sfbdivide; sfb += 3) if (s1 < scalefac[sfb]) s1 = scalefac[sfb];
    for (; sfb < cod_info->sfbmax; sfb += 3) if (s2 < scalefac[sfb]) s2 = scalefac[sfb];
    if (s1 < 16 && s2 < 8) continue;
    if (cod_info->subblock_gain[window] >= 7) return true;
    cod_info->subblock_gain[window]++;
    int j = e->sfb_l[cod_info->sfb_lmax];
    for (sfb = cod_info->sfb_lmax + window; sfb < cod_info->sfbmax; sfb += 3) {
      double amp;
      int width = cod_info->width[sfb];
      int s = scalefac[sfb];
      s = s - (4 >> cod_info->scalefac_scale);
      if (s >= 0) {
        scalefac[sfb] = s;
        j += width * 3;
        continue;
      }
      scalefac[sfb] = 0;
      {
        int gain = 210 + s * (1 << (cod_info->scalefac_scale + 1)); /* s < 0: JS `<<` is arithmetic */
        amp = e->ipow20[gain];
      }
      j += width * (window + 1);
      for (int l = -width; l < 0; l++) {
        xrpow[j + l] *= amp;
        if (xrpow[j + l] > cod_info->xrpow_max) cod_info->xrpow_max = xrpow[j + l];
      }
      j += width * (3 - window - 1);
    }
    {
      double amp = e->ipow20[202];
      j += cod_info->width[sfb] * (window + 1);
      for (int l = -cod_info->width[sfb]; l < 0; l++) {
        xrpow[j + l] *= amp;
        if (xrpow[j + l] > cod_info->xrpow_max) cod_info->xrpow_max = xrpow[j + l];
      }
    }
  }
  return false;
}

static bool balance_noise(LjEnc* e, GrInfo* cod_info, const F32* distort, F32* xrpow, bool bRefine) {
  amp_scalefac_bands(e, cod_info, distort, xrpow, bRefine);
  bool status = loop_break(cod_info);
  if (status) return false;
  status = e->mode_gr == 2 ? scale_bitcount(cod_info) : scale_bitcount_lsf(cod_info);
  if (!status) return true;
  if (e->noise_shaping > 1) {
    for (int i = 0; i < SFBMAX; i++) e->pseudohalf[i] = 0;
    if (0 == cod_info->scalefac_scale) {
      inc_scalefac_scale(cod_info, xrpow);
      status = false;
    } else {
      if (cod_info->block_type == SHORT_TYPE && e->subblock_gain > 0)
        status = (inc_subblock_gain(e, cod_info, xrpow) || loop_break(cod_info));
    }
  }
  if (!status) status = e->mode_gr == 2 ? scale_bitcount(cod_info) : scale_bitcount_lsf(cod_info);
  return !status;
}

static int outer_loop(LjEnc* e, GrInfo* cod_info, const F32* l3_xmin, F32* xrpow, int ch, int targ_bits) {
  static thread_local GrInfo cod_info_w;
  F32 save_xrpow[576];
  F32 distort[SFBMAX];
  CalcNoiseResult best_noise_info; memset(&best_noise_info, 0, sizeof best_noise_info);
  int better;
  CalcNoiseData prev_noise; memset((void*)&prev_noise, 0, sizeof prev_noise);
  int best_part2_3_length = 9999999;
  bool bEndOfSearch = false;
  bool bRefine = false;
  int best_ggain_pass1 = 0;
  bin_search_StepSize(e, cod_info, targ_bits, ch, xrpow);
  if (0 == e->noise_shaping) return 100;
  calc_noise(e, cod_info, l3_xmin, distort, &best_noise_info, &prev_noise);
  best_noise_info.bits = cod_info->part2_3_length;
  cod_info_w = *cod_info;
  int age = 0;
  memcpy(save_xrpow, xrpow, sizeof save_xrpow);
  while (!bEndOfSearch) {
    do {
      CalcNoiseResult noise_info; memset(&noise_info, 0, sizeof noise_info);
      int search_limit;
      int maxggain = 255;
      if ((e->substep_shaping & 2) != 0) search_limit = 20;
      else search_limit = 3;
      /* sfb21_extra == false */
      if (!balance_noise(e, &cod_info_w, distort, xrpow, bRefine)) break;
      if (cod_info_w.scalefac_scale != 0) maxggain = 254;
      int huff_bits = targ_bits - cod_info_w.part2_length;
      if (huff_bits <= 0) break;
      while ((cod_info_w.part2_3_length = count_bits(e, xrpow, &cod_info_w, &prev_noise)) > huff_bits &&
             cod_info_w.global_gain <= maxggain)
        cod_info_w.global_gain++;
      if (cod_info_w.global_gain > maxggain) break;
      if (best_noise_info.over_count == 0) {
        while ((cod_info_w.part2_3_length = count_bits(e, xrpow, &cod_info_w, &prev_noise)) > best_part2_3_length &&
               cod_info_w.global_gain <= maxggain)
          cod_info_w.global_gain++;
        if (cod_info_w.global_gain > maxggain) break;
      }
      calc_noise(e, &cod_info_w, l3_xmin, distort, &noise_info, &prev_noise);
      noise_info.bits = cod_info_w.part2_3_length;
      if (cod_info->block_type != SHORT_TYPE) better = e->quant_comp;
      else better = e->quant_comp_short;
      better = quant_compare(better, &best_noise_info, &noise_info) ? 1 : 0;
      if (better != 0) {
        best_part2_3_length = cod_info->part2_3_length; /* sic: read BEFORE the assign (Quantize.js:996-998) */
        best_noise_info = noise_info;
        *cod_info = cod_info_w;
        age = 0;
        memcpy(save_xrpow, xrpow, sizeof save_xrpow);
      } else {
        if (e->full_outer_loop == 0) {
          if (++age > search_limit && best_noise_info.over_count == 0) break;
          if ((e->noise_shaping_amp == 3) && bRefine && age > 30) break;
          if ((e->noise_shaping_amp == 3) && bRefine && (cod_info_w.global_gain - best_ggain_pass1) > 15) break;
        }
      }
    } while ((cod_info_w.global_gain + cod_info_w.scalefac_scale) < 255);
    if (e->noise_shaping_amp == 3) {
      if (!bRefine) {
        cod_info_w = *cod_info;
        memcpy(xrpow, save_xrpow, sizeof save_xrpow);
        age = 0;
        best_ggain_pass1 = cod_info_w.global_gain;
        bRefine = true;
      } else bEndOfSearch = true;
    } else bEndOfSearch = true;
  }
  /* substep_shaping & 1 == 0: no trancate_smallspectrums */
  return best_noise_info.over_count;
}

static void iteration_finish_one(LjEnc* e, int gr, int ch) {
  GrInfo* cod_info = &e->tt[gr][ch];
  best_scalefac_store(e, gr, ch);
  if (e->use_best_huffman == 1) best_huffman_divide(e, cod_info);
  e->ResvSize -= cod_info->part2_3_length + cod_info->part2_length; /* ResvAdjust */
}

/* Quantize.js:76-83 */
static void ms_convert(LjEnc* e, int gr) {
  for (int i = 0; i < 576; ++i) {
    double l = e->tt[gr][0].xr[i], r = e->tt[gr][1].xr[i];
    e->tt[gr][0].xr[i] = (l + r) * (LJ_SQRT2 * 0.5);
    e->tt[gr][1].xr[i] = (l - r) * (LJ_SQRT2 * 0.5);
  }
}

/* QuantizePVT.js:486-534; targ_bits is an Int32Array: every store truncates */
static void reduce_side(int* targ_bits, double ms_ener_ratio, double mean_bits, double max_bits) {
  double fac = .33 * (.5 - ms_ener_ratio) / .5;
  if (fac < 0) fac = 0;
  if (fac > .5) fac = .5;
  int move_bits = js_toint32(fac * .5 * (targ_bits[0] + targ_bits[1]));
  if (move_bits > MAX_BITS_PER_CHANNEL - targ_bits[0]) move_bits = MAX_BITS_PER_CHANNEL - targ_bits[0];
  if (move_bits < 0) move_bits = 0;
  if (targ_bits[1] >= 125) {
    if (targ_bits[1] - move_bits > 125) {
      if (targ_bits[0] < mean_bits) targ_bits[0] += move_bits;
      targ_bits[1] -= move_bits;
    } else {
      targ_bits[0] += targ_bits[1] - 125;
      targ_bits[1] = 125;
    }
  }
  move_bits = targ_bits[0] + targ_bits[1];
  if (move_bits > max_bits) {
    targ_bits[0] = js_toint32((max_bits * targ_bits[0]) / move_bits);
    targ_bits[1] = js_toint32((max_bits * targ_bits[1]) / move_bits);
  }
}

void lj_iteration_loop(LjEnc* e, double pe[2][2], const double* ms_ener_ratio, PsyRatio ratio[2][2]) {
  F32 l3_xmin[SFBMAX];
  F32 xrpow[576];
  int targ_bits[2] = {0, 0};
  double mean_bits = ResvFrameBegin(e);
  for (int gr = 0; gr < e->mode_gr; gr++) {
    double max_bits = on_pe(e, pe, targ_bits, mean_bits, gr, gr);
    if (e->mode_ext == 2) {                    /* MPG_MD_MS_LR (CBRNewIterationLoop.js:46-50) */
      ms_convert(e, gr);
      reduce_side(targ_bits, ms_ener_ratio[gr], mean_bits, max_bits);
    }
    for (int ch = 0; ch < e->channels_out; ch++) {
      double masking_lower_db;
      GrInfo* cod_info = &e->tt[gr][ch];
      if (cod_info->block_type != SHORT_TYPE) masking_lower_db = e->mask_adjust - 0;
      else masking_lower_db = e->mask_adjust_short - 0;
      e->masking_lower = js_pow(10.0, masking_lower_db * 0.1);
      init_outer_loop(e, cod_info);
      const bool have = init_xrpow(e, cod_info, xrpow);
      if (have) calc_xmin(e, &ratio[gr][ch], cod_info, l3_xmin);
      if (e->qtrace_cur) {                     /* test tap: what outer_loop starts from */
        LjQuantTrace* t = e->qtrace_cur;
        t->max_nonzero_coeff[gr][ch] = cod_info->max_nonzero_coeff;
        t->xrpow_max[gr][ch] = cod_info->xrpow_max;
        for (int i = 0; i < SFBMAX; i++) t->xmin[gr][ch][i] = (have && i < cod_info->psymax) ? l3_xmin[i].v : 0.0f;
        lj_quant_trace_rows(e, e->qtrace_cur, gr, ch, cod_info, xrpow, have);
      }
      if (have) outer_loop(e, cod_info, l3_xmin, xrpow, ch, targ_bits[ch]);
      iteration_finish_one(e, gr, ch);
    }
    if (e->qtrace_cur && gr == 0 && e->mode_gr == 2)
      for (int ch = 0; ch < 2; ch++) { e->qtrace_cur->old_value_mid[ch] = e->OldValue[ch]; e->qtrace_cur->cur_step_mid[ch] = e->CurrentStep[ch]; }
  }
  ResvFrameEnd(e, mean_bits);
}
