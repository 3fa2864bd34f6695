/* lj_psy.cpp -- FFT + psychoacoustic model of the oracle.  TEST INFRASTRUCTURE.
 * Follows src/js/FFT.js (fht :31-115, fft_short :140-183, fft_long :185-224, init_fft :226-242)
 * and src/js/PsyModel.js (compute_ffts :251-324, mask_add :403-473, calc_interchannel_masking
 * :525-543, convert_partition2scalefac_s/_l :644-734, compute_masking_s :736-782, block_type_set
 * :784-826, calc_energy :906, calc_mask_index_l :930, L3psycho_anal_ns :1000-1383, s3_func :2317,
 * freq2bark :2356, init_numline :2365, init_s3_values :2460, psymodel_init :2537-2822,
 * ATHformula(_GB) :2827-2894).  JS quirks reproduced on purpose: fractional array indices in
 * the attack detection (:1133,:1159-1161), `(b + 3) <= 6` in mask_add (:423), bm[] truncation (:2416).
 */
#include <stdlib.h>
#include "lj_encoder.h"
#include "lj_tables.h"

/* ------------------------------------------------------------------ FFT */
static void fht(F32* fz, int fzPos, int n) {
  int tri = 0;
  int k4;
  int fi, gi;
  n <<= 1;
  int fn = fzPos + n;
  k4 = 4;
  do {
    double s1, c1;
    int i, k1, k2, k3, kx;
    kx = k4 >> 1;
    k1 = k4;
    k2 = k4 << 1;
    k3 = k2 + k1;
    k4 = k2 << 1;
    fi = fzPos;
    gi = fi + kx;
    do {
      double f0, f1, f2, f3;
      f1 = fz[fi + 0] - fz[fi + k1];
      f0 = fz[fi + 0] + fz[fi + k1];
      f3 = fz[fi + k2] - fz[fi + k3];
      f2 = fz[fi + k2] + fz[fi + k3];
      fz[fi + k2] = f0 - f2;
      fz[fi + 0] = f0 + f2;
      fz[fi + k3] = f1 - f3;
      fz[fi + k1] = f1 + f3;
      f1 = fz[gi + 0] - fz[gi + k1];
      f0 = fz[gi + 0] + fz[gi + k1];
      f3 = (LJ_SQRT2 * fz[gi + k3]);
      f2 = (LJ_SQRT2 * fz[gi + k2]);
      fz[gi + k2] = f0 - f2;
      fz[gi + 0] = f0 + f2;
      fz[gi + k3] = f1 - f3;
      fz[gi + k1] = f1 + f3;
      gi += k4;
      fi += k4;
    } while (fi < fn);
    c1 = LJ_FHT_COSTAB[tri + 0];
    s1 = LJ_FHT_COSTAB[tri + 1];
    for (i = 1; i < kx; i++) {
      double c2, s2;
      c2 = 1 - (2 * s1) * s1;
      s2 = (2 * s1) * c1;
      fi = fzPos + i;
      gi = fzPos + k1 - i;
      do {
        double a, b, g0, f0, f1, g1, f2, g2, f3, g3;
        b = s2 * fz[fi + k1] - c2 * fz[gi + k1];
        a = c2 * fz[fi + k1] + s2 * fz[gi + k1];
        f1 = fz[fi + 0] - a;
        f0 = fz[fi + 0] + a;
        g1 = fz[gi + 0] - b;
        g0 = fz[gi + 0] + b;
        b = s2 * fz[fi + k3] - c2 * fz[gi + k3];
        a = c2 * fz[fi + k3] + s2 * fz[gi + k3];
        f3 = fz[fi + k2] - a;
        f2 = fz[fi + k2] + a;
        g3 = fz[gi + k2] - b;
        g2 = fz[gi + k2] + b;
        b = s1 * f2 - c1 * g3;
        a = c1 * f2 + s1 * g3;
        fz[fi + k2] = f0 - a;
        fz[fi + 0] = f0 + a;
        fz[gi + k3] = g1 - b;
        fz[gi + k1] = g1 + b;
        b = c1 * g2 - s1 * f3;
        a = s1 * g2 + c1 * f3;
        fz[gi + k2] = g0 - a;
        fz[gi + 0] = g0 + a;
        fz[fi + k3] = f1 - b;
        fz[fi + k1] = f1 + b;
        gi += k4;
        fi += k4;
      } while (fi < fn);
      c2 = c1;
      c1 = c2 * LJ_FHT_COSTAB[tri + 0] - s1 * LJ_FHT_COSTAB[tri + 1];
      s1 = c2 * LJ_FHT_COSTAB[tri + 1] + s1 * LJ_FHT_COSTAB[tri + 0];
    }
    tri += 2;
  } while (k4 < n);
}

static void fft_short(const LjEnc* e, F32 x_real[3][BLKSIZE_s], const F32* buffer, int bufPos) {
  const F32* window_s = e->fft_window_s;
  for (int b = 0; b < 3; b++) {
    int x = BLKSIZE_s / 2;
    int k = 0xffff & ((576 / 3) * (b + 1));
    int j = BLKSIZE_s / 8 - 1;
    do {
      double f0, f1, f2, f3, w;
      int i = LJ_FFT_RV[j << 2] & 0xff;
      f0 = window_s[i] * buffer[bufPos + i + k];
      w = window_s[0x7f - i] * buffer[bufPos + i + k + 0x80];
      f1 = f0 - w; f0 = f0 + w;
      f2 = window_s[i + 0x40] * buffer[bufPos + i + k + 0x40];
      w = window_s[0x3f - i] * buffer[bufPos + i + k + 0xc0];
      f3 = f2 - w; f2 = f2 + w;
      x -= 4;
      x_real[b][x + 0] = f0 + f2;
      x_real[b][x + 2] = f0 - f2;
      x_real[b][x + 1] = f1 + f3;
      x_real[b][x + 3] = f1 - f3;
      f0 = window_s[i + 0x01] * buffer[bufPos + i + k + 0x01];
      w = window_s[0x7e - i] * buffer[bufPos + i + k + 0x81];
      f1 = f0 - w; f0 = f0 + w;
      f2 = window_s[i + 0x41] * buffer[bufPos + i + k + 0x41];
      w = window_s[0x3e - i] * buffer[bufPos + i + k + 0xc1];
      f3 = f2 - w; f2 = f2 + w;
      x_real[b][x + BLKSIZE_s / 2 + 0] = f0 + f2;
      x_real[b][x + BLKSIZE_s / 2 + 2] = f0 - f2;
      x_real[b][x + BLKSIZE_s / 2 + 1] = f1 + f3;
      x_real[b][x + BLKSIZE_s / 2 + 3] = f1 - f3;
    } while (--j >= 0);
    fht(x_real[b], x, BLKSIZE_s / 2);
  }
}

static void fft_long(const LjEnc* e, F32* y, const F32* buffer, int bufPos) {
  const F32* window = e->fft_window;
  int jj = BLKSIZE / 8 - 1;
  int x = BLKSIZE / 2;
  do {
    double f0, f1, f2, f3, w;
    int i = LJ_FFT_RV[jj] & 0xff;
    f0 = window[i] * buffer[bufPos + i];
    w = window[i + 0x200] * buffer[bufPos + i + 0x200];
    f1 = f0 - w; f0 = f0 + w;
    f2 = window[i + 0x100] * buffer[bufPos + i + 0x100];
    w = window[i + 0x300] * buffer[bufPos + i + 0x300];
    f3 = f2 - w; f2 = f2 + w;
    x -= 4;
    y[x + 0] = f0 + f2;
    y[x + 2] = f0 - f2;
    y[x + 1] = f1 + f3;
    y[x + 3] = f1 - f3;
    f0 = window[i + 0x001] * buffer[bufPos + i + 0x001];
    w = window[i + 0x201] * buffer[bufPos + i + 0x201];
    f1 = f0 - w; f0 = f0 + w;
    f2 = window[i + 0x101] * buffer[bufPos + i + 0x101];
    w = window[i + 0x301] * buffer[bufPos + i + 0x301];
    f3 = f2 - w; f2 = f2 + w;
    y[x + BLKSIZE / 2 + 0] = f0 + f2;
    y[x + BLKSIZE / 2 + 2] = f0 - f2;
    y[x + BLKSIZE / 2 + 1] = f1 + f3;
    y[x + BLKSIZE / 2 + 3] = f1 - f3;
  } while (--jj >= 0);
  fht(y, x, BLKSIZE / 2);
}

static void init_fft(LjEnc* e) {
  for (int i = 0; i < BLKSIZE; i++)
    e->fft_window[i] = (0.42 - 0.5 * cos(2 * M_PI * (i + .5) / BLKSIZE) + 0.08 * cos(4 * M_PI * (i + .5) / BLKSIZE));
  for (int i = 0; i < BLKSIZE_s / 2; i++)
    e->fft_window_s[i] = (0.5 * (1.0 - cos(2.0 * M_PI * (i + 0.5) / BLKSIZE_s)));
}

/* ------------------------------------------------------------------ psy helpers */
static const double VO_SCALE = (1. / (14752. * 14752.) / (BLKSIZE / 2));
static const double rpelev = 2, rpelev2 = 16, rpelev_s = 2, rpelev2_s = 16;
static const double DELBARK = .34;
static const double LN_TO_LOG10 = 0.2302585093;
static const double LOG10_C = 2.30258509299404568402;

static const double tab[9] = {1.0, 0.79433, 0.63096, 0.63096, 0.63096, 0.63096, 0.63096, 0.25119, 0.11749};
static const double table1[25] = {3.3246 * 3.3246, 3.23837 * 3.23837, 3.15437 * 3.15437, 3.00412 * 3.00412,
  2.86103 * 2.86103, 2.65407 * 2.65407, 2.46209 * 2.46209, 2.284 * 2.284, 2.11879 * 2.11879, 1.96552 * 1.96552,
  1.82335 * 1.82335, 1.69146 * 1.69146, 1.56911 * 1.56911, 1.46658 * 1.46658, 1.37074 * 1.37074, 1.31036 * 1.31036,
  1.25264 * 1.25264, 1.20648 * 1.20648, 1.16203 * 1.16203, 1.12765 * 1.12765, 1.09428 * 1.09428, 1.0659 * 1.0659,
  1.03826 * 1.03826, 1.01895 * 1.01895, 1};
static const double table2[10] = {1.33352 * 1.33352, 1.35879 * 1.35879, 1.38454 * 1.38454, 1.39497 * 1.39497,
  1.40548 * 1.40548, 1.3537 * 1.3537, 1.30382 * 1.30382, 1.22321 * 1.22321, 1.14758 * 1.14758, 1};
static const double table3[14] = {2.35364 * 2.35364, 2.29259 * 2.29259, 2.23313 * 2.23313, 2.12675 * 2.12675,
  2.02545 * 2.02545, 1.87894 * 1.87894, 1.74303 * 1.74303, 1.61695 * 1.61695, 1.49999 * 1.49999, 1.39148 * 1.39148,
  1.29083 * 1.29083, 1.19746 * 1.19746, 1.11084 * 1.11084, 1.03826 * 1.03826};

static inline double FAST_LOG10_X(double x, double y) { return js_log10(x) * y; }

static double psycho_loudness_approx(const F32* energy, const LjEnc* e) {
  double loudness_power = 0.0;
  for (int i = 0; i < BLKSIZE / 2; ++i) loudness_power += energy[i] * e->ath_eql_w[i];
  loudness_power *= VO_SCALE;
  return loudness_power;
}

static void compute_ffts(LjEnc* e, F32* fftenergy, F32 fftenergy_s[3][HBLKSIZE_s], F32 (*wsamp_L)[BLKSIZE],
                         F32 (*wsamp_S)[3][BLKSIZE_s], int gr_out, int chn, const F32* const* buffers, int bufPos) {
  F32* wsamp_l = wsamp_L[chn & 1];
  F32 (*wsamp_s)[BLKSIZE_s] = wsamp_S[chn & 1];
  if (chn < 2) {
    fft_long(e, wsamp_l, buffers[chn], bufPos);
    fft_short(e, wsamp_s, buffers[chn], bufPos);
  } else if (chn == 2) {
    /* FFT data for mid and side channel is derived from L & R (PsyModel.js:258-275) */
    for (int j = BLKSIZE - 1; j >= 0; --j) {
      double l = wsamp_L[0][j], r = wsamp_L[1][j];
      wsamp_L[0][j] = (l + r) * LJ_SQRT2 * 0.5;
      wsamp_L[1][j] = (l - r) * LJ_SQRT2 * 0.5;
    }
    for (int b = 2; b >= 0; --b)
      for (int j = BLKSIZE_s - 1; j >= 0; --j) {
        double l = wsamp_S[0][b][j], r = wsamp_S[1][b][j];
        wsamp_S[0][b][j] = (l + r) * LJ_SQRT2 * 0.5;
        wsamp_S[1][b][j] = (l - r) * LJ_SQRT2 * 0.5;
      }
  }
  fftenergy[0] = wsamp_l[0];
  fftenergy[0] *= fftenergy[0];
  for (int j = BLKSIZE / 2 - 1; j >= 0; --j) {
    double re = wsamp_l[BLKSIZE / 2 - j];
    double im = wsamp_l[BLKSIZE / 2 + j];
    fftenergy[BLKSIZE / 2 - j] = (re * re + im * im) * 0.5;
  }
  for (int b = 2; b >= 0; --b) {
    fftenergy_s[b][0] = wsamp_s[b][0];
    fftenergy_s[b][0] *= fftenergy_s[b][0];
    for (int j = BLKSIZE_s / 2 - 1; j >= 0; --j) {
      double re = wsamp_s[b][BLKSIZE_s / 2 - j];
      double im = wsamp_s[b][BLKSIZE_s / 2 + j];
      fftenergy_s[b][BLKSIZE_s / 2 - j] = (re * re + im * im) * 0.5;
    }
  }
  {
    double totalenergy = 0.0;
    for (int j = 11; j < HBLKSIZE; j++) totalenergy += fftenergy[j];
    e->tot_ener[chn] = totalenergy;
  }
  /* athaa_loudapprox == 2; no loudness for mid / side */
  if (chn < 2) {
    e->loudness_sq[gr_out][chn] = e->loudness_sq_save[chn];
    e->loudness_sq_save[chn] = psycho_loudness_approx(fftenergy, e);
  }
}

static double mask_add(double m1, double m2, int kk, int b, const LjEnc* e, int shortblock) {
  double ratio;
  if (m2 > m1) {
    if (m2 < (m1 * e->ma_max_i2)) ratio = m2 / m1;
    else return (m1 + m2);
  } else {
    if (m1 >= (m2 * e->ma_max_i2)) return (m1 + m2);
    ratio = m1 / m2;
  }
  m1 += m2;
  if ((b + 3) <= 3 + 3) { /* sic: the unsigned cast of LAME is lost in lamejs */
    if (ratio >= e->ma_max_i1) return m1;
    int i = js_toint32(FAST_LOG10_X(ratio, 16.0));
    return m1 * table2[i];
  }
  int i = js_toint32(FAST_LOG10_X(ratio, 16.0));
  if (shortblock != 0) m2 = e->ath_cb_s[kk] * e->ath_adjust;
  else m2 = e->ath_cb_l[kk] * e->ath_adjust;
  if (m1 < e->ma_max_m * m2) {
    if (m1 > m2) {
      double f, r;
      f = 1.0;
      if (i <= 13) f = table3[i];
      r = FAST_LOG10_X(m1 / m2, 10.0 / 15.0);
      return m1 * ((table1[i] - f) * r + f);
    }
    if (i > 13) return m1;
    return m1 * table3[i];
  }
  return m1 * table1[i];
}

static void calc_interchannel_masking(LjEnc* e, double ratio) {
  if (e->channels_out > 1) {
    for (int sb = 0; sb < SBMAX_l; sb++) {
      double l = e->thm[0].l[sb];
      double r = e->thm[1].l[sb];
      e->thm[0].l[sb] += r * ratio;
      e->thm[1].l[sb] += l * ratio;
    }
    for (int sb = 0; sb < SBMAX_s; sb++) {
      for (int sblock = 0; sblock < 3; sblock++) {
        double l = e->thm[0].s[sb][sblock];
        double r = e->thm[1].s[sb][sblock];
        e->thm[0].s[sb][sblock] += r * ratio;
        e->thm[1].s[sb][sblock] += l * ratio;
      }
    }
  }
}

static void convert_partition2scalefac_s(LjEnc* e, const F32* eb, const F32* thr, int chn, int sblock) {
  int sb, b;
  double enn = 0.0, thmm = 0.0;
  for (sb = b = 0; sb < SBMAX_s; ++b, ++sb) {
    int bo_s_sb = e->bo_s[sb];
    int npart_s = e->npart_s;
    int b_lim = bo_s_sb < npart_s ? bo_s_sb : npart_s;
    while (b < b_lim) { enn += eb[b]; thmm += thr[b]; b++; }
    e->en[chn].s[sb][sblock] = enn;
    e->thm[chn].s[sb][sblock] = thmm;
    if (b >= npart_s) { ++sb; break; }
    {
      double w_curr = e->bo_s_weight[sb];
      double w_next = 1.0 - w_curr;
      enn = w_curr * eb[b];
      thmm = w_curr * thr[b];
      e->en[chn].s[sb][sblock] += enn;
      e->thm[chn].s[sb][sblock] += thmm;
      enn = w_next * eb[b];
      thmm = w_next * thr[b];
    }
  }
  for (; sb < SBMAX_s; ++sb) { e->en[chn].s[sb][sblock] = 0; e->thm[chn].s[sb][sblock] = 0; }
}

static void convert_partition2scalefac_l(LjEnc* e, const F32* eb, const F32* thr, int chn) {
  int sb, b;
  double enn = 0.0, thmm = 0.0;
  for (sb = b = 0; sb < SBMAX_l; ++b, ++sb) {
    int bo_l_sb = e->bo_l[sb];
    int npart_l = e->npart_l;
    int b_lim = bo_l_sb < npart_l ? bo_l_sb : npart_l;
    while (b < b_lim) { enn += eb[b]; thmm += thr[b]; b++; }
    e->en[chn].l[sb] = enn;
    e->thm[chn].l[sb] = thmm;
    if (b >= npart_l) { ++sb; break; }
    {
      double w_curr = e->bo_l_weight[sb];
      double w_next = 1.0 - w_curr;
      enn = w_curr * eb[b];
      thmm = w_curr * thr[b];
      e->en[chn].l[sb] += enn;
      e->thm[chn].l[sb] += thmm;
      enn = w_next * eb[b];
      thmm = w_next * thr[b];
    }
  }
  for (; sb < SBMAX_l; ++sb) { e->en[chn].l[sb] = 0; e->thm[chn].l[sb] = 0; }
}

static void compute_masking_s(LjEnc* e, F32 fftenergy_s[3][HBLKSIZE_s], F32* eb, F32* thr, int chn, int sblock) {
  int j, b;
  for (b = j = 0; b < e->npart_s; ++b) {
    double ebb = 0, m = 0;
    int n = e->numlines_s[b];
    for (int i = 0; i < n; ++i, ++j) {
      double el = fftenergy_s[sblock][j];
      ebb += el;
      if (m < el) m = el;
    }
    eb[b] = ebb;
  }
  for (j = b = 0; b < e->npart_s; b++) {
    int kk = e->s3ind_s[b][0];
    double ecb = e->s3_ss[j++] * eb[kk];
    ++kk;
    while (kk <= e->s3ind_s[b][1]) {
      ecb += e->s3_ss[j] * eb[kk];
      ++j;
      ++kk;
    }
    {
      double x = rpelev_s * e->nb_s1[chn][b];
      thr[b] = js_min(ecb, x);
    }
    if (e->blocktype_old[chn & 1] == SHORT_TYPE) {
      double x = rpelev2_s * e->nb_s2[chn][b];
      double y = thr[b];
      thr[b] = js_min(x, y);
    }
    e->nb_s2[chn][b] = e->nb_s1[chn][b];
    e->nb_s1[chn][b] = ecb;
  }
  for (; b <= CBANDS; ++b) { eb[b] = 0; thr[b] = 0; }
}

static void block_type_set(LjEnc* e, int* uselongblock, int* blocktype_d, int* blocktype) {
  if (e->short_blocks_coupled && !(uselongblock[0] != 0 && uselongblock[1] != 0))
    uselongblock[0] = uselongblock[1] = 0;
  for (int chn = 0; chn < e->channels_out; chn++) {
    blocktype[chn] = NORM_TYPE;
    if (uselongblock[chn] != 0) {
      if (e->blocktype_old[chn] == SHORT_TYPE) blocktype[chn] = STOP_TYPE;
    } else {
      blocktype[chn] = SHORT_TYPE;
      if (e->blocktype_old[chn] == NORM_TYPE) e->blocktype_old[chn] = START_TYPE;
      if (e->blocktype_old[chn] == STOP_TYPE) e->blocktype_old[chn] = SHORT_TYPE;
    }
    blocktype_d[chn] = e->blocktype_old[chn];
    e->blocktype_old[chn] = blocktype[chn];
  }
}

static double NS_INTERP(double x, double y, double r) {
  if (r >= 1.0) return x;
  if (r <= 0.0) return y;
  if (y > 0.0) return (js_pow(x / y, r) * y);
  return 0.0;
}

static const double regcoef_s[12] = {11.8, 13.6, 17.2, 32, 46.5, 51.3, 57.5, 67.1, 71.5, 84.6, 97.6, 130};
static const double regcoef_l[21] = {6.8, 5.8, 5.8, 6.4, 6.5, 9.9, 12.1, 14.4, 15, 18.9, 21.6, 26.9, 34.2, 40.2, 46.8,
                                     56.5, 60.7, 73.9, 85.7, 93.4, 126.1};

static double pecalc_s(const PsyRatio* mr, double masking_lower) {
  double pe_s = 1236.28 / 4;
  for (int sb = 0; sb < SBMAX_s - 1; sb++)
    for (int sblock = 0; sblock < 3; sblock++) {
      double thm = mr->thm.s[sb][sblock];
      if (thm > 0.0) {
        double x = thm * masking_lower;
        double en = mr->en.s[sb][sblock];
        if (en > x) {
          if (en > x * 1e10) pe_s += regcoef_s[sb] * (10.0 * LOG10_C);
          else pe_s += regcoef_s[sb] * js_log10(en / x);
        }
      }
    }
  return pe_s;
}
static double pecalc_l(const PsyRatio* mr, double masking_lower) {
  double pe_l = 1124.23 / 4;
  for (int sb = 0; sb < SBMAX_l - 1; sb++) {
    double thm = mr->thm.l[sb];
    if (thm > 0.0) {
      double x = thm * masking_lower;
      double en = mr->en.l[sb];
      if (en > x) {
        if (en > x * 1e10) pe_l += regcoef_l[sb] * (10.0 * LOG10_C);
        else pe_l += regcoef_l[sb] * js_log10(en / x);
      }
    }
  }
  return pe_l;
}

static void calc_energy(const LjEnc* e, const F32* fftenergy, F32* eb, F32* max, F32* avg) {
  int b, j;
  for (b = j = 0; b < e->npart_l; ++b) {
    double ebb = 0, m = 0;
    for (int i = 0; i < e->numlines_l[b]; ++i, ++j) {
      double el = fftenergy[j];
      ebb += el;
      if (m < el) m = el;
    }
    eb[b] = ebb;
    max[b] = m;
    avg[b] = ebb * e->rnumlines_l[b];
  }
}

static void calc_mask_index_l(const LjEnc* e, const F32* max, const F32* avg, int* mask_idx) {
  const int last_tab_entry = 8;
  int b = 0;
  double a = avg[b] + avg[b + 1];
  if (a > 0.0) {
    double m = max[b];
    if (m < max[b + 1]) m = max[b + 1];
    a = 20.0 * (m * 2.0 - a) / (a * (e->numlines_l[b] + e->numlines_l[b + 1] - 1));
    int k = js_toint32(a);
    if (k > last_tab_entry) k = last_tab_entry;
    mask_idx[b] = k;
  } else mask_idx[b] = 0;
  for (b = 1; b < e->npart_l - 1; b++) {
    a = avg[b - 1] + avg[b] + avg[b + 1];
    if (a > 0.0) {
      double m = max[b - 1];
      if (m < max[b]) m = max[b];
      if (m < max[b + 1]) m = max[b + 1];
      a = 20.0 * (m * 3.0 - a) / (a * (e->numlines_l[b - 1] + e->numlines_l[b] + e->numlines_l[b + 1] - 1));
      int k = js_toint32(a);
      if (k > last_tab_entry) k = last_tab_entry;
      mask_idx[b] = k;
    } else mask_idx[b] = 0;
  }
  a = avg[b - 1] + avg[b];
  if (a > 0.0) {
    double m = max[b - 1];
    if (m < max[b]) m = max[b];
    a = 20.0 * (m * 2.0 - a) / (a * (e->numlines_l[b - 1] + e->numlines_l[b] - 1));
    int k = js_toint32(a);
    if (k > last_tab_entry) k = last_tab_entry;
    mask_idx[b] = k;
  } else mask_idx[b] = 0;
}

static const double fircoef[10] = {-8.65163e-18 * 2, -0.00851586 * 2, -6.74764e-18 * 2, 0.0209036 * 2,
                                   -3.36639e-17 * 2, -0.0438162 * 2, -1.54175e-17 * 2, 0.0931738 * 2,
                                   -5.52212e-17 * 2, -0.313819 * 2};

/* PsyModel.js:548-585 */
static void msfix1(LjEnc* e) {
  for (int sb = 0; sb < SBMAX_l; sb++) {
    if (e->thm[0].l[sb] > 1.58 * e->thm[1].l[sb] || e->thm[1].l[sb] > 1.58 * e->thm[0].l[sb]) continue;
    double mld = e->mld_l[sb] * e->en[3].l[sb];
    double rmid = js_max(e->thm[2].l[sb], js_min(e->thm[3].l[sb], mld));
    mld = e->mld_l[sb] * e->en[2].l[sb];
    double rside = js_max(e->thm[3].l[sb], js_min(e->thm[2].l[sb], mld));
    e->thm[2].l[sb] = rmid;
    e->thm[3].l[sb] = rside;
  }
  for (int sb = 0; sb < SBMAX_s; sb++)
    for (int sblock = 0; sblock < 3; sblock++) {
      if (e->thm[0].s[sb][sblock] > 1.58 * e->thm[1].s[sb][sblock] || e->thm[1].s[sb][sblock] > 1.58 * e->thm[0].s[sb][sblock]) continue;
      double mld = e->mld_s[sb] * e->en[3].s[sb][sblock];
      double rmid = js_max(e->thm[2].s[sb][sblock], js_min(e->thm[3].s[sb][sblock], mld));
      mld = e->mld_s[sb] * e->en[2].s[sb][sblock];
      double rside = js_max(e->thm[3].s[sb][sblock], js_min(e->thm[2].s[sb][sblock], mld));
      e->thm[2].s[sb][sblock] = rmid;
      e->thm[3].s[sb][sblock] = rside;
    }
}

/* PsyModel.js:591-640 */
static void ns_msfix(LjEnc* e, double msfix, double athadjust) {
  double msfix2 = msfix;
  double athlower = js_pow(10, athadjust);
  msfix *= 2.0;
  msfix2 *= 2.0;
  for (int sb = 0; sb < SBMAX_l; sb++) {
    double thmLR, thmM, thmS, ath;
    ath = (e->ath_cb_l[e->bm_l[sb]]) * athlower;
    thmLR = js_min(js_max(e->thm[0].l[sb], ath), js_max(e->thm[1].l[sb], ath));
    thmM = js_max(e->thm[2].l[sb], ath);
    thmS = js_max(e->thm[3].l[sb], ath);
    if (thmLR * msfix < thmM + thmS) {
      double f = thmLR * msfix2 / (thmM + thmS);
      thmM *= f;
      thmS *= f;
    }
    e->thm[2].l[sb] = js_min(thmM, e->thm[2].l[sb]);
    e->thm[3].l[sb] = js_min(thmS, e->thm[3].l[sb]);
  }
  athlower *= ((double)BLKSIZE_s / BLKSIZE);
  for (int sb = 0; sb < SBMAX_s; sb++)
    for (int sblock = 0; sblock < 3; sblock++) {
      double thmLR, thmM, thmS, ath;
      ath = (e->ath_cb_s[e->bm_s[sb]]) * athlower;
      thmLR = js_min(js_max(e->thm[0].s[sb][sblock], ath), js_max(e->thm[1].s[sb][sblock], ath));
      thmM = js_max(e->thm[2].s[sb][sblock], ath);
      thmS = js_max(e->thm[3].s[sb][sblock], ath);
      if (thmLR * msfix < thmM + thmS) {
        double f = thmLR * msfix / (thmM + thmS);
        thmM *= f;
        thmS *= f;
      }
      e->thm[2].s[sb][sblock] = js_min(e->thm[2].s[sb][sblock], thmM);
      e->thm[3].s[sb][sblock] = js_min(e->thm[3].s[sb][sblock], thmS);
    }
}

int lj_psycho_anal_ns(LjEnc* e, const F32* buf0, const F32* buf1, int bufPos, int gr_out,
                      PsyRatio masking_ratio[2][2], PsyRatio masking_MS_ratio[2][2], double* percep_entropy,
                      double* percep_MS_entropy, F32* energy, int* blocktype_d) {
  const F32* buffer[2] = {buf0, buf1};
  static thread_local F32 wsamp_L[2][BLKSIZE];
  static thread_local F32 wsamp_S[2][3][BLKSIZE_s];
  F32 eb_l[CBANDS + 1], eb_s[CBANDS + 1], thr[CBANDS + 2];
  int blocktype[2], uselongblock[2] = {0, 0};
  int numchn, chn, b, i, j, k, sb, sblock;
  static thread_local F32 ns_hpfsmpl[2][576];
  double pcfact;
  int mask_idx_l[CBANDS + 2];
  const int NSFIRLEN = 21;

  numchn = e->channels_out;
  if (e->mode_joint) numchn = 4;           /* chn 2 and 3 = mid and side (PsyModel.js:1031-1034) */
  pcfact = e->ResvMax == 0 ? 0 : ((double)e->ResvSize) / e->ResvMax * 0.5;

  for (chn = 0; chn < e->channels_out; chn++) {
    const F32* firbuf = buffer[chn];
    int firbufPos = bufPos + 576 - 350 - NSFIRLEN + 192;
    for (i = 0; i < 576; i++) {
      double sum1, sum2;
      sum1 = firbuf[firbufPos + i + 10];
      sum2 = 0.0;
      for (j = 0; j < ((NSFIRLEN - 1) / 2) - 1; j += 2) {
        sum1 += fircoef[j] * (firbuf[firbufPos + i + j] + firbuf[firbufPos + i + NSFIRLEN - j]);
        sum2 += fircoef[j + 1] * (firbuf[firbufPos + i + j + 1] + firbuf[firbufPos + i + NSFIRLEN - j - 1]);
      }
      ns_hpfsmpl[chn][i] = sum1 + sum2;
    }
    masking_ratio[gr_out][chn].en = e->en[chn];
    masking_ratio[gr_out][chn].thm = e->thm[chn];
    if (numchn > 2) {
      masking_MS_ratio[gr_out][chn].en = e->en[chn + 2];
      masking_MS_ratio[gr_out][chn].thm = e->thm[chn + 2];
    }
  }

  for (chn = 0; chn < numchn; chn++) {
    F32 en_subshort[12];
    double en_short[4] = {0, 0, 0, 0};       /* plain JS array: doubles */
    F32 attack_intensity[12];
    int ns_uselongblock = 1;
    double attackThreshold;
    F32 max[CBANDS], avg[CBANDS];
    int ns_attacks[4] = {0, 0, 0, 0};
    F32 fftenergy[HBLKSIZE];
    F32 fftenergy_s[3][HBLKSIZE_s];

    for (i = 0; i < 3; i++) {
      en_subshort[i] = e->last_en_subshort[chn][i + 6];
      attack_intensity[i] = en_subshort[i] / e->last_en_subshort[chn][i + 4];
      en_short[0] += en_subshort[i];
    }
    if (chn == 2) {
      for (i = 0; i < 576; i++) {
        double l = ns_hpfsmpl[0][i], r = ns_hpfsmpl[1][i];
        ns_hpfsmpl[0][i] = l + r;
        ns_hpfsmpl[1][i] = l - r;
      }
    }
    {
      const F32* pf = ns_hpfsmpl[chn & 1];
      int pfPos = 0;
      for (i = 0; i < 9; i++) {
        int pfe = pfPos + 576 / 9;
        double p = 1.;
        for (; pfPos < pfe; pfPos++)
          if (p < fabs(pf[pfPos])) p = fabs(pf[pfPos]);
        e->last_en_subshort[chn][i] = en_subshort[i + 3] = p;
        /* en_short[1 + i / 3] += p  with a FRACTIONAL index: only i % 3 == 0 hits a real element */
        if (i % 3 == 0) en_short[1 + i / 3] += p;
        if (p > en_subshort[i + 3 - 2]) p = p / en_subshort[i + 3 - 2];
        else if (en_subshort[i + 3 - 2] > p * 10.0) p = en_subshort[i + 3 - 2] / (p * 10.0);
        else p = 0.0;
        attack_intensity[i + 3] = p;
      }
    }
    attackThreshold = (chn == 3) ? e->attackthre_s : e->attackthre;
    for (i = 0; i < 12; i++) {
      /* ns_attacks[i / 3] with a fractional index is `undefined`; 0 == undefined is false */
      if (i % 3 != 0) continue;
      if (0 == ns_attacks[i / 3] && attack_intensity[i] > attackThreshold) ns_attacks[i / 3] = (i % 3) + 1;
    }
    for (i = 1; i < 4; i++) {
      double ratio;
      if (en_short[i - 1] > en_short[i]) ratio = en_short[i - 1] / en_short[i];
      else ratio = en_short[i] / en_short[i - 1];
      if (ratio < 1.7) {
        ns_attacks[i] = 0;
        if (i == 1) ns_attacks[0] = 0;
      }
    }
    lj_psy_trace_attacks(e, gr_out, chn, en_subshort, ns_attacks);
    if (ns_attacks[0] != 0 && e->lastAttacks[chn] != 0) ns_attacks[0] = 0;
    if (e->lastAttacks[chn] == 3 || (ns_attacks[0] + ns_attacks[1] + ns_attacks[2] + ns_attacks[3]) != 0) {
      ns_uselongblock = 0;
      if (ns_attacks[1] != 0 && ns_attacks[0] != 0) ns_attacks[1] = 0;
      if (ns_attacks[2] != 0 && ns_attacks[1] != 0) ns_attacks[2] = 0;
      if (ns_attacks[3] != 0 && ns_attacks[2] != 0) ns_attacks[3] = 0;
    }
    if (chn < 2) uselongblock[chn] = ns_uselongblock;
    else if (ns_uselongblock == 0) uselongblock[0] = uselongblock[1] = 0;
    energy[chn] = e->tot_ener[chn];

    compute_ffts(e, fftenergy, fftenergy_s, wsamp_L, wsamp_S, gr_out, chn, buffer, bufPos);
    calc_energy(e, fftenergy, eb_l, max, avg);
    calc_mask_index_l(e, max, avg, mask_idx_l);
    lj_psy_trace_long(e, gr_out, chn, eb_l, mask_idx_l);
    for (sblock = 0; sblock < 3; sblock++) {
      double enn, thmm;
      compute_masking_s(e, fftenergy_s, eb_s, thr, chn, sblock);
      lj_psy_trace_short(e, gr_out, chn, sblock, eb_s);
      convert_partition2scalefac_s(e, eb_s, thr, chn, sblock);
      for (sb = 0; sb < SBMAX_s; sb++) {
        thmm = e->thm[chn].s[sb][sblock];
        thmm *= 0.8; /* NS_PREECHO_ATT0 */
        if (ns_attacks[sblock] >= 2 || ns_attacks[sblock + 1] == 1) {
          int idx = (sblock != 0) ? sblock - 1 : 2;
          double p = NS_INTERP(e->thm[chn].s[sb][idx], thmm, 0.6 * pcfact);
          thmm = js_min(thmm, p);
        }
        if (ns_attacks[sblock] == 1) {
          int idx = (sblock != 0) ? sblock - 1 : 2;
          double p = NS_INTERP(e->thm[chn].s[sb][idx], thmm, 0.3 * pcfact);
          thmm = js_min(thmm, p);
        } else if ((sblock != 0 && ns_attacks[sblock - 1] == 3) || (sblock == 0 && e->lastAttacks[chn] == 3)) {
          int idx = (sblock != 2) ? sblock + 1 : 0;
          double p = NS_INTERP(e->thm[chn].s[sb][idx], thmm, 0.3 * pcfact);
          thmm = js_min(thmm, p);
        }
        enn = en_subshort[sblock * 3 + 3] + en_subshort[sblock * 3 + 4] + en_subshort[sblock * 3 + 5];
        if (en_subshort[sblock * 3 + 5] * 6 < enn) {
          thmm *= 0.5;
          if (en_subshort[sblock * 3 + 4] * 6 < enn) thmm *= 0.5;
        }
        e->thm[chn].s[sb][sblock] = thmm;
      }
    }
    e->lastAttacks[chn] = ns_attacks[2];

    k = 0;
    for (b = 0; b < e->npart_l; b++) {
      int kk = e->s3ind[b][0];
      double eb2 = eb_l[kk] * tab[mask_idx_l[kk]];
      double ecb = e->s3_ll[k++] * eb2;
      while (++kk <= e->s3ind[b][1]) {
        eb2 = eb_l[kk] * tab[mask_idx_l[kk]];
        ecb = mask_add(ecb, e->s3_ll[k++] * eb2, kk, kk - b, e, 0);
      }
      ecb *= 0.158489319246111;
      if (e->blocktype_old[chn & 1] == SHORT_TYPE) thr[b] = ecb;
      else thr[b] = NS_INTERP(js_min(ecb, js_min(rpelev * e->nb_1[chn][b], rpelev2 * e->nb_2[chn][b])), ecb, pcfact);
      e->nb_2[chn][b] = e->nb_1[chn][b];
      e->nb_1[chn][b] = ecb;
    }
    for (; b <= CBANDS; ++b) { eb_l[b] = 0; thr[b] = 0; }
    convert_partition2scalefac_l(e, eb_l, thr, chn);
  }

  if (!e->mode_mono) {
    if (e->interChRatio > 0.0) calc_interchannel_masking(e, e->interChRatio);
  }
  if (e->mode_joint) {
    msfix1(e);
    double msfix = e->msfix;
    if (fabs(msfix) > 0.0) ns_msfix(e, msfix, e->ATHlower * e->ath_adjust);
  }
  block_type_set(e, uselongblock, blocktype_d, blocktype);
  for (chn = 0; chn < numchn; chn++) {
    if (chn > 1) {
      int type = NORM_TYPE;
      if (blocktype_d[0] == SHORT_TYPE || blocktype_d[1] == SHORT_TYPE) type = SHORT_TYPE;
      const PsyRatio* mr = &masking_MS_ratio[gr_out][chn - 2];
      if (type == SHORT_TYPE) percep_MS_entropy[chn - 2] = pecalc_s(mr, e->masking_lower);
      else percep_MS_entropy[chn - 2] = pecalc_l(mr, e->masking_lower);
    } else {
      int type = blocktype_d[chn];
      const PsyRatio* mr = &masking_ratio[gr_out][chn];
      if (type == SHORT_TYPE) percep_entropy[chn] = pecalc_s(mr, e->masking_lower);
      else percep_entropy[chn] = pecalc_l(mr, e->masking_lower);
    }
  }
  return 0;
}

/* ------------------------------------------------------------------ init */
static double ATHformula_GB(double f, double value) {
  if (f < -.3) f = 3410;
  f /= 1000;
  f = js_max(0.1, f);
  double ath = 3.640 * js_pow(f, -0.8) - 6.800 * js_exp(-0.6 * js_pow(f - 3.4, 2.0)) +
               6.000 * js_exp(-0.15 * js_pow(f - 8.7, 2.0)) + (0.6 + 0.04 * value) * 0.001 * js_pow(f, 4.0);
  return ath;
}
double lj_ATHformula(double f, const LjEnc* e) {
  switch (e->ATHtype) {
    case 0: return ATHformula_GB(f, 9);
    case 1: return ATHformula_GB(f, -1);
    case 2: return ATHformula_GB(f, 0);
    case 3: return ATHformula_GB(f, 1) + 6;
    case 4: return ATHformula_GB(f, e->ATHcurve);
    default: return ATHformula_GB(f, 0);
  }
}

static double s3_func(double bark) {
  double tempx, x, tempy, temp;
  tempx = bark;
  if (tempx >= 0) tempx *= 3;
  else tempx *= 1.5;
  if (tempx >= 0.5 && tempx <= 2.5) {
    temp = tempx - 0.5;
    x = 8.0 * (temp * temp - 2.0 * temp);
  } else x = 0.0;
  tempx += 0.474;
  tempy = 15.811389 + 7.5 * tempx - 17.5 * sqrt(1.0 + tempx * tempx);
  if (tempy <= -60.0) return 0.0;
  tempx = js_exp((x + tempy) * LN_TO_LOG10);
  tempx /= .6609193;
  return tempx;
}

static double freq2bark(double freq) {
  if (freq < 0) freq = 0;
  freq = freq * 0.001;
  return 13.0 * atan(.76 * freq) + 3.5 * atan(freq * freq / (7.5 * 7.5));
}

static int init_numline(int* numlines, int* bo, int* bm, F32* bval, F32* bval_width, F32* mld, F32* bo_w,
                        double sfreq, int blksize, const int* scalepos, double deltafreq, int sbmax) {
  F32 b_frq[CBANDS + 1];
  double sample_freq_frac = sfreq / (sbmax > 15 ? 2 * 576 : 2 * 192);
  int partition[HBLKSIZE];
  int i;
  memset(partition, 0, sizeof partition);
  sfreq /= blksize;
  int j = 0;
  int ni = 0;
  for (i = 0; i < CBANDS; i++) {
    double bark1;
    int j2;
    bark1 = freq2bark(sfreq * j);
    b_frq[i] = sfreq * j;
    for (j2 = j; freq2bark(sfreq * j2) - bark1 < DELBARK && j2 <= blksize / 2; j2++)
      ;
    numlines[i] = j2 - j;
    ni = i + 1;
    while (j < j2) partition[j++] = i;
    if (j > blksize / 2) {
      j = blksize / 2;
      ++i;
      break;
    }
  }
  b_frq[i] = sfreq * j;
  for (int sfb = 0; sfb < sbmax; sfb++) {
    int i1, i2, start, end;
    double arg;
    start = scalepos[sfb];
    end = scalepos[sfb + 1];
    i1 = js_toint32(floor(.5 + deltafreq * (start - .5)));
    if (i1 < 0) i1 = 0;
    i2 = js_toint32(floor(.5 + deltafreq * (end - .5)));
    if (i2 > blksize / 2) i2 = blksize / 2;
    bm[sfb] = js_toint32((partition[i1] + partition[i2]) / 2.0); /* JS float division, Int32Array store */
    bo[sfb] = partition[i2];
    double f_tmp = sample_freq_frac * end;
    bo_w[sfb] = (f_tmp - b_frq[bo[sfb]]) / (b_frq[bo[sfb] + 1] - b_frq[bo[sfb]]);
    if (bo_w[sfb] < 0) bo_w[sfb] = 0;
    else if (bo_w[sfb] > 1) bo_w[sfb] = 1;
    arg = freq2bark(sfreq * scalepos[sfb] * deltafreq);
    arg = (js_min(arg, 15.5) / 15.5);
    mld[sfb] = js_pow(10.0, 1.25 * (1 - cos(M_PI * arg)) - 2.5);
  }
  j = 0;
  for (int k = 0; k < ni; k++) {
    int w = numlines[k];
    double bark1, bark2;
    bark1 = freq2bark(sfreq * (j));
    bark2 = freq2bark(sfreq * (j + w - 1));
    bval[k] = .5 * (bark1 + bark2);
    bark1 = freq2bark(sfreq * (j - .5));
    bark2 = freq2bark(sfreq * (j + w - .5));
    bval_width[k] = bark2 - bark1;
    j += w;
  }
  return ni;
}

static F32* init_s3_values(int s3ind[CBANDS][2], int npart, const F32* bval, const F32* bval_width, const F32* norm, int* count) {
  static thread_local F32 s3[CBANDS][CBANDS];
  memset(s3, 0, sizeof s3);
  int j;
  int numberOfNoneZero = 0;
  for (int i = 0; i < npart; i++)
    for (j = 0; j < npart; j++) {
      double v = s3_func(bval[i] - bval[j]) * bval_width[j];
      s3[i][j] = v * norm[i];
    }
  for (int i = 0; i < npart; i++) {
    for (j = 0; j < npart; j++) if (s3[i][j] > 0.0) break;
    s3ind[i][0] = j;
    for (j = npart - 1; j > 0; j--) if (s3[i][j] > 0.0) break;
    s3ind[i][1] = j;
    numberOfNoneZero += (s3ind[i][1] - s3ind[i][0] + 1);
  }
  F32* p = (F32*)calloc(numberOfNoneZero > 0 ? numberOfNoneZero : 1, sizeof(F32));
  int k = 0;
  for (int i = 0; i < npart; i++)
    for (j = s3ind[i][0]; j <= s3ind[i][1]; j++) p[k++] = s3[i][j];
  *count = numberOfNoneZero;
  return p;
}

void lj_psymodel_init(LjEnc* e) {
  int i;
  double bvl_a = 13, bvl_b = 24;
  double snr_l_a = 0, snr_l_b = 0;
  double snr_s_a = -8.25, snr_s_b = -4.5;
  F32 bval[CBANDS], bval_width[CBANDS], norm[CBANDS];
  double sfreq = e->out_samplerate;

  e->blocktype_old[0] = e->blocktype_old[1] = NORM_TYPE;
  for (i = 0; i < 4; ++i) {
    for (int j = 0; j < CBANDS; ++j) {
      e->nb_1[i][j] = 1e20; e->nb_2[i][j] = 1e20;
      e->nb_s1[i][j] = e->nb_s2[i][j] = 1.0;
    }
    for (int sb = 0; sb < SBMAX_l; sb++) { e->en[i].l[sb] = 1e20; e->thm[i].l[sb] = 1e20; }
    for (int j = 0; j < 3; ++j) {
      for (int sb = 0; sb < SBMAX_s; sb++) { e->en[i].s[sb][j] = 1e20; e->thm[i].s[sb][j] = 1e20; }
      e->lastAttacks[i] = 0;
    }
    for (int j = 0; j < 9; j++) e->last_en_subshort[i][j] = 10.;
  }
  e->loudness_sq_save[0] = e->loudness_sq_save[1] = 0.0;

  e->npart_l = init_numline(e->numlines_l, e->bo_l, e->bm_l, bval, bval_width, e->mld_l, e->bo_l_weight, sfreq,
                            BLKSIZE, e->sfb_l, BLKSIZE / (2.0 * 576), SBMAX_l);
  for (i = 0; i < e->npart_l; i++) {
    double snr = snr_l_a;
    if (bval[i] >= bvl_a) snr = snr_l_b * (bval[i] - bvl_a) / (bvl_b - bvl_a) + snr_l_a * (bvl_b - bval[i]) / (bvl_b - bvl_a);
    norm[i] = js_pow(10.0, snr / 10.0);
    if (e->numlines_l[i] > 0) e->rnumlines_l[i] = 1.0 / e->numlines_l[i];
    else e->rnumlines_l[i] = 0;
  }
  e->s3_ll = init_s3_values(e->s3ind, e->npart_l, bval, bval_width, norm, &e->n_s3_ll);

  int j = 0;
  for (i = 0; i < e->npart_l; i++) {
    double x;
    x = 3.4028235e+38;
    for (int k = 0; k < e->numlines_l[i]; k++, j++) {
      double freq = sfreq * j / (1000.0 * BLKSIZE);
      double level;
      level = lj_ATHformula(freq * 1000, e) - 20;
      level = js_pow(10., 0.1 * level);
      level *= e->numlines_l[i];
      if (x > level) x = level;
    }
    e->ath_cb_l[i] = x;
    x = -20 + bval[i] * 20 / 10;
    if (x > 6) x = 100;
    if (x < -15) x = -15;
    x -= 8.;
    e->minval_l[i] = (js_pow(10.0, x / 10.) * e->numlines_l[i]);
  }

  e->npart_s = init_numline(e->numlines_s, e->bo_s, e->bm_s, bval, bval_width, e->mld_s, e->bo_s_weight, sfreq,
                            BLKSIZE_s, e->sfb_s, BLKSIZE_s / (2.0 * 192), SBMAX_s);
  j = 0;
  for (i = 0; i < e->npart_s; i++) {
    double x;
    double snr = snr_s_a;
    if (bval[i] >= bvl_a) snr = snr_s_b * (bval[i] - bvl_a) / (bvl_b - bvl_a) + snr_s_a * (bvl_b - bval[i]) / (bvl_b - bvl_a);
    norm[i] = js_pow(10.0, snr / 10.0);
    x = 3.4028235e+38;
    for (int k = 0; k < e->numlines_s[i]; k++, j++) {
      double freq = sfreq * j / (1000.0 * BLKSIZE_s);
      double level;
      level = lj_ATHformula(freq * 1000, e) - 20;
      level = js_pow(10., 0.1 * level);
      level *= e->numlines_s[i];
      if (x > level) x = level;
    }
    e->ath_cb_s[i] = x;
    x = (-7.0 + bval[i] * 7.0 / 12.0);
    if (bval[i] > 12) x *= 1 + js_log(1 + x) * 3.1;
    if (bval[i] < 12) x *= 1 + js_log(1 - x) * 2.3;
    if (x < -15) x = -15;
    x -= 8;
    e->minval_s[i] = js_pow(10.0, x / 10) * e->numlines_s[i];
  }
  e->s3_ss = init_s3_values(e->s3ind_s, e->npart_s, bval, bval_width, norm, &e->n_s3_ss);

  e->ma_max_i1 = js_pow(10, (8 + 1) / 16.0);
  e->ma_max_i2 = js_pow(10, (23 + 1) / 16.0);
  e->ma_max_m = js_pow(10, (15) / 10.0);
  init_fft(e);

  e->decay = js_exp(-1.0 * LOG10_C / (0.01 * sfreq / 192.0));
  {
    double msfix = 3.5;
    if ((e->exp_nspsytune & 2) != 0) msfix = 1.0;
    if (fabs(e->msfix) > 0.0) msfix = e->msfix;
    e->msfix = msfix;
    for (int b = 0; b < e->npart_l; b++)
      if (e->s3ind[b][1] > e->npart_l - 1) e->s3ind[b][1] = e->npart_l - 1;
  }
  double frame_duration = (576. * e->mode_gr / sfreq);
  e->ath_decay = js_pow(10., -12. / 10. * frame_duration);
  e->ath_adjust = 0.01;
  e->ath_adjustLimit = 1.0;
  {
    double freq;
    double freq_inc = (double)e->out_samplerate / (BLKSIZE);
    double eql_balance = 0.0;
    freq = 0.0;
    for (i = 0; i < BLKSIZE / 2; ++i) {
      freq += freq_inc;
      e->ath_eql_w[i] = 1. / js_pow(10, lj_ATHformula(freq, e) / 10);
      eql_balance += e->ath_eql_w[i];
    }
    eql_balance = 1.0 / eql_balance;
    for (i = BLKSIZE / 2; --i >= 0;) e->ath_eql_w[i] *= eql_balance;
  }
  /* mld_cb_l / mld_cb_s are only read by the M/S path: not built */
}
