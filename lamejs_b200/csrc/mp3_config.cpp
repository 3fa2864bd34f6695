/* mp3_config.cpp -- host-side derivation of the per-configuration constant block (see mp3_config.h).
 *
 * Product code (not the oracle).  The formulas are the ones lamejs evaluates at construction time; each
 * builder below cites the reference lines it must agree with.  Arithmetic discipline: doubles everywhere,
 * rounding to float32 exactly where lamejs stores into a Float32Array (the `float` members of Mp3Tables),
 * ToInt32 where it stores into an Int32Array.  Math.pow/log10/exp/log come from mp3_math.cuh (fdlibm);
 * cos/atan/sqrt from libm (init-time only, see DESIGN.md "transcendentals").
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "mp3_config.h"
#include "mp3_math.cuh"
#include "mp3_tables.h"

namespace {

/* Tables.js:494-498: [0] MPEG-2, [1] MPEG-1, [2] MPEG-2.5 */
const int kBitrates[3][15] = {{0, 8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160},
                              {0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320},
                              {0, 8, 16, 24, 32, 40, 48, 56, 64, -1, -1, -1, -1, -1, -1}};
const int kFullBitrates[17] = {8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320};
/* optimum_bandwidth() low-pass table, Lame.js:456-464 */
const int kLowpassHz[17] = {2000, 3700, 3900, 5500, 7000, 7500, 10000, 11000, 13500, 15100, 15600,
                            17000, 17500, 18600, 19400, 19700, 20500};
/* the columns of abr_switch_map that Mp3Encoder can reach (Presets.js:226-244) */
struct Preset { int safejoint; double attack, scale, mask_adj, ath_lower, ath_curve, interch; int sfscale; };
const Preset kPresets[17] = {
    {0, 6.60, 0.95, 0, -30.0, 11, 0.0012, 1}, {0, 6.60, 0.95, 0, -25.0, 11, 0.0010, 1},
    {0, 6.60, 0.95, 0, -20.0, 11, 0.0010, 1}, {0, 6.60, 0.95, 0, -15.0, 11, 0.0010, 1},
    {0, 6.60, 0.95, 0, -10.0, 11, 0.0009, 1}, {0, 6.60, 0.95, 0, -10.0, 11, 0.0009, 1},
    {0, 6.60, 0.95, 0, -6.0, 11, 0.0008, 1},  {0, 6.60, 0.95, 0, -2.0, 11, 0.0008, 1},
    {0, 6.60, 0.95, 0, .0, 8, 0.0007, 1},     {0, 6.60, 0.95, 0, 1.0, 5.5, 0.0006, 1},
    {0, 6.60, 0.95, 0, 2.0, 4.5, 0.0005, 1},  {0, 6.40, 0.95, 0, 3.0, 4, 0.0002, 1},
    {1, 6.00, 0.95, -2, 5.0, 3.5, 0, 1},      {1, 5.60, 0.97, -4, 7.0, 3, 0, 0},
    {1, 5.20, 0.98, -6, 9.0, 2, 0, 0},        {1, 5.20, 1.00, -8, 10.0, 1, 0, 0},
    {1, 5.20, 1.00, -10, 12.0, 0, 0, 0}};

/* QuantizePVT.js:137-204 sfBandIndex, index = samplerate_index + 3 * version + 6 * (rate < 16 kHz):
 * 22.05, 24, 16 kHz (MPEG-2); 44.1, 48, 32 kHz (MPEG-1); 11.025, 12, 8 kHz (MPEG-2.5) */
const int kSfbLong[9][23] = {
    {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576},
    {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 114, 136, 162, 194, 232, 278, 332, 394, 464, 540, 576},
    {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576},
    {0, 4, 8, 12, 16, 20, 24, 30, 36, 44, 52, 62, 74, 90, 110, 134, 162, 196, 238, 288, 342, 418, 576},
    {0, 4, 8, 12, 16, 20, 24, 30, 36, 42, 50, 60, 72, 88, 106, 128, 156, 190, 230, 276, 330, 384, 576},
    {0, 4, 8, 12, 16, 20, 24, 30, 36, 44, 54, 66, 82, 102, 126, 156, 194, 240, 296, 364, 448, 550, 576},
    {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576},
    {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576},
    {0, 12, 24, 36, 48, 60, 72, 88, 108, 132, 160, 192, 232, 280, 336, 400, 476, 566, 568, 570, 572, 574, 576}};
const int kSfbShort[9][14] = {{0, 4, 8, 12, 18, 24, 32, 42, 56, 74, 100, 132, 174, 192},
                              {0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 136, 180, 192},
                              {0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 134, 174, 192},
                              {0, 4, 8, 12, 16, 22, 30, 40, 52, 66, 84, 106, 136, 192},
                              {0, 4, 8, 12, 16, 22, 28, 38, 50, 64, 80, 100, 126, 192},
                              {0, 4, 8, 12, 16, 22, 30, 42, 58, 78, 104, 138, 180, 192},
                              {0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 134, 174, 192},
                              {0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 134, 174, 192},
                              {0, 8, 16, 24, 36, 52, 72, 96, 124, 160, 162, 164, 166, 192}};

inline int to_i32(double d) {  /* ToInt32 for the finite, in-range values that occur at init */
  return (int)d;
}
inline double dmin(double a, double b) { return a < b ? a : b; }

/* index of the nearest entry of the 17-step bitrate ladder (Lame.js:248-283) */
int ladder_index(int kbps) {
  int lo = 16, hi = 16;
  for (int b = 0; b < 16; b++) {
    if (kFullBitrates[b + 1] > kbps) { hi = b + 1; lo = b; break; }
  }
  return (kFullBitrates[hi] - kbps) > (kbps - kFullBitrates[lo]) ? lo : hi;
}

/* output sample rate lamejs would pick (Lame.js:285-364); we only accept in == out */
int suggested_out_rate(int lowpass, int in_rate) {
  static const int rates[9] = {48000, 44100, 32000, 24000, 22050, 16000, 12000, 11025, 8000};
  int s = 44100;
  for (int i = 0; i < 9; i++) if (in_rate >= rates[i]) { s = rates[i]; break; }
  static const int lp_limit[8] = {15960, 15250, 11220, 9970, 7230, 5420, 4510, 3970};
  static const int lp_rate[8] = {44100, 32000, 24000, 22050, 16000, 12000, 11025, 8000};
  for (int i = 0; i < 8; i++) if (lowpass <= lp_limit[i]) s = lp_rate[i];
  if (in_rate < s) {
    static const int up[8] = {44100, 32000, 24000, 22050, 16000, 12000, 11025, 8000};
    static const int to[8] = {48000, 44100, 32000, 24000, 22050, 16000, 12000, 11025};
    for (int i = 0; i < 8; i++) if (in_rate > up[i]) return to[i];
    return 8000;
  }
  return s;
}

/* absolute threshold of hearing, dB (PsyModel.js:2827-2894, ATHtype 4) */
double ath_db(double f_hz, double curve) {
  double f = f_hz;
  if (f < -.3) f = 3410;
  f /= 1000;
  if (!(f > 0.1)) f = 0.1;
  return 3.640 * m3_pow(f, -0.8) - 6.800 * m3_exp(-0.6 * m3_pow(f - 3.4, 2.0)) +
         6.000 * m3_exp(-0.15 * m3_pow(f - 8.7, 2.0)) + (0.6 + 0.04 * curve) * 0.001 * m3_pow(f, 4.0);
}

double bark_of(double freq) {  /* PsyModel.js:2356-2363 */
  if (freq < 0) freq = 0;
  freq = freq * 0.001;
  return 13.0 * atan(.76 * freq) + 3.5 * atan(freq * freq / (7.5 * 7.5));
}

double spreading(double bark) {  /* s3_func, PsyModel.js:2317-2351 */
  double tx = bark, x, ty;
  tx *= (tx >= 0) ? 3 : 1.5;
  if (tx >= 0.5 && tx <= 2.5) { double tmp = tx - 0.5; x = 8.0 * (tmp * tmp - 2.0 * tmp); }
  else x = 0.0;
  tx += 0.474;
  ty = 15.811389 + 7.5 * tx - 17.5 * sqrt(1.0 + tx * tx);
  if (ty <= -60.0) return 0.0;
  tx = m3_exp((x + ty) * 0.2302585093);
  tx /= .6609193;
  return tx;
}

struct PartitionLayout { float bval[MP3_CBANDS], bwidth[MP3_CBANDS]; int npart; };

/* init_numline(), PsyModel.js:2365-2458.  Outputs numlines, bo, bo_weight and the bark centre/width of
 * each partition (mld/bm are only used by the M/S path and are not produced). */
void layout_partitions(double sfreq, int blksize, const int* sfb_edges, int nsfb, double deltafreq, int* numlines,
                       int* bo, float* bo_w, PartitionLayout* lay) {
  float b_frq[MP3_CBANDS + 1];
  int part_of_line[513];
  memset(part_of_line, 0, sizeof part_of_line);
  const double frac = sfreq / (nsfb > 15 ? 2 * 576 : 2 * 192);
  const double bin_hz = sfreq / blksize;
  int j = 0, ni = 0, i;
  for (i = 0; i < MP3_CBANDS; i++) {
    const double bark1 = bark_of(bin_hz * j);
    b_frq[i] = (float)(bin_hz * j);
    int j2 = j;
    while (bark_of(bin_hz * j2) - bark1 < .34 && j2 <= blksize / 2) j2++;
    numlines[i] = j2 - j;
    ni = i + 1;
    while (j < j2) part_of_line[j++] = i;
    if (j > blksize / 2) { j = blksize / 2; ++i; break; }
  }
  b_frq[i] = (float)(bin_hz * j);
  for (int sfb = 0; sfb < nsfb; sfb++) {
    const int end = sfb_edges[sfb + 1];
    int i2 = to_i32(floor(.5 + deltafreq * (end - .5)));
    if (i2 > blksize / 2) i2 = blksize / 2;
    bo[sfb] = part_of_line[i2];
    const double f_tmp = frac * end;
    float w = (float)((f_tmp - (double)b_frq[bo[sfb]]) / ((double)b_frq[bo[sfb] + 1] - (double)b_frq[bo[sfb]]));
    if (w < 0) w = 0; else if (w > 1) w = 1;
    bo_w[sfb] = w;
  }
  j = 0;
  for (int k = 0; k < ni; k++) {
    const int w = numlines[k];
    lay->bval[k] = (float)(.5 * (bark_of(bin_hz * j) + bark_of(bin_hz * (j + w - 1))));
    lay->bwidth[k] = (float)(bark_of(bin_hz * (j + w - .5)) - bark_of(bin_hz * (j - .5)));
    j += w;
  }
  lay->npart = ni;
}

/* init_s3_values(), PsyModel.js:2460-2520 (useOldS3): ragged rows of the spreading matrix */
int build_spreading(const PartitionLayout& lay, const float* norm, int* lo, int* hi, int* off, float* flat) {
  const int n = lay.npart;
  static thread_local float s3[MP3_CBANDS][MP3_CBANDS];
  for (int i = 0; i < n; i++)
    for (int j = 0; j < n; j++)
      s3[i][j] = (float)((spreading((double)lay.bval[i] - (double)lay.bval[j]) * (double)lay.bwidth[j]) * (double)norm[i]);
  int total = 0;
  for (int i = 0; i < n; i++) {
    int j;
    for (j = 0; j < n; j++) if (s3[i][j] > 0.0f) break;
    lo[i] = j;
    for (j = n - 1; j > 0; j--) if (s3[i][j] > 0.0f) break;
    hi[i] = j;
    off[i] = total;
    for (j = lo[i]; j <= hi[i]; j++) {
      if (total >= MP3_S3_MAX) return -1;
      flat[total++] = s3[i][j];
    }
  }
  off[n] = total;
  return total;
}

float snr_norm(double bval, double a, double b) {  /* PsyModel.js:2609-2614 / 2681-2686 */
  double snr = a;
  if (bval >= 13) snr = b * (bval - 13) / (24 - 13) + a * (24 - bval) / (24 - 13);
  return (float)m3_pow(10.0, snr / 10.0);
}

}  // namespace

namespace {

/* blackman() of the resampler (Lame.js:1691-1714) */
double rs_blackman(double x, double fcn, int l) {
  const double PI = 3.141592653589793;
  const double wcn = PI * fcn;
  x /= l;
  if (x < 0) x = 0;
  if (x > 1) x = 1;
  const double x2 = x - .5;
  const double bkwn = 0.42 - 0.5 * cos(2 * x * PI) + 0.08 * cos(4 * x * PI);
  if (fabs(x2) < 1e-9) return wcn / PI;
  return bkwn * sin(l * wcn * x2) / (PI * l * x2);
}

/* the filter row an integer ratio uses (Lame.js:1746-1760 with bpc = 1, j = 1: offset 0, filter_l = 32).  Each tap is stored
 * to the Float32Array, the sum adds the unrounded double, and the normalised tap is stored again. */
void rs_filter(double resample_ratio, float* h) {
  double fcn = 1.00 / resample_ratio;
  if (fcn > 1.00) fcn = 1.00;
  double sum = 0.;
  for (int i = 0; i < MP3_RS_TAPS; i++) {
    const double v = rs_blackman(i, fcn, MP3_RS_TAPS - 1);
    h[i] = (float)v;
    sum += v;
  }
  for (int i = 0; i < MP3_RS_TAPS; i++) h[i] = (float)((double)h[i] / sum);
}

/* the low-pass optimum_bandwidth picks (Lame.js:838-885), before the output rate is known: it sees the UNSNAPPED kbps and the
 * INPUT rate */
double input_lowpass(int channels, int samplerate, int kbps) {
  double lowpass = kLowpassHz[ladder_index(kbps)];
  if (channels == 1) lowpass *= 1.5;
  double lp = (double)to_i32(lowpass);
  if (2 * lp > samplerate) lp = samplerate / 2.0;
  return lp;
}

}  // namespace

int mp3_out_samplerate(int channels, int samplerate, int kbps) {
  if (channels != 1 && channels != 2) return 0;
  return suggested_out_rate(to_i32(input_lowpass(channels, samplerate, kbps)), samplerate);
}

int mp3_build_config(int channels, int samplerate, int kbps, int flags, Mp3Tables* t, Mp3Resample* rs, Mp3TagParams* tag) {
  memset(t, 0, sizeof *t);
  memset(rs, 0, sizeof *rs);
  memset(tag, 0, sizeof *tag);
  rs->in_rate = samplerate;
  rs->ratio = 1;
  if (channels != 1 && channels != 2) return -1;
  t->nch = channels;
  t->mono = channels == 1;

  /* ---- rate / bandwidth decisions (Lame.js:838-896, 1044-1061) ---- */
  double lp = input_lowpass(channels, samplerate, kbps);
  const int out_rate = suggested_out_rate(to_i32(lp), samplerate);
  lp = dmin(20500, lp);
  lp = dmin(out_rate / 2.0, lp);
  if (out_rate != samplerate) {                        /* fill_buffer_resample */
    const double ratio = (double)samplerate / out_rate;
    if (!(flags & 1) || !(fabs(ratio - floor(.5 + ratio)) < .0001)) return -1;   /* intratio (Lame.js:1735) */
    rs->ratio = samplerate / out_rate;
    rs_filter(ratio, rs->h);
    samplerate = out_rate;                             /* everything below is at the rate lamejs encodes at */
  }
  switch (samplerate) {                                /* SmpFrqIndex (Lame.js:369-402) */
    case 44100: t->version = 1; t->samplerate_index = 0; break;
    case 48000: t->version = 1; t->samplerate_index = 1; break;
    case 32000: t->version = 1; t->samplerate_index = 2; break;
    case 22050: case 11025: t->version = 0; t->samplerate_index = 0; break;
    case 24000: case 12000: t->version = 0; t->samplerate_index = 1; break;
    case 16000: case 8000: t->version = 0; t->samplerate_index = 2; break;
    default: return -1;
  }
  t->samplerate = samplerate;
  t->mpeg25 = samplerate < 16000;
  t->mode_gr = samplerate <= 24000 ? 1 : 2;
  {
    /* FindNearestBitrate / BitrateIndex (Lame.js:408-443): below 16 kHz the MPEG-2.5 row is searched */
    const int* bt = kBitrates[t->mpeg25 ? 2 : t->version];
    int best = bt[1];
    for (int i = 2; i <= 14; i++)
      if (bt[i] > 0 && abs(bt[i] - kbps) < abs(best - kbps)) best = bt[i];
    t->kbps = best;
    t->bitrate_index = -1;
    for (int i = 1; i <= 14; i++) if (bt[i] > 0 && bt[i] == best) { t->bitrate_index = i; break; }
    if (t->bitrate_index <= 0) return -1;
  }
  if (t->version == 1) t->sideinfo_len = t->mono ? 21 : 36;
  else t->sideinfo_len = t->mono ? 13 : 21;
  t->frac_SpF = ((t->version + 1) * 72000 * t->kbps) % samplerate;
  t->frame_bytes_nopad = (int)((double)((t->version + 1) * 72000 * t->kbps) / samplerate);
  const Preset& ps = kPresets[ladder_index(t->kbps)];  /* apply_preset runs on the snapped rate */
  t->noise_shaping = ps.sfscale > 0 ? 2 : 1;
  t->quant_comp = t->quant_comp_short = 9;
  t->coupled_short_blocks = t->mono ? 0 : 1;
  t->scale = ps.scale;
  t->scale_applied = (ps.scale != 1.0);
  t->interch_ratio = ps.interch;
  t->attack_threshold = ps.attack;
  const double mask_adj_short = ps.mask_adj > 0 ? ps.mask_adj * .9 : ps.mask_adj * 1.1;
  t->masking_lower_long = m3_pow(10.0, ps.mask_adj * 0.1);
  t->masking_lower_short = m3_pow(10.0, mask_adj_short * 0.1);
  const double ath_lower = -ps.ath_lower / 10.;
  const double ath_curve = ps.ath_curve;
  t->aa_sensitivity_p = m3_pow(10.0, 0.0 / -10.0);

  /* ---- polyphase low-pass gains (Lame.js:470-558) ---- */
  {
    double lp2 = 2. * lp / samplerate, lp1 = lp2;
    if (lp1 > 0) {
      int lowpass_band = 32, minband = 999;
      for (int band = 0; band <= 31; band++) {
        const double f = band / 31.0;
        if (f >= lp2 && band < lowpass_band) lowpass_band = band;
        if (lp1 < f && f < lp2 && band < minband) minband = band;
      }
      lp1 = ((minband == 999 ? lowpass_band : minband) - .75) / 31.0;
      lp2 = lowpass_band / 31.0;
    }
    for (int band = 0; band < 32; band++) {
      const double f = band / 31.0;
      double g = 1.0;
      if (lp2 > lp1) {
        const double x = (f - lp1) / (lp2 - lp1 + 1e-20);
        g = x > 1.0 ? 0.0 : (x <= 0.0 ? 1.0 : cos(M_PI / 2 * x));
      }
      t->amp_filter[band] = (float)(1.0 * g);
    }
  }

  /* ---- scalefactor band edges, incl. the fractional pseudo bands (Lame.js:1079-1101) ---- */
  {
    const int j = t->samplerate_index + 3 * t->version + 6 * (t->mpeg25 ? 1 : 0);
    memcpy(t->sfb_l, kSfbLong[j], sizeof t->sfb_l);
    memcpy(t->sfb_s, kSfbShort[j], sizeof t->sfb_s);
  }
  for (int i = 0; i < 7; i++) {
    t->psfb21[i] = to_i32(t->sfb_l[21] + i * ((t->sfb_l[22] - t->sfb_l[21]) / 6.0));
    t->psfb12[i] = to_i32(t->sfb_s[12] + i * ((t->sfb_s[13] - t->sfb_s[12]) / 6.0));
  }
  t->psfb21[6] = 576;
  t->psfb12[6] = 192;
  {
    Mp3Geo& L = t->geo[0];
    Mp3Geo& S = t->geo[1];
    memset(&L, 0, sizeof L); memset(&S, 0, sizeof S);
    for (int sfb = 0; sfb < MP3_SFBMAX; sfb++) {
      L.width[sfb] = (unsigned char)(sfb < 22 ? t->sfb_l[sfb + 1] - t->sfb_l[sfb] : 0);
      L.window[sfb] = 3;
      S.width[sfb] = (unsigned char)(t->sfb_s[sfb / 3 + 1] - t->sfb_s[sfb / 3]);
      S.window[sfb] = (unsigned char)(sfb % 3);
    }
    for (int g = 0; g < 2; g++) {
      int j = 0;
      for (int sfb = 0; sfb <= MP3_SFBMAX; sfb++) { t->geo[g].start[sfb] = (short)j; if (sfb < MP3_SFBMAX) j += t->geo[g].width[sfb]; }
    }
    for (int i = 0; i < 576; i++) {
      int s = 0;
      while (t->sfb_l[s + 1] <= i) s++;
      L.sfb_of_line[i] = (unsigned char)s;
      L.reorder[i] = (short)i;
      const int l = i / 3, w = i - 3 * l;
      int sb = 0;
      while (t->sfb_s[sb + 1] <= l) sb++;
      const int st = t->sfb_s[sb], wd = t->sfb_s[sb + 1] - st;
      const int dst = 3 * st + w * wd + (l - st);
      S.reorder[i] = (short)dst;
      S.sfb_of_line[dst] = (unsigned char)(3 * sb + w);
    }
  }

  /* ---- quantizer tables (QuantizePVT.js:344-356) ---- */
  t->pow43[0] = 0.0f;
  for (int i = 1; i < MP3_PRECALC; i++) t->pow43[i] = (float)m3_pow(i, 4.0 / 3.0);
  for (int i = 0; i < MP3_PRECALC - 1; i++)
    t->adj43[i] = (float)((i + 1) - m3_pow(0.5 * ((double)t->pow43[i] + (double)t->pow43[i + 1]), 0.75));
  t->adj43[MP3_PRECALC - 1] = 0.5f;
  for (int i = 0; i < MP3_QMAX; i++) t->ipow20[i] = (float)m3_pow(2.0, (i - 210) * -0.1875);
  for (int i = 0; i < MP3_QMAX; i++) {
    const double istep = (double)t->ipow20[i];
    t->ixmax_over_istep[i] = 8206.0 / istep;
    t->cmp01_over_istep[i] = (1.0 - 0.4054) / istep;
  }
  for (int i = 0; i <= MP3_QMAX + MP3_QMAX2; i++) t->pow20[i] = (float)m3_pow(2.0, (i - 210 - MP3_QMAX2) * 0.25);
  for (int i = 0; i < MP3_SBMAX_L; i++) t->longfact[i] = (float)m3_pow(10, 0 / 4.0 / 10.0);   /* nspsytune bits 2.. are 0 */
  for (int i = 0; i < MP3_SBMAX_S; i++) t->shortfact[i] = (float)m3_pow(10, 0 / 4.0 / 10.0);

  /* ---- region split lookup (Takehiro.js:1141-1172) ---- */
  {
    static const int subdv[23][2] = {{0, 0}, {0, 0}, {0, 0}, {0, 0}, {0, 0}, {0, 1}, {1, 1}, {1, 1}, {1, 2}, {2, 2}, {2, 3},
      {2, 3}, {3, 4}, {3, 4}, {3, 4}, {4, 5}, {4, 5}, {4, 6}, {5, 6}, {5, 6}, {5, 7}, {6, 7}, {6, 7}};
    for (int i = 2; i <= 576; i += 2) {
      int nb = 0;
      while (t->sfb_l[++nb] < i) {}
      int r0 = subdv[nb][0];
      while (t->sfb_l[r0 + 1] > i) r0--;
      if (r0 < 0) r0 = subdv[nb][0];
      t->bv_scf[i - 2] = r0;
      int r1 = subdv[nb][1];
      while (t->sfb_l[r1 + r0 + 2] > i) r1--;
      if (r1 < 0) r1 = subdv[nb][1];
      t->bv_scf[i - 1] = r1;
    }
  }

  /* ---- ATH per scalefactor band in MDCT units (QuantizePVT.js:229-318) ---- */
  {
    auto ath_mdct = [&](double f) { return m3_pow(10.0, (ath_db(f, ath_curve) - 100) / 10.0 + ath_lower); };
    auto band_min = [&](int start, int end, int denom) {
      float m = 3.4028235e+38f;
      for (int i = start; i < end; i++) {
        const double a = ath_mdct(i * (double)samplerate / denom);
        if (a < (double)m) m = (float)a;       /* Math.min then Float32 store */
      }
      return m;
    };
    for (int s = 0; s < MP3_SBMAX_L; s++) t->ath_l[s] = band_min(t->sfb_l[s], t->sfb_l[s + 1], 2 * 576);
    for (int s = 0; s < 6; s++) t->ath_psfb21[s] = band_min(t->psfb21[s], t->psfb21[s + 1], 2 * 576);
    for (int s = 0; s < MP3_SBMAX_S; s++)
      t->ath_s[s] = (float)((double)band_min(t->sfb_s[s], t->sfb_s[s + 1], 2 * 192) * (t->sfb_s[s + 1] - t->sfb_s[s]));
    for (int s = 0; s < 6; s++)
      t->ath_psfb12[s] = (float)((double)band_min(t->psfb12[s], t->psfb12[s + 1], 2 * 192) * (t->sfb_s[13] - t->sfb_s[12]));
    t->ath_floor = 10. * m3_log10(ath_mdct(-1.));
  }

  /* ---- psycho-acoustic partitions, spreading rows, ATH per partition (PsyModel.js:2602-2729) ---- */
  {
    const double sfreq = samplerate;
    PartitionLayout lay;
    float norm[MP3_CBANDS];
    layout_partitions(sfreq, 1024, t->sfb_l, MP3_SBMAX_L, 1024 / (2.0 * 576), t->numlines_l, t->bo_l, t->bo_l_weight, &lay);
    t->npart_l = lay.npart;
    int line = 0;
    for (int i = 0; i < t->npart_l; i++) {
      norm[i] = snr_norm(lay.bval[i], 0, 0);
      t->rnumlines_l[i] = t->numlines_l[i] > 0 ? (float)(1.0 / t->numlines_l[i]) : 0.0f;
      t->line0_l[i] = line;
      double x = 3.4028235e+38;
      for (int k = 0; k < t->numlines_l[i]; k++, line++) {
        const double freq = sfreq * line / (1000.0 * 1024);
        double level = m3_pow(10., 0.1 * (ath_db(freq * 1000, ath_curve) - 20));
        level *= t->numlines_l[i];
        if (x > level) x = level;
      }
      t->ath_cb_l[i] = (float)x;
    }
    t->line0_l[t->npart_l] = line;
    if (build_spreading(lay, norm, t->s3lo_l, t->s3hi_l, t->s3off_l, t->s3_ll) < 0) return -1;
    for (int b = 0; b < t->npart_l; b++)             /* PsyModel.js:2751-2753 */
      if (t->s3hi_l[b] > t->npart_l - 1) t->s3hi_l[b] = t->npart_l - 1;

    layout_partitions(sfreq, 256, t->sfb_s, MP3_SBMAX_S, 256 / (2.0 * 192), t->numlines_s, t->bo_s, t->bo_s_weight, &lay);
    t->npart_s = lay.npart;
    line = 0;
    for (int i = 0; i < t->npart_s; i++) {
      norm[i] = snr_norm(lay.bval[i], -8.25, -4.5);
      t->line0_s[i] = line;
      double x = 3.4028235e+38;
      for (int k = 0; k < t->numlines_s[i]; k++, line++) {
        const double freq = sfreq * line / (1000.0 * 256);
        double level = m3_pow(10., 0.1 * (ath_db(freq * 1000, ath_curve) - 20));
        level *= t->numlines_s[i];
        if (x > level) x = level;
      }
      t->ath_cb_s[i] = (float)x;
    }
    t->line0_s[t->npart_s] = line;
    if (build_spreading(lay, norm, t->s3lo_s, t->s3hi_s, t->s3off_s, t->s3_ss) < 0) return -1;
  }
  /* band slices of convert_partition2scalefac_l/_s: replay the cursor walk on the tables alone */
  for (int pass = 0; pass < 2; pass++) {
    Mp3Conv& cv = pass == 0 ? t->conv_l : t->conv_s;
    const int nb = pass == 0 ? MP3_SBMAX_L : MP3_SBMAX_S, np = pass == 0 ? t->npart_l : t->npart_s;
    const int* bo = pass == 0 ? t->bo_l : t->bo_s;
    int sbi, p, init = -1;
    for (sbi = p = 0; sbi < nb; ++p, ++sbi) {
      const int b_lim = bo[sbi] < np ? bo[sbi] : np;
      cv.init[sbi] = (short)init; cv.start[sbi] = (short)p;
      while (p < b_lim) p++;
      cv.end[sbi] = (short)p;
      if (p >= np) { cv.bound[sbi] = -1; ++sbi; break; }
      cv.bound[sbi] = (short)p; init = p;
    }
    for (; sbi < nb; ++sbi) { cv.init[sbi] = -2; cv.start[sbi] = cv.end[sbi] = 0; cv.bound[sbi] = -1; }
  }
  {
    /* thresholds of 0 | (log10(r) * 16): see mp3_config.h */
    auto idx = [](double r) { return (int)(m3_log10(r) * 16.0); };
    auto bits = [](double d) { uint64_t u; memcpy(&u, &d, 8); return u; };
    auto from = [](uint64_t u) { double d; memcpy(&d, &u, 8); return d; };
    t->l16_ok = 1;
    t->l16_thr[0] = 0.0;
    for (int k = 1; k <= 24; k++) {
      uint64_t lo = bits(1.0), hi = bits(64.0);          /* idx(lo) < k <= idx(hi); positive doubles order like their bits */
      while (hi - lo > 1) { const uint64_t mid = lo + (hi - lo) / 2; if (idx(from(mid)) >= k) hi = mid; else lo = mid; }
      t->l16_thr[k] = from(hi);
      for (int d = 1; d <= 4096; d++)                    /* a clean step: nothing at or above the threshold falls below k ... */
        if (idx(from(hi + d - 1)) < k || idx(from(hi - d)) >= k) t->l16_ok = 0;
    }
  }
  t->ma_max_i1 = m3_pow(10, (8 + 1) / 16.0);
  t->ma_max_i2 = m3_pow(10, (23 + 1) / 16.0);
  t->ma_max_m = m3_pow(10, 15 / 10.0);
  t->decay = m3_exp(-1.0 * 2.30258509299404568402 / (0.01 * samplerate / 192.0));

  /* ---- equal-loudness weights (PsyModel.js:2770-2788) ---- */
  {
    const double inc = (double)samplerate / 1024;
    double f = 0.0, bal = 0.0;
    for (int i = 0; i < 512; ++i) {
      f += inc;
      t->eql_w[i] = (float)(1. / m3_pow(10, ath_db(f, ath_curve) / 10));
      bal += (double)t->eql_w[i];
    }
    bal = 1.0 / bal;
    for (int i = 512; --i >= 0;) t->eql_w[i] = (float)((double)t->eql_w[i] * bal);
  }

  /* ---- FFT windows and FHT twiddles (FFT.js:226-242, :70-111) ---- */
  for (int i = 0; i < 1024; i++)
    t->fft_window[i] = (float)(0.42 - 0.5 * cos(2 * M_PI * (i + .5) / 1024) + 0.08 * cos(4 * M_PI * (i + .5) / 1024));
  for (int i = 0; i < 128; i++) t->fft_window_s[i] = (float)(0.5 * (1.0 - cos(2.0 * M_PI * (i + 0.5) / 256)));
  {
    int off = 0;
    for (int stage = 0, kx = 2; stage < 4; stage++, kx *= 4) {
      t->tw_off[stage] = off;
      double c1 = MP3_FHT_COSTAB[2 * stage], s1 = MP3_FHT_COSTAB[2 * stage + 1];
      for (int i = 1; i < kx; i++) {
        double* e = &t->tw[4 * (off + i)];
        e[0] = c1; e[1] = s1;
        e[2] = 1 - (2 * s1) * s1;
        e[3] = (2 * s1) * c1;
        const double c2 = c1;
        c1 = c2 * MP3_FHT_COSTAB[2 * stage] - s1 * MP3_FHT_COSTAB[2 * stage + 1];
        s1 = c2 * MP3_FHT_COSTAB[2 * stage + 1] + s1 * MP3_FHT_COSTAB[2 * stage];
      }
      off += kx;
    }
    t->tw_off[4] = off;
  }

  /* ---- the tag's fields (VBRTag.js:281-364, 558-802) ----
   * lowpassfreq as lame_init_params leaves it, the preset's safejoint bit (Presets.js:262-263), and the "non optimal
   * settings" rule of putLameVBR (VBRTag.js:722-731), which for Mp3Encoder reduces to: reservoir disabled below 320 kbps, or
   * a source rate of 32 kHz and below.  With resampling, the low-pass and the source-rate fields see the input rate, the
   * rest the output rate. */
  tag->version = t->version; tag->mpeg25 = t->mpeg25; tag->samplerate = t->samplerate; tag->kbps = t->kbps; tag->mono = t->mono;
  tag->bitrate_index = t->bitrate_index; tag->samplerate_index = t->samplerate_index; tag->sideinfo_len = t->sideinfo_len;
  tag->frame_bytes = t->frame_bytes_nopad;
  tag->fits = tag->frame_bytes >= tag->sideinfo_len + 156 && tag->frame_bytes <= 2880;
  const double lb = lp / 100.0 + .5;
  tag->lowpass_byte = to_i32(lb > 255 ? 255 : lb);
  tag->quality_byte = 100 - 10 * 4 - 3;
  tag->flags_byte = 4 + (1 << 4) + ((ps.safejoint ? 1 : 0) << 5);
  const int in_rate = rs->in_rate;
  const int source_class = in_rate <= 32000 ? 0 : in_rate == 48000 ? 2 : in_rate > 48000 ? 3 : 1;
  const int non_optimal = (t->kbps < 320 || in_rate <= 32000) ? 1 : 0;
  tag->misc_byte = t->noise_shaping + ((t->mono ? 0 : 1) << 2) + (non_optimal << 5) + (source_class << 6);
  return 0;
}
