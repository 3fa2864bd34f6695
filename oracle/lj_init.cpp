/* lj_init.cpp -- parameter derivation, stream driver and C API of the oracle.
 * TEST INFRASTRUCTURE (see lj_core.h).  Follows:
 *   src/js/index.js:66-136        Mp3Encoder ctor / encodeBuffer / flush
 *   src/js/Lame.js:121-225        lame_init_old defaults
 *   src/js/Lame.js:239-558        filter_coef, nearestBitrateFullIndex, optimum_*, ppflt
 *   src/js/Lame.js:560-690        lame_init_qval
 *   src/js/Lame.js:747-1371       lame_init_params
 *   src/js/Lame.js:1381-1667      lame_encode_flush / lame_encode_buffer(_sample)
 *   src/js/Presets.js:226-358     abr_switch_map / apply_abr_preset
 *   src/js/Encoder.js:166-243,287-326,388-659  adjust_ATH, frame init, lame_encode_mp3_frame
 */
#include <stdio.h>
#include <stdlib.h>
#include <math.h>
#include "lj_encoder.h"

static const int bitrate_table_mpeg1[16] = {0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, -1};
/* Tables.js:494-498: [0] MPEG-2, [1] MPEG-1, [2] MPEG-2.5 */
static const int bitrate_table[3][16] = {
  {0, 8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160, -1},
  {0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, -1},
  {0, 8, 16, 24, 32, 40, 48, 56, 64, -1, -1, -1, -1, -1, -1, -1}};

/* Lame.js:248-283 */
static int nearestBitrateFullIndex(int bitrate) {
  static const int full_bitrate_table[17] = {8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320};
  int lower_range = 16, lower_range_kbps = 320, upper_range = 16, upper_range_kbps = 320;
  for (int b = 0; b < 16; b++) {
    if ((bitrate > full_bitrate_table[b + 1] ? bitrate : full_bitrate_table[b + 1]) != bitrate) {
      upper_range_kbps = full_bitrate_table[b + 1];
      upper_range = b + 1;
      lower_range_kbps = full_bitrate_table[b];
      lower_range = b;
      break;
    }
  }
  if ((upper_range_kbps - bitrate) > (bitrate - lower_range_kbps)) return lower_range;
  return upper_range;
}

/* Lame.js:285-364 */
static int optimum_samplefreq(int lowpassfreq, int input_samplefreq) {
  int suggested = 44100;
  if (input_samplefreq >= 48000) suggested = 48000;
  else if (input_samplefreq >= 44100) suggested = 44100;
  else if (input_samplefreq >= 32000) suggested = 32000;
  else if (input_samplefreq >= 24000) suggested = 24000;
  else if (input_samplefreq >= 22050) suggested = 22050;
  else if (input_samplefreq >= 16000) suggested = 16000;
  else if (input_samplefreq >= 12000) suggested = 12000;
  else if (input_samplefreq >= 11025) suggested = 11025;
  else if (input_samplefreq >= 8000) suggested = 8000;
  if (lowpassfreq == -1) return suggested;
  if (lowpassfreq <= 15960) suggested = 44100;
  if (lowpassfreq <= 15250) suggested = 32000;
  if (lowpassfreq <= 11220) suggested = 24000;
  if (lowpassfreq <= 9970) suggested = 22050;
  if (lowpassfreq <= 7230) suggested = 16000;
  if (lowpassfreq <= 5420) suggested = 12000;
  if (lowpassfreq <= 4510) suggested = 11025;
  if (lowpassfreq <= 3970) suggested = 8000;
  if (input_samplefreq < suggested) {
    if (input_samplefreq > 44100) return 48000;
    if (input_samplefreq > 32000) return 44100;
    if (input_samplefreq > 24000) return 32000;
    if (input_samplefreq > 22050) return 24000;
    if (input_samplefreq > 16000) return 22050;
    if (input_samplefreq > 12000) return 16000;
    if (input_samplefreq > 11025) return 12000;
    if (input_samplefreq > 8000) return 11025;
    return 8000;
  }
  return suggested;
}

static double filter_coef(double x) {
  if (x > 1.0) return 0.0;
  if (x <= 0.0) return 1.0;
  return cos(M_PI / 2 * x);
}

/* Lame.js:470-558 */
static void init_params_ppflt(LjEnc* e) {
  int lowpass_band = 32;
  if (e->lowpass1 > 0) {
    int minband = 999;
    for (int band = 0; band <= 31; band++) {
      double freq = band / 31.0;
      if (freq >= e->lowpass2) lowpass_band = lowpass_band < band ? lowpass_band : band;
      if (e->lowpass1 < freq && freq < e->lowpass2) minband = minband < band ? minband : band;
    }
    if (minband == 999) e->lowpass1 = (lowpass_band - .75) / 31.0;
    else e->lowpass1 = (minband - .75) / 31.0;
    e->lowpass2 = lowpass_band / 31.0;
  }
  /* highpass2 == 0 for Mp3Encoder (highpassfreq = 0) */
  for (int band = 0; band < 32; band++) {
    double fc1, fc2;
    double freq = band / 31.0;
    if (e->highpass2 > e->highpass1) fc1 = filter_coef((e->highpass2 - freq) / (e->highpass2 - e->highpass1 + 1e-20));
    else fc1 = 1.0;
    if (e->lowpass2 > e->lowpass1) fc2 = filter_coef((freq - e->lowpass1) / (e->lowpass2 - e->lowpass1 + 1e-20));
    else fc2 = 1.0;
    e->amp_filter[band] = fc1 * fc2;
  }
}

struct AbrPreset { int kbps, quant_comp, quant_comp_s, safejoint; double nsmsfix, st_lrm, st_s, nsbass, scale, masking_adj, ath_lower, ath_curve, interch; int sfscale; };
/* Presets.js:226-244 */
static const AbrPreset abr_switch_map[17] = {
  {8, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, -30.0, 11, 0.0012, 1},
  {16, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, -25.0, 11, 0.0010, 1},
  {24, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, -20.0, 11, 0.0010, 1},
  {32, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, -15.0, 11, 0.0010, 1},
  {40, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, -10.0, 11, 0.0009, 1},
  {48, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, -10.0, 11, 0.0009, 1},
  {56, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, -6.0, 11, 0.0008, 1},
  {64, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, -2.0, 11, 0.0008, 1},
  {80, 9, 9, 0, 0, 6.60, 145, 0, 0.95, 0, .0, 8, 0.0007, 1},
  {96, 9, 9, 0, 2.50, 6.60, 145, 0, 0.95, 0, 1.0, 5.5, 0.0006, 1},
  {112, 9, 9, 0, 2.25, 6.60, 145, 0, 0.95, 0, 2.0, 4.5, 0.0005, 1},
  {128, 9, 9, 0, 1.95, 6.40, 140, 0, 0.95, 0, 3.0, 4, 0.0002, 1},
  {160, 9, 9, 1, 1.79, 6.00, 135, 0, 0.95, -2, 5.0, 3.5, 0, 1},
  {192, 9, 9, 1, 1.49, 5.60, 125, 0, 0.97, -4, 7.0, 3, 0, 0},
  {224, 9, 9, 1, 1.25, 5.20, 125, 0, 0.98, -6, 9.0, 2, 0, 0},
  {256, 9, 9, 1, 0.97, 5.20, 125, 0, 1.00, -8, 10.0, 1, 0, 0},
  {320, 9, 9, 1, 0.90, 5.20, 125, 0, 1.00, -10, 12.0, 0, 0, 0}};

/* Presets.js:246-358 with enforce = 0 and the lame_init_old defaults (-1 / 0 = "unset") */
static void apply_abr_preset(LjEnc* e, int preset) {
  int r = nearestBitrateFullIndex(preset);
  const AbrPreset& p = abr_switch_map[r];
  /* gfp.brate = clamp(preset, 8, 320): preset is already a legal MPEG-1 rate here */
  if (p.safejoint > 0) e->exp_nspsytune |= 2;
  if (p.sfscale > 0) e->noise_shaping = 2;
  /* nsbass == 0 for every row: the (int) cast at Presets.js:268 is never reached */
  e->quant_comp = p.quant_comp;           /* was -1 */
  e->quant_comp_short = p.quant_comp_s;   /* was -1 */
  e->msfix = p.nsmsfix;                   /* was -1 */
  e->attackthre = p.st_lrm;               /* was -1 */
  e->attackthre_s = p.st_s;               /* was -1 */
  e->scale = p.scale;                     /* was -1 */
  e->maskingadjust = p.masking_adj;       /* was 0 */
  if (p.masking_adj > 0) e->maskingadjust_short = p.masking_adj * .9;
  else e->maskingadjust_short = p.masking_adj * 1.1;
  e->ATHlower = -p.ath_lower / 10.;       /* was 0 */
  e->ATHcurve = p.ath_curve;              /* was -1 */
  e->interChRatio = p.interch;            /* was -1 */
}

static int framebits(int version, int bitrate_index, int out_samplerate, int padding) {
  /* BitStream.js:83-98: bitrate_index != 0 always; `0 | a/b + padding` */
  int bit_rate = bitrate_table[version][bitrate_index];
  int bytes = js_toint32((double)((version + 1) * 72000 * bit_rate) / out_samplerate + padding);
  return 8 * bytes;
}
int lj_getframebits(const LjEnc* e) { return framebits(e->version, e->bitrate_index, e->out_samplerate, e->padding); }

int lj_init_params(LjEnc* e, int channels, int samplerate, int kbps) {
  /* lame_init_old defaults that matter */
  e->num_channels = channels; e->in_samplerate = samplerate; e->brate = kbps;
  e->quality = 3;
  e->disable_reservoir = 1;      /* index.js:108 */
  e->OldValue[0] = e->OldValue[1] = 180;
  e->CurrentStep[0] = e->CurrentStep[1] = 4;
  e->masking_lower = 1;
  e->attackthre = -1; e->attackthre_s = -1;
  e->scale = -1; e->ATHcurve = -1; e->ATHtype = -1; e->interChRatio = -1;
  e->quant_comp = -1; e->quant_comp_short = -1; e->msfix = -1;
  e->subblock_gain = -1;
  e->mf_samples_to_encode = ENCDELAY + POSTDELAY;
  e->mf_size = ENCDELAY - MDCTDELAY;
  e->maskingadjust = e->maskingadjust_short = 0; e->ATHlower = 0; e->exp_nspsytune = 0;

  /* lame_init_params */
  e->mode_mono = (channels == 1);
  e->channels_out = e->mode_mono ? 1 : 2;
  e->mode_ext = 2; /* MPG_MD_MS_LR, overwritten every frame */
  /* lowpass (Lame.js:838-885), VBR == vbr_off */
  {
    static const int lowpass_map[17] = {2000, 3700, 3900, 5500, 7000, 7500, 10000, 11000, 13500, 15100, 15600,
                                        17000, 17500, 18600, 19400, 19700, 20500};
    double lowpass = lowpass_map[nearestBitrateFullIndex(e->brate)];
    if (e->mode_mono) lowpass *= 1.5;
    e->lowpassfreq = js_toint32(lowpass);
  }
  double lowpassfreq = e->lowpassfreq;
  if (2 * lowpassfreq > e->in_samplerate) lowpassfreq = e->in_samplerate / 2.0;
  e->out_samplerate = optimum_samplefreq(js_toint32(lowpassfreq), e->in_samplerate);
  lowpassfreq = js_min(20500, lowpassfreq);
  lowpassfreq = js_min(e->out_samplerate / 2.0, lowpassfreq);
  e->lowpass_final = lowpassfreq;
  switch (e->out_samplerate) {   /* SmpFrqIndex (Lame.js:369-402): version 1 = MPEG-1, 0 = MPEG-2 and MPEG-2.5 */
    case 44100: e->version = 1; e->samplerate_index = 0; break;
    case 48000: e->version = 1; e->samplerate_index = 1; break;
    case 32000: e->version = 1; e->samplerate_index = 2; break;
    case 22050: e->version = 0; e->samplerate_index = 0; break;
    case 24000: e->version = 0; e->samplerate_index = 1; break;
    case 16000: e->version = 0; e->samplerate_index = 2; break;
    case 11025: e->version = 0; e->samplerate_index = 0; break;
    case 12000: e->version = 0; e->samplerate_index = 1; break;
    case 8000: e->version = 0; e->samplerate_index = 2; break;
    default: return -1;
  }
  e->compression_ratio = e->out_samplerate * 16 * e->channels_out / (1.e3 * e->brate);
  e->mode_gr = e->out_samplerate <= 24000 ? 1 : 2;
  e->framesize = 576 * e->mode_gr;
  e->resample_ratio = (double)e->in_samplerate / e->out_samplerate;
  e->highpass1 = e->highpass2 = 0;
  if (lowpassfreq > 0) {
    e->lowpass2 = 2. * lowpassfreq;
    e->lowpass1 = (1 - 0.00) * 2. * lowpassfreq; /* lowpasswidth = -1 */
    e->lowpass1 /= e->out_samplerate;
    e->lowpass2 /= e->out_samplerate;
  } else { e->lowpass1 = e->lowpass2 = 0; }
  init_params_ppflt(e);
  /* FindNearestBitrate / BitrateIndex (Lame.js:408-443): below 16 kHz the MPEG-2.5 row is searched */
  {
    const int* bt = bitrate_table[e->out_samplerate < 16000 ? 2 : e->version];
    int bitrate = bt[1];
    for (int i = 2; i <= 14; i++)
      if (bt[i] > 0 && abs(bt[i] - e->brate) < abs(bitrate - e->brate)) bitrate = bt[i];
    e->brate = bitrate;
    e->bitrate_index = -1;
    for (int i = 0; i <= 14; i++) if (bt[i] > 0 && bt[i] == e->brate) { e->bitrate_index = i; break; }
    if (e->bitrate_index <= 0) return -1;
  }
  /* bitstream init */
  e->bs_byteidx = -1; e->bs_bitidx = 0; e->bs_totbit = 0;
  e->h_ptr = e->w_ptr = 0; e->header[0].write_timing = 0;      /* init_bit_stream_w (BitStream.js:1012-1020) */
  /* sfb tables (Lame.js:1079-1101; QuantizePVT.js:137-204) */
  {
    /* QuantizePVT.js:137-204 sfBandIndex: 22.05, 24, 16 kHz (MPEG-2); 44.1, 48, 32 kHz (MPEG-1); 11.025, 12, 8 kHz (MPEG-2.5) */
    static const int sfl[9][23] = {
      {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576},
      {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 114, 136, 162, 194, 232, 278, 332, 394, 464, 540, 576},
      {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576},
      {0, 4, 8, 12, 16, 20, 24, 30, 36, 44, 52, 62, 74, 90, 110, 134, 162, 196, 238, 288, 342, 418, 576},
      {0, 4, 8, 12, 16, 20, 24, 30, 36, 42, 50, 60, 72, 88, 106, 128, 156, 190, 230, 276, 330, 384, 576},
      {0, 4, 8, 12, 16, 20, 24, 30, 36, 44, 54, 66, 82, 102, 126, 156, 194, 240, 296, 364, 448, 550, 576},
      {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576},
      {0, 6, 12, 18, 24, 30, 36, 44, 54, 66, 80, 96, 116, 140, 168, 200, 238, 284, 336, 396, 464, 522, 576},
      {0, 12, 24, 36, 48, 60, 72, 88, 108, 132, 160, 192, 232, 280, 336, 400, 476, 566, 568, 570, 572, 574, 576}};
    static const int sfs[9][14] = {
      {0, 4, 8, 12, 18, 24, 32, 42, 56, 74, 100, 132, 174, 192},
      {0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 136, 180, 192},
      {0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 134, 174, 192},
      {0, 4, 8, 12, 16, 22, 30, 40, 52, 66, 84, 106, 136, 192},
      {0, 4, 8, 12, 16, 22, 28, 38, 50, 64, 80, 100, 126, 192},
      {0, 4, 8, 12, 16, 22, 30, 42, 58, 78, 104, 138, 180, 192},
      {0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 134, 174, 192},
      {0, 4, 8, 12, 18, 26, 36, 48, 62, 80, 104, 134, 174, 192},
      {0, 8, 16, 24, 36, 52, 72, 96, 124, 160, 162, 164, 166, 192}};
    int j = e->samplerate_index + 3 * e->version + 6 * (e->out_samplerate < 16000 ? 1 : 0);
    for (int i = 0; i < SBMAX_l + 1; i++) e->sfb_l[i] = sfl[j][i];
    for (int i = 0; i < PSFB21 + 1; i++) {
      double size = (e->sfb_l[22] - e->sfb_l[21]) / (double)PSFB21;   /* JS float division */
      double start = e->sfb_l[21] + i * size;
      e->psfb21[i] = js_toint32(start);                               /* Int32Array store */
    }
    e->psfb21[PSFB21] = 576;
    for (int i = 0; i < SBMAX_s + 1; i++) e->sfb_s[i] = sfs[j][i];
    for (int i = 0; i < PSFB12 + 1; i++) {
      double size = (e->sfb_s[13] - e->sfb_s[12]) / (double)PSFB12;
      double start = e->sfb_s[12] + i * size;
      e->psfb12[i] = js_toint32(start);
    }
    e->psfb12[PSFB12] = 192;
  }
  if (e->version == 1) e->sideinfo_len = (e->channels_out == 1) ? 4 + 17 : 4 + 32;
  else e->sideinfo_len = (e->channels_out == 1) ? 4 + 9 : 4 + 17;
  for (int k = 0; k < 19; k++) e->pefirbuf[k] = 700 * e->mode_gr * e->channels_out;
  if (e->ATHtype == -1) e->ATHtype = 4;
  /* cbr: apply_preset(brate) */
  e->sfb21_extra = 0;
  apply_abr_preset(e, e->brate);
  e->mask_adjust = e->maskingadjust;
  e->mask_adjust_short = e->maskingadjust_short;
  /* lame_init_qval, quality 3 (Lame.js:626-636) */
  e->psymodel = 1;
  if (e->noise_shaping == 0) e->noise_shaping = 1;
  e->noise_shaping_amp = 1;
  e->noise_shaping_stop = 1;
  if (e->subblock_gain == -1) e->subblock_gain = 1;
  e->use_best_huffman = 1;
  e->full_outer_loop = 0;
  e->ath_useAdjust = 3;
  e->ath_aaSensitivityP = js_pow(10.0, 0.0 / -10.0);
  e->short_blocks_coupled = e->mode_mono ? 0 : 1;
  if (e->quant_comp < 0) e->quant_comp = 1;
  if (e->quant_comp_short < 0) e->quant_comp_short = 0;
  if (e->msfix < 0) e->msfix = 0;
  e->exp_nspsytune |= 1;
  if (e->attackthre < 0) e->attackthre = 4.4;
  if (e->attackthre_s < 0) e->attackthre_s = 25;
  if (e->scale < 0) e->scale = 1;
  if (e->ATHtype < 0) e->ATHtype = 4;
  if (e->ATHcurve < 0) e->ATHcurve = 4;
  if (e->interChRatio < 0) e->interChRatio = 0;
  e->useTemporal = 1;
  e->slot_lag = e->frac_SpF = (((e->version + 1) * 72000 * e->brate) % e->out_samplerate);
  lj_iteration_init(e);
  lj_psymodel_init(e);
  return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* Encoder.js:166-243 */
static void adjust_ATH(LjEnc* e) {
  double gr2_max, max_pow;
  if (e->ath_useAdjust == 0) { e->ath_adjust = 1.0; return; }
  max_pow = e->loudness_sq[0][0];
  gr2_max = e->loudness_sq[1][0];
  if (e->channels_out == 2) { max_pow += e->loudness_sq[0][1]; gr2_max += e->loudness_sq[1][1]; }
  else { max_pow += max_pow; gr2_max += gr2_max; }
  if (e->mode_gr == 2) max_pow = js_max(max_pow, gr2_max);
  max_pow *= 0.5;
  max_pow *= e->ath_aaSensitivityP;
  if (max_pow > 0.03125) {
    if (e->ath_adjust >= 1.0) e->ath_adjust = 1.0;
    else if (e->ath_adjust < e->ath_adjustLimit) e->ath_adjust = e->ath_adjustLimit;
    e->ath_adjustLimit = 1.0;
  } else {
    double adj_lim_new = 31.98 * max_pow + 0.000625;
    if (e->ath_adjust >= adj_lim_new) {
      e->ath_adjust *= adj_lim_new * 0.075 + 0.925;
      if (e->ath_adjust < adj_lim_new) e->ath_adjust = adj_lim_new;
    } else {
      if (e->ath_adjustLimit >= adj_lim_new) e->ath_adjust = adj_lim_new;
      else if (e->ath_adjust < e->ath_adjustLimit) e->ath_adjust = e->ath_adjustLimit;
    }
    e->ath_adjustLimit = adj_lim_new;
  }
}

/* the psy trace (lj_set_psy_trace): called by lj_psycho_anal_ns at the points each field is final */
void lj_psy_trace_attacks(LjEnc* e, int gr, int chn, const F32* en_subshort, const int* ns_attacks) {
  LjPsyTrace* const t = e->ptrace_cur;
  if (!t || chn >= 2) return;
  for (int i = 0; i < 9; i++) t->peaks[gr][chn][i] = en_subshort[i + 3].v;
  for (int i = 0; i < 4; i++) t->attack[gr][chn][i] = ns_attacks[i];
  const int row = (int)(t - e->ptrace);
  if (e->pbtrace && row < e->pbtrace_cap) e->pbtrace[row].blocktype_old[gr][chn] = e->blocktype_old[chn];
}
void lj_psy_trace_long(LjEnc* e, int gr, int chn, const F32* eb_l, const int* mask_idx_l) {
  LjPsyTrace* const t = e->ptrace_cur;
  if (!t || chn >= 2) return;
  t->loudness[gr][chn] = e->loudness_sq_save[chn].v;
  for (int b = 0; b < e->npart_l; b++) { t->eb_l[gr][chn][b] = eb_l[b].v; t->mask_idx_l[gr][chn][b] = mask_idx_l[b]; }
}
/* after compute_masking_s of short block sblock: its partition energies and the spreading sums it stored into nb_s1 */
void lj_psy_trace_short(LjEnc* e, int gr, int chn, int sblock, const F32* eb_s) {
  LjPsyTrace* const t = e->ptrace_cur;
  if (!t || chn >= 2) return;
  for (int b = 0; b < e->npart_s; b++) { t->eb_s[gr][chn][sblock][b] = eb_s[b].v; t->ecb_s[gr][chn][sblock][b] = e->nb_s1[chn][b].v; }
}
/* the quantizer trace (lj_set_quant_trace): what lj_iteration_loop hands outer_loop, after init_xrpow */
void lj_quant_trace_rows(LjEnc* e, const LjQuantTrace* t, int gr, int ch, const GrInfo* cod_info, const F32* xrpow, bool have) {
  if (!t || ch >= 2) return;
  const int row = (int)(t - e->qtrace);
  if (!e->qrtrace || row >= e->qrtrace_cap) return;
  LjQuantRowTrace* const r = &e->qrtrace[row];
  for (int i = 0; i < 576; i++) { r->xrq[gr][ch][i] = cod_info->xr[i].v; r->xrpow[gr][ch][i] = xrpow[i].v; }
  r->have[gr][ch] = have ? 1 : 0;
}

/* Encoder.js:287-326 */
static void encode_frame_init(LjEnc* e) {
  if (e->frame_init_done) return;
  e->frame_init_done = 1;
  F32 primebuff0[286 + 1152 + 576], primebuff1[286 + 1152 + 576];
  for (int i = 0, j = 0; i < 286 + 576 * (1 + e->mode_gr); ++i) {
    if (i < 576 * e->mode_gr) {
      primebuff0[i] = 0;
      if (e->channels_out == 2) primebuff1[i] = 0;
    } else {
      primebuff0[i] = e->mfbuf[0][j];
      if (e->channels_out == 2) primebuff1[i] = e->mfbuf[1][j];
      ++j;
    }
  }
  for (int gr = 0; gr < e->mode_gr; gr++)
    for (int ch = 0; ch < e->channels_out; ch++) e->tt[gr][ch].block_type = SHORT_TYPE;
  lj_mdct_sub48(e, primebuff0, primebuff1);
}

/* Encoder.js:388-659 */
static int encode_mp3_frame(LjEnc* e, uint8_t* mp3buf, int mp3buf_size) {
  PsyRatio masking_LR[2][2], masking_MS[2][2];
  F32 tot_ener[2][4];
  double pe[2][2] = {{0., 0.}, {0., 0.}}, pe_MS[2][2] = {{0., 0.}, {0., 0.}};
  double ms_ener_ratio[2] = {.5, .5};
  LjFrameTrace tr; /* filled progressively when tracing */
  bool tracing = e->trace && e->trace_n < e->trace_cap;
  if (tracing) memset(&tr, 0, sizeof tr);

  encode_frame_init(e);
  e->padding = 0;
  if ((e->slot_lag -= e->frac_SpF) < 0) { e->slot_lag += e->out_samplerate; e->padding = 1; }

  int blocktype[2];
  e->ptrace_cur = (e->ptrace && e->ptrace_n < e->ptrace_cap) ? &e->ptrace[e->ptrace_n++] : NULL;
  if (e->ptrace_cur) memset(e->ptrace_cur, 0, sizeof *e->ptrace_cur);
  for (int gr = 0; gr < e->mode_gr; gr++) {
    int bufpPos = 576 + gr * 576 - FFTOFFSET;
    int ret = lj_psycho_anal_ns(e, e->mfbuf[0], e->mfbuf[1], bufpPos, gr, masking_LR, masking_MS, pe[gr], pe_MS[gr], tot_ener[gr], blocktype);
    if (ret != 0) return -4;
    if (e->mode_joint) {                       /* Encoder.js:482-486 */
      ms_ener_ratio[gr] = tot_ener[gr][2] + tot_ener[gr][3];
      if (ms_ener_ratio[gr] > 0) ms_ener_ratio[gr] = tot_ener[gr][3] / ms_ener_ratio[gr];
    }
    for (int ch = 0; ch < e->channels_out; ch++) {
      e->tt[gr][ch].block_type = blocktype[ch];
      e->tt[gr][ch].mixed_block_flag = 0;
    }
  }
  e->ptrace_cur = NULL;
  adjust_ATH(e);
  lj_mdct_sub48(e, e->mfbuf[0], e->mfbuf[1]);
  e->mode_ext = 0; /* MPG_MD_LR_LR */
  if (e->mode_joint) {                         /* Encoder.js:524-561: M/S when its perceptual entropy is not higher and the block types agree */
    double sum_pe_MS = 0., sum_pe_LR = 0.;
    for (int gr = 0; gr < e->mode_gr; gr++)
      for (int ch = 0; ch < e->channels_out; ch++) { sum_pe_MS += pe_MS[gr][ch]; sum_pe_LR += pe[gr][ch]; }
    if (sum_pe_MS <= 1.00 * sum_pe_LR) {
      const GrInfo* gi0 = e->tt[0];
      const GrInfo* gi1 = e->tt[e->mode_gr - 1];
      if (gi0[0].block_type == gi0[1].block_type && gi1[0].block_type == gi1[1].block_type) e->mode_ext = 2; /* MPG_MD_MS_LR */
    }
  }
  PsyRatio (*masking)[2] = e->mode_ext == 2 ? masking_MS : masking_LR;
  double (*pe_use)[2] = e->mode_ext == 2 ? pe_MS : pe;

  if (tracing) {
    for (int gr = 0; gr < 2; gr++) for (int ch = 0; ch < e->channels_out; ch++) {
      for (int i = 0; i < 576; i++) tr.xr[gr][ch][i] = e->tt[gr][ch].xr[i].v;
      for (int sb = 0; sb < SBMAX_l; sb++) { tr.en_l[gr][ch][sb] = masking[gr][ch].en.l[sb].v; tr.thm_l[gr][ch][sb] = masking[gr][ch].thm.l[sb].v; }
      for (int sb = 0; sb < SBMAX_s; sb++) for (int b = 0; b < 3; b++) { tr.en_s[gr][ch][sb][b] = masking[gr][ch].en.s[sb][b].v; tr.thm_s[gr][ch][sb][b] = masking[gr][ch].thm.s[sb][b].v; }
      tr.blocktype[gr][ch] = e->tt[gr][ch].block_type;
    }
    tr.ath_adjust = e->ath_adjust;
    tr.padding = e->padding;
    for (int ch = 0; ch < 2; ch++) { tr.old_value_in[ch] = e->OldValue[ch]; tr.cur_step_in[ch] = e->CurrentStep[ch]; }
  }

  /* PE FIR (Encoder.js:602-627): kept for fidelity; PE is dead under disable_reservoir */
  {
    for (int i = 0; i < 18; i++) e->pefirbuf[i] = e->pefirbuf[i + 1];
    double f = 0.0;
    for (int gr = 0; gr < e->mode_gr; gr++) for (int ch = 0; ch < e->channels_out; ch++) f += pe_use[gr][ch];
    e->pefirbuf[18] = f;
    static const double fircoef[9] = {-0.0207887 * 5, -0.0378413 * 5, -0.0432472 * 5, -0.031183 * 5, 7.79609e-18 * 5,
                                      0.0467745 * 5, 0.10091 * 5, 0.151365 * 5, 0.187098 * 5};
    f = e->pefirbuf[9];
    for (int i = 0; i < 9; i++) f += (e->pefirbuf[i] + e->pefirbuf[18 - i]) * fircoef[i];
    f = (670 * 5 * e->mode_gr * e->channels_out) / f;
    for (int gr = 0; gr < e->mode_gr; gr++) for (int ch = 0; ch < e->channels_out; ch++) pe_use[gr][ch] *= f;
  }
  e->qtrace_cur = (tracing && e->qtrace && e->trace_n < e->qtrace_cap) ? &e->qtrace[e->trace_n] : NULL;
  if (e->qtrace_cur) memset(e->qtrace_cur, 0, sizeof *e->qtrace_cur);
  if (e->qtrace_cur && e->qrtrace && e->trace_n < e->qrtrace_cap) memset(&e->qrtrace[e->trace_n], 0, sizeof *e->qrtrace);
  lj_iteration_loop(e, pe_use, ms_ener_ratio, masking);
  e->qtrace_cur = NULL;
  lj_format_bitstream(e);
  /* the frame lamejs throws on is traced (frame_bytes = LJ_ERR_BITSTREAM) but not handed out */
  int mp3count = e->bs_fatal ? LJ_ERR_BITSTREAM : lj_copy_buffer(e, mp3buf, mp3buf_size, 1);
  if (!e->bs_fatal) lj_add_vbr_frame(e);             /* Encoder.js:640-641 */
  if (tracing) {
    for (int gr = 0; gr < 2; gr++) for (int ch = 0; ch < e->channels_out; ch++) {
      const GrInfo& gi = e->tt[gr][ch];
      memcpy(tr.l3_enc[gr][ch], gi.l3_enc, sizeof gi.l3_enc);
      memcpy(tr.scalefac[gr][ch], gi.scalefac, sizeof gi.scalefac);
      tr.global_gain[gr][ch] = gi.global_gain; tr.part2_3_length[gr][ch] = gi.part2_3_length;
      tr.part2_length[gr][ch] = gi.part2_length; tr.big_values[gr][ch] = gi.big_values; tr.count1[gr][ch] = gi.count1;
      tr.scalefac_compress[gr][ch] = gi.scalefac_compress;
      for (int i = 0; i < 3; i++) { tr.table_select[gr][ch][i] = gi.table_select[i]; tr.subblock_gain[gr][ch][i] = gi.subblock_gain[i]; }
      tr.region0[gr][ch] = gi.region0_count; tr.region1[gr][ch] = gi.region1_count;
      tr.preflag[gr][ch] = gi.preflag; tr.scalefac_scale[gr][ch] = gi.scalefac_scale; tr.count1table[gr][ch] = gi.count1table_select;
    }
    for (int ch = 0; ch < 2; ch++) { for (int i = 0; i < 4; i++) tr.scfsi[ch][i] = e->scfsi[ch][i]; tr.old_value_out[ch] = e->OldValue[ch]; tr.cur_step_out[ch] = e->CurrentStep[ch]; }
    tr.frame_bytes = mp3count;
    e->trace[e->trace_n++] = tr;
  }
  return mp3count;
}

/* ---- resampler: fill_buffer_resample (Lame.js:1719-1843), blackman (:1691-1714), gcd (:1684) ---- */
static int rs_gcd(int i, int j) { return j != 0 ? rs_gcd(j, i % j) : i; }
static double rs_blackman(double x, double fcn, int l) {
  const double PI = 3.141592653589793;
  double wcn = (PI * fcn);
  x /= l;
  if (x < 0) x = 0;
  if (x > 1) x = 1;
  double x2 = x - .5;
  double bkwn = 0.42 - 0.5 * cos(2 * x * PI) + 0.08 * cos(4 * x * PI);
  if (fabs(x2) < 1e-9) return (wcn / PI);
  return (bkwn * sin(l * wcn * x2) / (PI * l * x2));
}
/* a read `arr[idx]` of a Float32Array of length n with a JS number index: undefined (-> NaN in arithmetic) unless idx is an
 * integer inside the array */
static inline double f32arr_get(const F32* arr, int n, double idx) {
  if (!(idx >= 0) || idx != floor(idx) || idx >= n) return NAN;
  return (double)arr[(int)idx];
}
static int fill_buffer_resample(LjEnc* e, F32* outbuf, int outbufPos, int desired_len, const F32* inbuf, int inbuf_n,
                                double in_bufferPos, double len, double* num_used, int ch) {
  int i, j = 0, k;
  int bpc = e->out_samplerate / rs_gcd(e->out_samplerate, e->in_samplerate);
  if (bpc > 320) bpc = 320;
  const int intratio = (fabs(e->resample_ratio - floor(.5 + e->resample_ratio)) < .0001) ? 1 : 0;
  double fcn = 1.00 / e->resample_ratio;
  if (fcn > 1.00) fcn = 1.00;
  int filter_l = 31;
  filter_l += intratio;
  const int BLACKSIZE = filter_l + 1;
  const double half = filter_l / 2.0;          /* `filter_l / 2` is a float division in JS: 15.5 or 16 */
  if (e->resample_init == 0) {
    memset(e->inbuf_old, 0, sizeof e->inbuf_old);
    e->blackfilt = (F32(*)[33])calloc(2 * bpc + 1, sizeof(F32[33]));
    e->itime[0] = e->itime[1] = 0;
    for (j = 0; j <= 2 * bpc; j++) {
      double sum = 0.;
      double offset = (j - bpc) / (2. * bpc);
      for (i = 0; i <= filter_l; i++) {
        const double v = rs_blackman(i - offset, fcn, filter_l);
        e->blackfilt[j][i] = v;                 /* `sum += a[i] = v` adds the unrounded double */
        sum += v;
      }
      for (i = 0; i <= filter_l; i++) e->blackfilt[j][i] /= sum;
    }
    e->resample_init = 1;
    j = 0;
  }
  e->rs_bpc = bpc; e->rs_filter_l = filter_l;
  F32* inbuf_old = e->inbuf_old[ch];
  for (k = 0; k < desired_len; k++) {
    double time0 = k * e->resample_ratio;
    j = js_toint32(floor(time0 - e->itime[ch]));
    if ((filter_l + j - half) >= len) break;
    double offset = (time0 - e->itime[ch] - (j + .5 * (filter_l % 2)));
    int joff = js_toint32(floor((offset * 2 * bpc) + bpc + .5));
    double xvalue = 0.;
    for (i = 0; i <= filter_l; ++i) {
      int j2 = js_toint32(i + j - half);       /* 0 | x truncates toward zero */
      double y = (j2 < 0) ? f32arr_get(inbuf_old, BLACKSIZE, BLACKSIZE + j2) : f32arr_get(inbuf, inbuf_n, in_bufferPos + j2);
      xvalue += y * (double)e->blackfilt[joff][i];
    }
    outbuf[outbufPos + k] = xvalue;
  }
  double nu = filter_l + j - half;
  if (len < nu) nu = len;                       /* Math.min(len, ...) (no NaN operands here) */
  *num_used = nu;
  e->itime[ch] += nu - k * e->resample_ratio;
  if (nu >= BLACKSIZE) {
    for (i = 0; i < BLACKSIZE; i++) inbuf_old[i] = f32arr_get(inbuf, inbuf_n, in_bufferPos + nu + i - BLACKSIZE);
  } else {
    double n_shift = BLACKSIZE - nu;
    F32 tmp[33];
    memcpy(tmp, inbuf_old, sizeof tmp);        /* the JS loop reads ahead of what it writes (i + num_used >= i): in place is safe */
    for (i = 0; i < n_shift; ++i) inbuf_old[i] = f32arr_get(inbuf_old, BLACKSIZE, i + nu);
    for (j = 0; i < BLACKSIZE; ++i, ++j) inbuf_old[i] = f32arr_get(inbuf, inbuf_n, in_bufferPos + j);
    (void)tmp;
  }
  return k;
}

/* Lame.js:1527-1667.  nsamples is a JS number: lame_encode_flush passes a fractional count when it resamples. */
static int encode_buffer_sample(LjEnc* e, F32* in0, F32* in1, int in_n, double nsamples, uint8_t* mp3buf, int mp3buf_size) {
  int mp3size = 0;
  if (nsamples == 0) return 0;
  int mp3out = lj_copy_buffer(e, mp3buf, mp3buf_size, 0);   /* tags written into the bitstream (Lame.js:1541) */
  if (mp3out < 0) return mp3out;
  mp3buf += mp3out; mp3size += mp3out;
  if (bs_NEQ(e->scale, 0) && bs_NEQ(e->scale, 1.0)) {
    for (int i = 0; i < nsamples && i < in_n; ++i) {
      in0[i] *= e->scale;
      if (e->channels_out == 2) in1[i] *= e->scale;
    }
  }
  const int mf_needed = e->framesize + 752; /* calcNeeded (Lame.js:1516-1525): max(1024 + framesize - 272, 512 + framesize - 32) */
  const bool resample = (e->resample_ratio < .9999) || (e->resample_ratio > 1.0001);
  double pos = 0;
  while (nsamples > 0) {
    int n_out; double n_in;
    if (resample) {
      n_out = 0; n_in = 0;
      for (int ch = 0; ch < e->channels_out; ch++) {
        double used;
        n_out = fill_buffer_resample(e, e->mfbuf[ch], e->mf_size, e->framesize, ch == 0 ? in0 : in1, in_n, pos, nsamples, &used, ch);
        n_in = used;
      }
    } else {
      n_out = e->framesize < nsamples ? e->framesize : (int)nsamples;
      n_in = n_out;
      for (int i = 0; i < n_out; ++i) {
        e->mfbuf[0][e->mf_size + i] = in0[(int)pos + i];
        if (e->channels_out == 2) e->mfbuf[1][e->mf_size + i] = in1[(int)pos + i];
      }
    }
    nsamples -= n_in; pos += n_in;
    e->mf_size += n_out;
    if (e->mf_samples_to_encode < 1) e->mf_samples_to_encode = ENCDELAY + POSTDELAY;
    e->mf_samples_to_encode += n_out;
    if (e->mf_size >= mf_needed) {
      int buf_size = mp3buf_size - mp3size;
      if (mp3buf_size == 0) buf_size = 0;
      int ret = encode_mp3_frame(e, mp3buf, buf_size);
      e->frameNum++;
      if (ret < 0) return ret;
      mp3buf += ret; mp3size += ret;
      e->mf_size -= e->framesize;
      e->mf_samples_to_encode -= e->framesize;
      for (int ch = 0; ch < e->channels_out; ch++)
        for (int i = 0; i < e->mf_size; i++) e->mfbuf[ch][i] = e->mfbuf[ch][i + e->framesize];
    }
  }
  return mp3size;
}

/* lame_encode_buffer (Lame.js:1490-1514) incl. update_inbuffer_size (:1373-1379) */
static int encode_buffer(LjEnc* e, const int16_t* left, const int16_t* right, int src_n, double nsamples, uint8_t* out, int cap) {
  if (nsamples == 0) return 0;
  if (e->inb[0] == NULL || e->inb_nsamples < nsamples) {
    const int n = (int)nsamples;               /* new Float32Array(x): ToIndex truncates */
    free(e->inb[0]); free(e->inb[1]);
    e->inb[0] = (F32*)calloc(n > 0 ? n : 1, sizeof(F32));
    e->inb[1] = (F32*)calloc(n > 0 ? n : 1, sizeof(F32));
    e->inb_len = n; e->inb_nsamples = nsamples;
  }
  for (int i = 0; i < nsamples; i++) {
    if (i >= e->inb_len) break;                /* writes past the typed array are dropped */
    e->inb[0][i] = i < src_n ? left[i] : 0;
    if (e->num_channels > 1) e->inb[1][i] = i < src_n ? right[i] : 0;
  }
  return encode_buffer_sample(e, e->inb[0], e->inb[1], e->inb_len, nsamples, out, cap);
}

extern "C" {

LjEnc* lj_create(int channels, int samplerate, int kbps) {
  LjEnc* e = (LjEnc*)calloc(1, sizeof(LjEnc));
  if (!e) return NULL;
  if (lj_init_params(e, channels, samplerate, kbps) != 0) { free(e->s3_ll); free(e->s3_ss); free(e); return NULL; }
  return e;
}
/* output sample rate lame_init_params chooses (0 if the configuration is rejected before that point) */
int lj_query_out_samplerate(int channels, int samplerate, int kbps) {
  LjEnc* e = (LjEnc*)calloc(1, sizeof(LjEnc));
  if (!e) return 0;
  lj_init_params(e, channels, samplerate, kbps);
  const int r = e->out_samplerate;
  free(e->s3_ll); free(e->s3_ss); free(e);
  return r;
}
/* gfp.disable_reservoir = false (index.js:108 sets it true): a per-frame switch (Reservoir.js:158,217; BitStream.js:208),
 * so it can be flipped on a fresh encoder.  SURVEY.md 8(f2), oracle only. */
/* gfp.mode = JOINT_STEREO (index.js:104 fixes STEREO): lame_init_params derives the same parameters for both modes
 * (Lame.js:755-766,1310-1315); the difference is per frame -- four psycho-acoustic channels, the M/S decision, ms_convert and
 * reduce_side, the mode bits of the header.  SURVEY.md 8(f2), oracle only. */
int lj_enable_joint_stereo(LjEnc* e) {
  if (!e || e->frameNum != 0 || e->channels_out != 2) return -1;
  e->mode_joint = 1;
  return 0;
}
int lj_enable_reservoir(LjEnc* e) {
  if (!e || e->frameNum != 0) return -1;
  e->disable_reservoir = 0;
  return 0;
}
/* NOT lamejs: the reservoir with Java's integer division at Reservoir.js:283 (`Math.min(...) / 8`).  In JavaScript that
 * quotient has eighths, the sub-byte remainder of the stuffing is then drained IN FRONT of the next frame's main data and the
 * header's main_data_begin (truncated) no longer points at it: lamejs's reservoir streams do not decode
 * (tests/test_modes_oracle.py shows both).  This switch exists so that the reservoir machinery of the oracle can also be
 * checked by the independent decoder. */
int lj_enable_reservoir_integer_bytes(LjEnc* e) {
  if (lj_enable_reservoir(e) != 0) return -1;
  e->java_int_div = 1;
  return 0;
}
void lj_destroy(LjEnc* e) { if (e) { free(e->s3_ll); free(e->s3_ss); free(e->blackfilt); free(e->inb[0]); free(e->inb[1]); free(e); } }

/* index.js:117-130 + Lame.js:1490-1514.  Returns bytes written or a negative lame error. */
int lj_encode(LjEnc* e, const int16_t* left, const int16_t* right, int n, uint8_t* out, int cap) {
  if (!e) return -3;
  if (e->bs_fatal) return LJ_ERR_BITSTREAM;
  if (n == 0) return 0;
  if (e->channels_out == 1 || e->num_channels == 1) right = left;
  return encode_buffer(e, left, right, n, (double)n, out, cap);
}

/* index.js:132-135 + Lame.js:1381-1488; sample counts are JS numbers (fractional when resampling) */
int lj_flush(LjEnc* e, uint8_t* out, int cap) {
  if (!e) return -3;
  if (e->bs_fatal) return LJ_ERR_BITSTREAM;
  static const int16_t zeros[1152] = {0};
  int imp3 = 0, mp3count = 0;
  double samples_to_encode = e->mf_samples_to_encode - POSTDELAY;
  const int mf_needed = e->framesize + 752;
  if (e->mf_samples_to_encode < 1) return 0;
  if (e->in_samplerate != e->out_samplerate) samples_to_encode += 16. * e->out_samplerate / e->in_samplerate;
  double end_padding = e->framesize - fmod(samples_to_encode, (double)e->framesize);
  if (end_padding < 576) end_padding += e->framesize;
  e->encoder_padding = js_toint32(end_padding);
  double frames_left = (samples_to_encode + end_padding) / e->framesize;
  while (frames_left > 0 && imp3 >= 0) {
    double bunch = mf_needed - e->mf_size;
    int frame_num = e->frameNum;
    bunch *= e->in_samplerate;
    bunch /= e->out_samplerate;
    if (bunch > 1152) bunch = 1152;
    if (bunch < 1) bunch = 1;
    int remaining = cap - mp3count;
    if (cap == 0) remaining = 0;
    imp3 = encode_buffer(e, zeros, zeros, 1152, bunch, out, remaining);
    if (imp3 > 0) { out += imp3; mp3count += imp3; }
    frames_left -= (frame_num != e->frameNum) ? 1 : 0;
  }
  e->mf_samples_to_encode = 0;
  if (imp3 < 0) return imp3;
  lj_flush_bitstream(e);                  /* BitStream.js:757-815; with the reservoir disabled flushbits == 0 */
  int remaining = cap - mp3count;
  if (cap == 0) remaining = 0;
  imp3 = lj_copy_buffer(e, out, remaining, 1);
  if (imp3 < 0) return imp3;
  mp3count += imp3;
  return mp3count;
}

/* gfp.scale after lame_init_params: what lamejs multiplies every input sample by (the preset's, 1 when unset) */
double lj_get_scale(const LjEnc* e) { return e->scale; }
int lj_gain_clamps(const LjEnc* e) { return e->gain_clamps; }
void lj_set_trace(LjEnc* e, LjFrameTrace* buf, int cap) { e->trace = buf; e->trace_cap = cap; e->trace_n = 0; }
/* quantizer rows next to the frame trace: row k is filled together with lj_set_trace's row k (call it after lj_set_trace) */
void lj_set_quant_trace(LjEnc* e, LjQuantTrace* buf, int cap) { e->qtrace = buf; e->qtrace_cap = cap; }
int lj_quant_trace_size(void) { return (int)sizeof(LjQuantTrace); }
/* the rows lj_iteration_loop hands outer_loop, beside the quantizer rows: row k is filled together with lj_set_quant_trace's
 * row k (call it after lj_set_quant_trace) */
void lj_set_quant_row_trace(LjEnc* e, LjQuantRowTrace* buf, int cap) { e->qrtrace = buf; e->qrtrace_cap = cap; }
int lj_quant_row_trace_size(void) { return (int)sizeof(LjQuantRowTrace); }
/* psy rows, one per frame encoded from now on (independent of lj_set_trace) */
void lj_set_psy_trace(LjEnc* e, LjPsyTrace* buf, int cap) {
  e->ptrace = buf; e->ptrace_cap = cap; e->ptrace_n = 0;
  e->pbtrace = NULL; e->pbtrace_cap = 0;
}
/* block types beside the psy rows: row k is filled together with lj_set_psy_trace's row k (call it after lj_set_psy_trace) */
void lj_set_psy_block_trace(LjEnc* e, LjPsyBlockTrace* buf, int cap) { e->pbtrace = buf; e->pbtrace_cap = cap; }
int lj_psy_block_trace_size(void) { return (int)sizeof(LjPsyBlockTrace); }
int lj_psy_trace_count(const LjEnc* e) { return e->ptrace_n; }
int lj_psy_trace_size(void) { return (int)sizeof(LjPsyTrace); }
/* the attack threshold of the long-block channels (NsPsy attackthre, the preset's st_lrm) */
double lj_psy_attack_threshold(const LjEnc* e) { return e->attackthre; }
double lj_ath_aa_sensitivity(const LjEnc* e) { return e->ath_aaSensitivityP; }
/* partitions of the long (shortblock 0) or short blocks: the defined prefix of the psy trace's partition rows */
int lj_psy_npart(const LjEnc* e, int shortblock) { return shortblock ? e->npart_s : e->npart_l; }
int lj_trace_count(const LjEnc* e) { return e->trace_n; }
int lj_trace_size(void) { return (int)sizeof(LjFrameTrace); }
int lj_state_size(void) { return (int)sizeof(LjState); }
/* the state an encoder carries into its next call (the counterpart of a handle's state blob) */
int lj_get_state(const LjEnc* e, LjState* s) {
  memset(s, 0, sizeof *s);
  s->ath_adjust = e->ath_adjust; s->ath_adjust_limit = e->ath_adjustLimit;
  for (int ch = 0; ch < 2; ch++) {
    s->blocktype_old[ch] = e->blocktype_old[ch]; s->last_attacks[ch] = e->lastAttacks[ch];
    s->old_value[ch] = e->OldValue[ch]; s->current_step[ch] = e->CurrentStep[ch];
    for (int sb = 0; sb < SBMAX_l; sb++) { s->en_l[ch][sb] = e->en[ch].l[sb].v; s->thm_l[ch][sb] = e->thm[ch].l[sb].v; }
    for (int sb = 0; sb < SBMAX_s; sb++)
      for (int b = 0; b < 3; b++) { s->en_s[ch][sb][b] = e->en[ch].s[sb][b].v; s->thm_s[ch][sb][b] = e->thm[ch].s[sb][b].v; }
  }
  s->frames_done = e->frameNum; s->mf_size = e->mf_size; s->mf_samples_to_encode = e->mf_samples_to_encode;
  return (int)sizeof *s;
}
int lj_frame_bytes_for(const LjEnc* e, int padding) {
  return framebits(e->version, e->bitrate_index, e->out_samplerate, padding) / 8;
}

} /* extern "C" */
