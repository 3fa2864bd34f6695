/* mp3_config.h -- per-(channels, samplerate, kbps) constants of the H100 MP3 encoder.
 *
 * Everything lamejs derives once in `new Mp3Encoder(ch, sr, kbps)` (reference src/js/index.js:66-115 ->
 * src/js/Lame.js:747-1371 lame_init_params, src/js/Presets.js:246-358, src/js/QuantizePVT.js:229-414
 * iteration_init, src/js/PsyModel.js:2537-2822 psymodel_init, src/js/FFT.js:226-242 init_fft) is
 * computed on the host into one flat, trivially-copyable block (`Mp3Tables`) that is uploaded to HBM
 * once per configuration and read by every kernel through a single pointer.
 */
#ifndef MP3B200_CONFIG_H
#define MP3B200_CONFIG_H
#include <stdint.h>

#define MP3_CBANDS 64
#define MP3_SBMAX_L 22
#define MP3_SBMAX_S 13
#define MP3_SFBMAX 39
#define MP3_S3_MAX 2048     /* ragged spreading rows, flattened */
#define MP3_PRECALC 8208
#define MP3_QMAX 257
#define MP3_QMAX2 116

/* Band geometry of one granule-channel as the quantizer walks it: [0] long / start / stop blocks (22 bands of the long
 * partition, window 3), [1] short blocks (13 bands x 3 windows, lines reordered band-major, Quantize.js:262-278). */
struct Mp3Geo {
  unsigned char width[MP3_SFBMAX + 1], window[MP3_SFBMAX + 1];
  short start[MP3_SFBMAX + 1];
  unsigned char sfb_of_line[576];
  short reorder[576];             /* position of MDCT line i in the quantizer's line order */
};

/* convert_partition2scalefac (PsyModel.js:1206-1266) walks partitions and bands with one cursor; its control flow depends
 * only on the tables, so each band's slice is worked out once: band sbi starts from (1 - weight[sbi-1]) * x[init] (init >= 0),
 * adds x[start..end) in order, is stored, then gains weight[sbi] * x[bound] (bound >= 0).  init == -2: band stays 0. */
struct Mp3Conv { short init[MP3_SBMAX_L], start[MP3_SBMAX_L], end[MP3_SBMAX_L], bound[MP3_SBMAX_L]; };

struct Mp3Tables {
  /* ---- scalars ---- */
  int nch, samplerate, kbps, mono;
  int bitrate_index, samplerate_index, sideinfo_len, frac_SpF;
  int frame_bytes_nopad;          /* floor((version + 1) * 72000 * kbps / sr) */
  int version;                    /* header version bit: 1 = MPEG-1 (32/44.1/48 kHz), 0 = MPEG-2 and MPEG-2.5 (LSF) */
  int mode_gr;                    /* granules per frame: 2 (MPEG-1) or 1 (LSF); a frame carries 576 * mode_gr samples */
  int mpeg25;                     /* output rate below 16 kHz: sync word 0xFFE */
  int noise_shaping;              /* 1 or 2 (sfscale) */
  int quant_comp, quant_comp_short;
  int coupled_short_blocks;
  int npart_l, npart_s;
  int scale_applied;              /* gfp.scale != 1 */
  double scale;
  double masking_lower_long, masking_lower_short;   /* 10^(mask_adjust*0.1), CBRNewIterationLoop.js:64 */
  double interch_ratio;
  double attack_threshold;
  double aa_sensitivity_p, ath_floor, decay;
  double ma_max_i1, ma_max_i2, ma_max_m;
  /* mask_add needs i = 0 | (Math.log10(ratio) * 16) for 1 <= ratio < 10^1.5 (PsyModel.js:433,461): l16_thr[k] is the smallest
   * double whose value of that expression (with this library's fdlibm log10) is >= k, found by bisection over the bit
   * patterns and checked to be a clean step around it; then i = #{k in 1..24 : ratio >= l16_thr[k]} -- 24 comparisons instead
   * of an fdlibm log10 (one division, ~40 FP64 operations) per spreading term.  l16_ok == 0: fall back to log10. */
  double l16_thr[25];
  int l16_ok;
  /* ---- filterbank ---- */
  float amp_filter[32];
  /* ---- scalefactor bands ---- */
  int sfb_l[MP3_SBMAX_L + 1], sfb_s[MP3_SBMAX_S + 1], psfb21[7], psfb12[7];
  int bv_scf[576];
  Mp3Geo geo[2];
  /* ---- psycho-acoustic partitions ---- */
  int numlines_l[MP3_CBANDS], numlines_s[MP3_CBANDS];
  int line0_l[MP3_CBANDS + 1], line0_s[MP3_CBANDS + 1];   /* prefix sums of numlines (ours) */
  float rnumlines_l[MP3_CBANDS];
  int s3lo_l[MP3_CBANDS], s3hi_l[MP3_CBANDS], s3off_l[MP3_CBANDS + 1];
  int s3lo_s[MP3_CBANDS], s3hi_s[MP3_CBANDS], s3off_s[MP3_CBANDS + 1];
  float s3_ll[MP3_S3_MAX], s3_ss[MP3_S3_MAX];
  int bo_l[MP3_SBMAX_L], bo_s[MP3_SBMAX_S];
  float bo_l_weight[MP3_SBMAX_L], bo_s_weight[MP3_SBMAX_S];
  Mp3Conv conv_l, conv_s;
  float ath_cb_l[MP3_CBANDS], ath_cb_s[MP3_CBANDS];
  float eql_w[512];
  /* ---- ATH per scalefactor band ---- */
  float ath_l[MP3_SBMAX_L], ath_s[MP3_SBMAX_S], ath_psfb21[6], ath_psfb12[6];
  float longfact[MP3_SBMAX_L], shortfact[MP3_SBMAX_S];
  /* ---- FFT ---- */
  float fft_window[1024], fft_window_s[128];
  /* FHT twiddles per stage: entry i holds (c1, s1, c2, s2) for butterfly index i (1..kx-1);
   * stage t has kx = 2*4^t entries starting at tw_off[t].  Produced by the same double recurrence
   * the reference runs inside fht() (FFT.js:70-111). */
  int tw_off[5];
  double tw[4 * 176];
  /* ---- quantizer ---- */
  float pow20[MP3_QMAX + MP3_QMAX2 + 1], ipow20[MP3_QMAX], pow43[MP3_PRECALC], adj43[MP3_PRECALC];
  /* per global_gain: IXMAX_VAL / ipow20 (count_bits range check) and (1 - 0.4054) / ipow20 (0/1 quantizer threshold),
   * the same IEEE double divisions the encoder would do per call (Takehiro.js:178,633) */
  double ixmax_over_istep[MP3_QMAX], cmp01_over_istep[MP3_QMAX];
};

/* What the Xing / Info / LAME tag frame says about a configuration (reference src/js/VBRTag.js:281-364,558-802): the
 * values `lame_init_params` leaves in gfp / gfc for the fields of the tag.  Host only; not part of Mp3Tables. */
struct Mp3TagParams {
  int version, mpeg25, samplerate, kbps, mono;
  int bitrate_index, samplerate_index, sideinfo_len;
  int frame_bytes;                /* VBR_seek_table.TotalFrameSize: (version + 1) * 72000 * kbps / samplerate, integer quotient */
  int fits;                       /* InitVbrTag keeps the tag only if the frame holds side info + 156 bytes (VBRTag.js:508-513) */
  int lowpass_byte;               /* trunc(min(255, lowpassfreq / 100 + .5)) */
  int quality_byte;               /* 100 - 10 * VBR_q - quality = 57 (VBR_q 4, quality 3) */
  int flags_byte;                 /* ATHtype | nspsytune << 4 | safejoint << 5 */
  int misc_byte;                  /* noise_shaping | stereo mode << 2 | non-optimal << 5 | source rate class << 6 */
};

/* lamejs's resampler for an integer rate ratio r = in / out (fill_buffer_resample, Lame.js:1719-1843): one 33-tap filter,
 * output m = Float32(sum_i (double)h[i] * x[r m - 16 + i]) over the (scaled) input x, zero before 0 and past the end. */
#define MP3_RS_TAPS 33
#define MP3_RS_HALF 16
struct Mp3Resample {
  int in_rate;                    /* the caller's rate; Mp3Tables::samplerate is the rate lamejs encodes at */
  int ratio;                      /* in_rate / samplerate: 1 = no resampling */
  float h[MP3_RS_TAPS];           /* blackfilt[1] of the filter bank (Lame.js:1746-1760) */
};

/* the output rate lame_init_params picks (Lame.js:285-364), or 0 for a channel count lamejs cannot take */
int mp3_out_samplerate(int channels, int samplerate, int kbps);

/* Derives everything about the caller's (channels, samplerate, kbps) in one pass: the tables, the resampler and the tag's
 * fields.  Returns 0, or -1 when lamejs itself would fail or would resample (out_samplerate != samplerate).  With flags &
 * MP3B200_RESAMPLE a configuration whose output rate divides the input rate (|ratio - round(ratio)| < 1e-4, lamejs's own
 * test) is also accepted: the tables are then those of the output rate and `rs` holds the filter. */
int mp3_build_config(int channels, int samplerate, int kbps, int flags, Mp3Tables* t, Mp3Resample* rs, Mp3TagParams* tag);

#endif
