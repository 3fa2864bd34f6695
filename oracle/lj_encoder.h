/* lj_encoder.h -- encoder state of the oracle (merged LameGlobalFlags + LameInternalFlags
 * restricted to what Mp3Encoder reaches; reference src/js/LameGlobalFlags.js,
 * src/js/LameInternalFlags.js, src/js/ATH.js, src/js/NsPsy.js).  TEST INFRASTRUCTURE. */
#ifndef LJ_ENCODER_H
#define LJ_ENCODER_H
#include "lj_core.h"

struct LjEnc {
  /* ---- user / derived global flags (gfp) ---- */
  int num_channels, in_samplerate, out_samplerate, brate, version;
  int mode_mono;                 /* gfp.mode == MONO */
  int quality;
  double scale;
  int lowpassfreq;
  double compression_ratio;
  int quant_comp, quant_comp_short;
  int exp_nspsytune;
  double msfix;
  double maskingadjust, maskingadjust_short;
  double ATHlower, ATHcurve; int ATHtype;
  double interChRatio;
  int short_blocks_coupled;      /* ShortBlock.short_block_coupled vs allowed */
  int useTemporal;
  int framesize;
  int frameNum;
  /* ---- internal flags (gfc) ---- */
  int channels_out, mode_gr, mode_ext;
  int bitrate_index, samplerate_index;
  double lowpass1, lowpass2, highpass1, highpass2;
  int noise_shaping, noise_shaping_amp, noise_shaping_stop, subblock_gain, use_best_huffman,
      full_outer_loop, substep_shaping, psymodel, sfb21_extra;
  int padding, frac_SpF, slot_lag;
  int OldValue[2], CurrentStep[2];
  double masking_lower;
  int bv_scf[576];
  int pseudohalf[SFBMAX];
  int sideinfo_len;
  F32 sb_sample[2][2][18][SBLIMIT];
  F32 amp_filter[32];
  double ResvSize, ResvMax;      /* JS numbers (Reservoir.js): integers as long as the reservoir is off */
  int sfb_l[SBMAX_l + 1], sfb_s[SBMAX_s + 1], psfb21[PSFB21 + 1], psfb12[PSFB12 + 1];
  /* psy tables */
  F32 minval_l[CBANDS], minval_s[CBANDS];
  F32 nb_1[4][CBANDS], nb_2[4][CBANDS], nb_s1[4][CBANDS], nb_s2[4][CBANDS];
  F32 *s3_ss, *s3_ll; int n_s3_ss, n_s3_ll;
  double decay;
  PsyXmin thm[4], en[4];
  F32 tot_ener[4];
  F32 loudness_sq[2][2];
  F32 loudness_sq_save[2];
  F32 mld_l[SBMAX_l], mld_s[SBMAX_s];
  int bm_l[SBMAX_l], bo_l[SBMAX_l], bm_s[SBMAX_s], bo_s[SBMAX_s];
  int npart_l, npart_s;
  int s3ind[CBANDS][2], s3ind_s[CBANDS][2];
  int numlines_s[CBANDS], numlines_l[CBANDS];
  F32 rnumlines_l[CBANDS];
  F32 mld_cb_l[CBANDS], mld_cb_s[CBANDS];
  int blocktype_old[2];
  /* nsPsy */
  F32 last_en_subshort[4][9];
  int lastAttacks[4];
  F32 pefirbuf[19];
  F32 longfact[SBMAX_l], shortfact[SBMAX_s];
  double attackthre, attackthre_s;
  /* PSY */
  double mask_adjust, mask_adjust_short;
  F32 bo_l_weight[SBMAX_l], bo_s_weight[SBMAX_s];
  /* ATH */
  int ath_useAdjust; double ath_aaSensitivityP, ath_adjust, ath_adjustLimit, ath_decay, ath_floor;
  F32 ath_l[SBMAX_l], ath_s[SBMAX_s], ath_psfb21[PSFB21], ath_psfb12[PSFB12], ath_cb_l[CBANDS],
      ath_cb_s[CBANDS], ath_eql_w[BLKSIZE / 2];
  /* side info */
  GrInfo tt[2][2];
  double main_data_begin, resvDrain_pre, resvDrain_post;   /* JS numbers: `/ 8` is not an integer division (Reservoir.js:283, BitStream.js:849) */
  int scfsi[2][4];
  /* resampler (Lame.js:1691-1843): per-call state exactly as lamejs keeps it */
  double resample_ratio;
  int resample_init;
  int rs_bpc, rs_filter_l;
  F32 inbuf_old[2][33];
  F32 (*blackfilt)[33];          /* [2 * bpc + 1][BLACKSIZE] */
  double itime[2];
  /* gfc.in_buffer_0/1 (Lame.js:1373-1379): grow-only Float32Arrays; a fractional length truncates, stale contents stay */
  F32* inb[2]; int inb_len; double inb_nsamples;
  /* stream driver */
  F32 mfbuf[2][MFSIZE];
  int mf_size, mf_samples_to_encode;
  int frame_init_done;
  /* quantizer tables (QuantizePVT.js:206-211) */
  F32 pow20[Q_MAX + Q_MAX2 + 1], ipow20[Q_MAX], pow43[PRECALC_SIZE], adj43[PRECALC_SIZE];
  /* FFT windows (FFT.js:21-22) */
  F32 fft_window[BLKSIZE], fft_window_s[BLKSIZE_s / 2];
  double ma_max_i1, ma_max_i2, ma_max_m;
  /* bitstream (BitStream.js closure state, one frame at a time) */
  uint8_t bs_buf[16384 + 131072];
  int bs_totbit, bs_byteidx, bs_bitidx;
  /* gfc.header[MAX_HEADER_BUF] ring (LameInternalFlags.js, BitStream.js:96-101,218-229,407-419) */
  struct LjHeader { int write_timing; int ptr; uint8_t buf[40]; } header[256];
  int h_ptr, w_ptr;
  int ancillary_flag;
  /* trace */
  LjFrameTrace* trace; int trace_cap, trace_n;
  LjQuantTrace* qtrace; int qtrace_cap;
  LjQuantTrace* qtrace_cur;      /* the quantizer row of the frame being encoded while tracing, else NULL (lj_quant.cpp) */
  LjQuantRowTrace* qrtrace; int qrtrace_cap;   /* rows beside qtrace's (lj_set_quant_row_trace), or NULL */
  LjPsyTrace* ptrace; int ptrace_cap, ptrace_n;
  LjPsyTrace* ptrace_cur;        /* the psy row of the frame being encoded while tracing, else NULL (lj_psy_trace_*) */
  LjPsyBlockTrace* pbtrace; int pbtrace_cap;   /* rows beside ptrace's (lj_set_psy_block_trace), or NULL */
  /* Xing / LAME tag state (VBRSeekInfo.js, LameInternalFlags.js:170; lj_vbrtag.cpp).  nMusicCRC and nBytesWritten are
   * maintained by copy_buffer on every call whether or not a tag is written (BitStream.js:924-935). */
  int nMusicCRC; long long nBytesWritten;
  int bWriteVbrTag, vbr_TotalFrameSize, vbr_nframes, vbr_sum, vbr_seen, vbr_want, vbr_pos;
  int vbr_bag[400];
  /* modes Mp3Encoder does not reach (SURVEY.md 8(f2)): gfp.disable_reservoir (index.js:108 sets it), gfp.mode == JOINT_STEREO */
  int disable_reservoir, mode_joint;
  int java_int_div;                /* test switch: integer byte counts where Java (and LAME) divide integers, see lj_quant.cpp ResvFrameEnd */
  int encoder_padding;             /* gfp.encoder_padding, set by lame_encode_flush (Lame.js:1412) */
  int gain_clamps;                 /* times bin_search_StepSize clamped global_gain > 255 (coverage of loud input) */
  int bs_fatal;                    /* format_bitstream's consistency check failed: lamejs threw (LJ_ERR_BITSTREAM) */
  double lowpass_final;            /* gfp.lowpassfreq after lame_init_params (Lame.js:884-896) */
};

/* returned by lj_encode / lj_encode_f32 / lj_flush for the call in which lamejs throws, and for every later call */
#define LJ_ERR_BITSTREAM (-10)

/* lj_init.cpp */
int  lj_init_params(LjEnc* e, int channels, int samplerate, int kbps);
/* lj_mdct.cpp */
void lj_mdct_sub48(LjEnc* e, const F32* w0, const F32* w1);
/* lj_psy.cpp */
int  lj_psycho_anal_ns(LjEnc* e, const F32* buf0, const F32* buf1, int bufPos, int gr_out,
                       PsyRatio masking_ratio[2][2], PsyRatio masking_MS_ratio[2][2], double* percep_entropy,
                       double* percep_MS_entropy, F32* energy, int* blocktype_d);
void lj_psymodel_init(LjEnc* e);
/* lj_init.cpp: the psy trace's row of psy call (gr, chn) of the frame being encoded (lj_set_psy_trace); no-ops when the
 * trace is off and for the mid / side channels.  Kept out of lj_psy.cpp, whose per-frame branches the tests account for. */
void lj_psy_trace_attacks(LjEnc* e, int gr, int chn, const F32* en_subshort, const int* ns_attacks);
void lj_psy_trace_long(LjEnc* e, int gr, int chn, const F32* eb_l, const int* mask_idx_l);
void lj_psy_trace_short(LjEnc* e, int gr, int chn, int sblock, const F32* eb_s);
/* lj_init.cpp: the hand-over rows of granule (gr, ch) beside the quant trace's row t (LjQuantRowTrace); a no-op when t is
 * NULL (the trace is off) or no row trace is set.  Kept out of lj_quant.cpp for the same reason; its caller is a tap line
 * there. */
void lj_quant_trace_rows(LjEnc* e, const LjQuantTrace* t, int gr, int ch, const GrInfo* cod_info, const F32* xrpow, bool have);
double lj_ATHformula(double f, const LjEnc* e);
/* lj_quant.cpp */
void lj_iteration_init(LjEnc* e);
void lj_iteration_loop(LjEnc* e, double pe[2][2], const double* ms_ener_ratio, PsyRatio ratio[2][2]);
int  lj_getframebits(const LjEnc* e);
/* lj_bitstream.cpp */
void lj_format_bitstream(LjEnc* e);
void lj_flush_bitstream(LjEnc* e);
int  lj_copy_buffer(LjEnc* e, uint8_t* out, int cap, int mp3data);
/* lj_vbrtag.cpp */
void lj_update_music_crc(LjEnc* e, const uint8_t* buf, int size);
void lj_add_vbr_frame(LjEnc* e);
#endif
