/* lj_core.h -- types shared by the oracle translation units.
 *
 * TEST INFRASTRUCTURE.  The oracle is a single-threaded CPU restatement of
 * zhuker/lamejs (src/js, commit 582bbba) for the Mp3Encoder configuration
 * (CBR, mode STEREO/MONO, quality 3, no reservoir; reference src/js/index.js:66-136),
 * plus the Xing / Info / LAME tag writer Mp3Encoder leaves switched off (lj_vbrtag.cpp).  It is the parity checker for the CUDA product and
 * the timed CPU baseline.  Nothing in the product links or imports it.
 *
 * PINNED against the reference itself: the unmodified lamejs sources run in the
 * build image under Qt's QJSEngine (tools/jsrun/); tests/test_lamejs_pin.py checks
 * this restatement byte for byte against 306 lamejs-made fixtures (every sample
 * rate x bitrate x channel count, long streams, odd chunkings, the resampling
 * configurations) and against lamejs's own per-frame intermediates;
 * tests/test_tag_oracle.py does the same for the tag / CRC / WAV-header row.
 * Older, independent checks remain: derivable known answers
 * (tests/test_oracle_kat.py) and an ISO 11172-3 decoder round trip
 * (tests/test_oracle_decode.py).
 *
 * Arithmetic model (SURVEY.md fact 2): every JS local is an IEEE double; a
 * store into a Float32Array rounds to float32 (RNE), a store into an
 * Int32Array applies ToInt32.  `F32` below makes that automatic: reading it
 * yields a double, writing it rounds.
 */
#ifndef LJ_CORE_H
#define LJ_CORE_H

#include <math.h>
#include <stdint.h>
#include <string.h>
#include "js_math.h"

struct F32 {
  float v;
  F32() : v(0.0f) {}
  operator double() const { return (double)v; }
  F32& operator=(double d) { v = (float)d; return *this; }
  F32& operator+=(double d) { v = (float)((double)v + d); return *this; }
  F32& operator-=(double d) { v = (float)((double)v - d); return *this; }
  F32& operator*=(double d) { v = (float)((double)v * d); return *this; }
  F32& operator/=(double d) { v = (float)((double)v / d); return *this; }
};

/* ToInt32 (ECMA-262 7.1.6): the `0 | x` idiom and Int32Array stores. */
static inline int32_t js_toint32(double d) {
  if (d != d || d == INFINITY || d == -INFINITY) return 0;
  if (d > -2147483649.0 && d < 2147483648.0) return (int32_t)d; /* truncation */
  double t = trunc(d);
  double m = fmod(t, 4294967296.0);
  if (m < 0) m += 4294967296.0;
  return (int32_t)(uint32_t)m;
}
/* Math.max / Math.min: NaN-propagating, -0 < +0. */
static inline double js_max(double a, double b) {
  if (a != a || b != b) return NAN;
  if (a == 0.0 && b == 0.0) return signbit(a) ? b : a;
  return a > b ? a : b;
}
static inline double js_min(double a, double b) {
  if (a != a || b != b) return NAN;
  if (a == 0.0 && b == 0.0) return signbit(a) ? a : b;
  return a < b ? a : b;
}
/* BitStream.EQ / NEQ (src/js/BitStream.js:22-30) */
static inline bool bs_EQ(double a, double b) {
  return (fabs(a) > fabs(b)) ? (fabs(a - b) <= (fabs(a) * 1e-6)) : (fabs(a - b) <= (fabs(b) * 1e-6));
}
static inline bool bs_NEQ(double a, double b) { return !bs_EQ(a, b); }

#define LJ_SQRT2 1.41421356237309504880

enum { SBLIMIT = 32, CBANDS = 64, SBPSY_l = 21, SBPSY_s = 12, SBMAX_l = 22, SBMAX_s = 13,
       PSFB21 = 6, PSFB12 = 6, BLKSIZE = 1024, HBLKSIZE = 513, BLKSIZE_s = 256, HBLKSIZE_s = 129,
       NORM_TYPE = 0, START_TYPE = 1, SHORT_TYPE = 2, STOP_TYPE = 3, SFBMAX = 39,
       ENCDELAY = 576, POSTDELAY = 1152, MDCTDELAY = 48, FFTOFFSET = 272, MFSIZE = 3984,
       MAX_BITS_PER_CHANNEL = 4095, MAX_BITS_PER_GRANULE = 7680, LARGE_BITS = 100000,
       IXMAX_VAL = 8206, PRECALC_SIZE = 8208, Q_MAX = 257, Q_MAX2 = 116 };

struct GrInfo {
  F32 xr[576];
  int l3_enc[576];
  int scalefac[SFBMAX];
  double xrpow_max;
  int part2_3_length, big_values, count1, global_gain, scalefac_compress, block_type, mixed_block_flag;
  int table_select[3];
  int subblock_gain[4];
  int region0_count, region1_count, preflag, scalefac_scale, count1table_select, part2_length;
  int sfb_lmax, sfb_smin, psy_lmax, sfbmax, psymax, sfbdivide;
  int width[SFBMAX], window[SFBMAX];
  int count1bits;
  int slen[4];
  const int* sfb_partition_table;   /* MPEG-2 LSF: row of nr_of_sfb_block (QuantizePVT.js:116-122) */
  int max_nonzero_coeff;
};

struct PsyXmin { F32 l[SBMAX_l]; F32 s[SBMAX_s][3]; };
struct PsyRatio { PsyXmin thm, en; };

struct CalcNoiseResult { double over_noise, tot_noise, max_noise; int over_count; double over_SSD; int bits; };
struct CalcNoiseData { int global_gain; int sfb_count1; int step[SFBMAX]; F32 noise[SFBMAX]; F32 noise_log[SFBMAX]; };

/* per-frame trace record handed to the tests (all intermediates the CUDA stages are compared with) */
struct LjFrameTrace {
  float xr[2][2][576];            /* [gr][ch] MDCT output (before quantizer reorder/zeroing) */
  float en_l[2][2][SBMAX_l], thm_l[2][2][SBMAX_l];
  float en_s[2][2][SBMAX_s][3], thm_s[2][2][SBMAX_s][3];
  int   blocktype[2][2];
  double ath_adjust;              /* ATH.adjust after adjust_ATH of this frame */
  int   l3_enc[2][2][576];
  int   global_gain[2][2], part2_3_length[2][2], part2_length[2][2], big_values[2][2], count1[2][2];
  int   scalefac[2][2][SFBMAX];
  int   scalefac_compress[2][2], table_select[2][2][3], region0[2][2], region1[2][2];
  int   preflag[2][2], scalefac_scale[2][2], count1table[2][2], subblock_gain[2][2][3];
  int   scfsi[2][4];
  int   frame_bytes, padding;
  int   old_value_in[2], old_value_out[2], cur_step_in[2], cur_step_out[2];
};

/* per-frame record of the quantizer's inputs (lj_set_quant_trace), row k belonging to LjFrameTrace row k.  A record of its own,
 * so that the layout of LjFrameTrace, which callers size their buffers by, stays as it was.
 * What outer_loop receives (lj_iteration_loop): calc_xmin's l3_xmin (psymax bands; 0 elsewhere and for granules without
 * energy), max_nonzero_coeff after calc_xmin, xrpow_max after init_xrpow (before the rate loop raises it). */
struct LjQuantTrace {
  float xmin[2][2][SFBMAX];
  int   max_nonzero_coeff[2][2];
  double xrpow_max[2][2];
  int   old_value_mid[2], cur_step_mid[2];   /* MPEG-1: OldValue / CurrentStep after gr0, where gr1's search starts; 0 for LSF */
};

/* per-frame record of the rows lj_iteration_loop hands outer_loop (lj_set_quant_row_trace), row k belonging to LjQuantTrace
 * row k.  A record of its own, so that LjQuantTrace, which callers size their buffers by, keeps its layout.
 *   xrq    cod_info.xr as outer_loop receives it: short blocks in the quantizer's band order, analog silence zeroed
 *   xrpow  init_xrpow's |xr|^(3/4), every line (the rate loop rescales it later)
 *   have   init_xrpow's result: 0 for a granule without energy, which skips calc_xmin and outer_loop */
struct LjQuantRowTrace {
  float xrq[2][2][576];
  float xrpow[2][2][576];
  int   have[2][2];
};

/* per-frame record of the psy model's per-granule analysis (lj_set_psy_trace), [gr][ch] = psy call G k + gr of frame k.  A
 * record of its own, like LjQuantTrace.  Only the first npart_l / npart_s partitions are defined (0 beyond).
 *   eb_l, mask_idx_l  calc_energy's partition energies and calc_mask_index_l's indices
 *   peaks             en_subshort[3..11]: max(1, |high-passed sample|) over each 64-sample sub-block
 *   loudness          loudness_sq_save[ch] after the call (psycho_loudness_approx of this granule)
 *   attack            ns_attacks after the `ratio < 1.7` pass, before the lastAttacks rule
 *   eb_s, ecb_s       compute_masking_s of each short block: its partition energies and the spreading sum it stores into nb_s1 */
struct LjPsyTrace {
  float eb_l[2][2][CBANDS];
  float peaks[2][2][9];
  float loudness[2][2];
  float eb_s[2][2][3][CBANDS];
  float ecb_s[2][2][3][CBANDS];
  int   mask_idx_l[2][2][CBANDS];
  int   attack[2][2][4];
};

/* per-frame record of the block type each psy call found (lj_set_psy_block_trace), row k belonging to LjPsyTrace row k.  A
 * record of its own, like LjQuantTrace, so that LjPsyTrace keeps its layout.
 *   blocktype_old     gfc.blocktype_old as call G k + gr found it: what compute_masking_s and the long-block thresholds read,
 *                     before block_type_set turns it into the granule's block type */
struct LjPsyBlockTrace {
  int   blocktype_old[2][2];
};

/* what an encoder carries from one call to the next (lj_get_state) */
struct LjState {
  double ath_adjust, ath_adjust_limit;
  int   blocktype_old[2], last_attacks[2], old_value[2], current_step[2];
  int   frames_done, mf_size, mf_samples_to_encode, pad_;
  /* gfc.en / gfc.thm: the masking the psy model hands the next granule */
  float en_l[2][SBMAX_l], thm_l[2][SBMAX_l], en_s[2][SBMAX_s][3], thm_s[2][SBMAX_s][3];
};

#endif
