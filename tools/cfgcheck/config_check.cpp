// CPU cross-check of the PRODUCT's per-configuration constant block (lamejs_b200/csrc/mp3_config.cpp, Mp3Tables) against
// the ORACLE's lame_init_params restatement (oracle/lj_init.cpp, LjEnc) for every configuration both accept.  The product's
// tables are built with MP3B200_RESAMPLE, so the configurations lamejs resamples by an integer ratio are compared too: their
// tables are those of the output rate, with the low-pass lamejs computed from the input rate.
// Test infrastructure (links oracle/): run by tests/test_config_tables.py; no GPU needed.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../lamejs_b200/csrc/mp3_config.h"
#include "../../oracle/lj_encoder.h"
extern "C" { LjEnc* lj_create(int, int, int); void lj_destroy(LjEnc*); }

static int bad = 0;
static int resampled = 0;        /* resampled configurations compared */
#define CHK(cond, ...) do { if (!(cond)) { if (bad < 40) { printf("  MISMATCH "); printf(__VA_ARGS__); printf("\n"); } bad++; } } while (0)
static bool feq(float a, float b) { return memcmp(&a, &b, 4) == 0; }
static bool deq(double a, double b) { return memcmp(&a, &b, 8) == 0; }

static int check(int ch, int sr, int kbps) {
  Mp3Tables* t = (Mp3Tables*)malloc(sizeof(Mp3Tables));
  Mp3Resample rs;
  Mp3TagParams tag;
  const int rc = mp3_build_config(ch, sr, kbps, 1 /* MP3B200_RESAMPLE */, t, &rs, &tag);
  LjEnc* e = lj_create(ch, sr, kbps);
  /* the flagged product takes what lamejs encodes at the input rate and what it resamples by an integer ratio (lamejs's own
   * test, |in / out - round(in / out)| < 1e-4) */
  const double ratio = e ? (double)e->in_samplerate / e->out_samplerate : 0;
  const bool integer_ratio = e && fabs(ratio - floor(.5 + ratio)) < 1e-4;
  const bool oracle_takes = e && (e->out_samplerate == e->in_samplerate || integer_ratio);
  if (rc != 0 || !oracle_takes) {
    int r = 0;
    if ((rc == 0) != oracle_takes) { printf("cfg %d %d %d: acceptance differs (product rc %d, oracle in %d out %d)\n", ch, sr, kbps, rc, e ? e->in_samplerate : 0, e ? e->out_samplerate : 0); r = 1; }
    free(t); if (e) lj_destroy(e);
    return r;
  }
  const int before = bad;
  CHK(t->samplerate == e->out_samplerate && rs.in_rate == sr && rs.ratio == e->in_samplerate / e->out_samplerate,
      "rates: product %d / %d (ratio %d) vs oracle in %d out %d", rs.in_rate, t->samplerate, rs.ratio, e->in_samplerate, e->out_samplerate);
  if (e->out_samplerate != e->in_samplerate) resampled++;
  CHK(t->version == e->version && t->mode_gr == e->mode_gr, "version/mode_gr");
  CHK(t->bitrate_index == e->bitrate_index && t->samplerate_index == e->samplerate_index && t->kbps == e->brate, "indices %d %d %d vs %d %d %d", t->bitrate_index, t->samplerate_index, t->kbps, e->bitrate_index, e->samplerate_index, e->brate);
  CHK(t->sideinfo_len == e->sideinfo_len && t->frac_SpF == e->frac_SpF, "sideinfo/frac");
  CHK(t->noise_shaping == e->noise_shaping, "noise_shaping %d vs %d", t->noise_shaping, e->noise_shaping);
  CHK(t->coupled_short_blocks == e->short_blocks_coupled, "coupled");
  CHK(deq(t->scale, e->scale) && deq(t->interch_ratio, e->interChRatio) && deq(t->attack_threshold, e->attackthre), "scale/interch/attack");
  CHK(deq(t->aa_sensitivity_p, e->ath_aaSensitivityP) && deq(t->ath_floor, e->ath_floor) && deq(t->decay, e->decay), "aa/athfloor/decay %g %g | %g %g", t->ath_floor, e->ath_floor, t->decay, e->decay);
  CHK(deq(t->ma_max_i1, e->ma_max_i1) && deq(t->ma_max_i2, e->ma_max_i2) && deq(t->ma_max_m, e->ma_max_m), "ma_max");
  for (int i = 0; i < 32; i++) CHK(feq(t->amp_filter[i], e->amp_filter[i].v), "amp_filter[%d] %g vs %g", i, t->amp_filter[i], e->amp_filter[i].v);
  for (int i = 0; i < 23; i++) CHK(t->sfb_l[i] == e->sfb_l[i], "sfb_l[%d]", i);
  for (int i = 0; i < 14; i++) CHK(t->sfb_s[i] == e->sfb_s[i], "sfb_s[%d]", i);
  for (int i = 0; i < 7; i++) CHK(t->psfb21[i] == e->psfb21[i] && t->psfb12[i] == e->psfb12[i], "psfb[%d]", i);
  for (int i = 0; i < 576; i++) CHK(t->bv_scf[i] == e->bv_scf[i], "bv_scf[%d] %d vs %d", i, t->bv_scf[i], e->bv_scf[i]);
  CHK(t->npart_l == e->npart_l && t->npart_s == e->npart_s, "npart %d %d vs %d %d", t->npart_l, t->npart_s, e->npart_l, e->npart_s);
  for (int i = 0; i < t->npart_l && i < e->npart_l; i++) {
    CHK(t->numlines_l[i] == e->numlines_l[i], "numlines_l[%d]", i);
    CHK(feq(t->rnumlines_l[i], e->rnumlines_l[i].v), "rnumlines_l[%d]", i);
    CHK(feq(t->ath_cb_l[i], e->ath_cb_l[i].v), "ath_cb_l[%d] %g vs %g", i, t->ath_cb_l[i], e->ath_cb_l[i].v);
    CHK(t->s3lo_l[i] == e->s3ind[i][0] && t->s3hi_l[i] == e->s3ind[i][1], "s3ind_l[%d] %d %d vs %d %d", i, t->s3lo_l[i], t->s3hi_l[i], e->s3ind[i][0], e->s3ind[i][1]);
  }
  for (int i = 0; i < t->npart_s && i < e->npart_s; i++) {
    CHK(t->numlines_s[i] == e->numlines_s[i], "numlines_s[%d]", i);
    CHK(feq(t->ath_cb_s[i], e->ath_cb_s[i].v), "ath_cb_s[%d]", i);
    CHK(t->s3lo_s[i] == e->s3ind_s[i][0] && t->s3hi_s[i] == e->s3ind_s[i][1], "s3ind_s[%d]", i);
  }
  /* spreading rows: the oracle packs rows back to back over the UNCLAMPED index range, the product likewise (s3off) */
  {
    int k = 0;
    for (int b = 0; b < e->npart_l; b++) {
      CHK(t->s3off_l[b] == k, "s3off_l[%d] %d vs %d", b, t->s3off_l[b], k);
      const int off = t->s3off_l[b];
      const int n = t->s3off_l[b + 1] - off;
      for (int j = 0; j < n && k + j < e->n_s3_ll; j++) CHK(feq(t->s3_ll[off + j], e->s3_ll[k + j].v), "s3_ll row %d col %d", b, j);
      k += n;
    }
    CHK(k == e->n_s3_ll, "s3_ll count %d vs %d", k, e->n_s3_ll);
    k = 0;
    for (int b = 0; b < e->npart_s; b++) {
      const int off = t->s3off_s[b], n = t->s3off_s[b + 1] - off;
      for (int j = 0; j < n && k + j < e->n_s3_ss; j++) CHK(feq(t->s3_ss[off + j], e->s3_ss[k + j].v), "s3_ss row %d col %d", b, j);
      k += n;
    }
    CHK(k == e->n_s3_ss, "s3_ss count %d vs %d", k, e->n_s3_ss);
  }
  for (int i = 0; i < 22; i++) {
    CHK(t->bo_l[i] == e->bo_l[i], "bo_l[%d] %d vs %d", i, t->bo_l[i], e->bo_l[i]);
    CHK(feq(t->bo_l_weight[i], e->bo_l_weight[i].v), "bo_l_weight[%d]", i);
    CHK(feq(t->ath_l[i], e->ath_l[i].v), "ath_l[%d] %g vs %g", i, t->ath_l[i], e->ath_l[i].v);
    CHK(feq(t->longfact[i], e->longfact[i].v), "longfact[%d]", i);
  }
  for (int i = 0; i < 13; i++) {
    CHK(t->bo_s[i] == e->bo_s[i], "bo_s[%d]", i);
    CHK(feq(t->bo_s_weight[i], e->bo_s_weight[i].v), "bo_s_weight[%d]", i);
    CHK(feq(t->ath_s[i], e->ath_s[i].v), "ath_s[%d]", i);
    CHK(feq(t->shortfact[i], e->shortfact[i].v), "shortfact[%d]", i);
  }
  for (int i = 0; i < 6; i++) CHK(feq(t->ath_psfb21[i], e->ath_psfb21[i].v) && feq(t->ath_psfb12[i], e->ath_psfb12[i].v), "ath_psfb[%d]", i);
  for (int i = 0; i < 512; i++) CHK(feq(t->eql_w[i], e->ath_eql_w[i].v), "eql_w[%d]", i);
  for (int i = 0; i < 1024; i++) CHK(feq(t->fft_window[i], e->fft_window[i].v), "fft_window[%d]", i);
  for (int i = 0; i < 128; i++) CHK(feq(t->fft_window_s[i], e->fft_window_s[i].v), "fft_window_s[%d]", i);
  /* 10^(mask_adjust * 0.1) with lamejs's Math.pow (js_math.h), CBRNewIterationLoop.js:64 */
  CHK(deq(t->masking_lower_long, js_pow(10.0, e->mask_adjust * 0.1)), "masking_lower_long %.17g vs %.17g", t->masking_lower_long, js_pow(10.0, e->mask_adjust * 0.1));
  CHK(deq(t->masking_lower_short, js_pow(10.0, e->mask_adjust_short * 0.1)), "masking_lower_short %.17g vs %.17g", t->masking_lower_short, js_pow(10.0, e->mask_adjust_short * 0.1));
  {
    /* the threshold table must reproduce 0 | (log10(r) * 16) of the ORACLE's log10 (js_math.h) on random ratios and around
     * every threshold */
    CHK(t->l16_ok == 1, "l16 thresholds not a clean step");
    unsigned long long st = 0x9E3779B97F4A7C15ull;
    for (int n = 0; n < 200000; n++) {
      st = st * 6364136223846793005ull + 1442695040888963407ull;
      const double r = 1.0 + (double)(st >> 11) * (1.0 / 9007199254740992.0) * 30.6;     /* [1, 31.6) */
      int i = 0;
      for (int k = 1; k <= 24; k++) i += r >= t->l16_thr[k] ? 1 : 0;
      CHK(i == (int)(js_log10(r) * 16.0), "l16 random r=%.17g", r);
    }
    for (int k = 1; k <= 24; k++) for (int d = -300; d <= 300; d++) {
      unsigned long long u; memcpy(&u, &t->l16_thr[k], 8); u += d; double r; memcpy(&r, &u, 8);
      int i = 0;
      for (int kk = 1; kk <= 24; kk++) i += r >= t->l16_thr[kk] ? 1 : 0;
      CHK(i == (int)(js_log10(r) * 16.0), "l16 near threshold %d", k);
    }
  }
  const int r = bad != before;
  if (r) printf("cfg ch=%d sr=%d kbps=%d: %d mismatches\n", ch, sr, kbps, bad - before);
  free(t); lj_destroy(e);
  return r;
}

int main() {
  static const int rates[9] = {8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000};
  static const int kb[19] = {8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 123, 128, 144, 160, 192, 224, 256, 320};
  int fails = 0, n = 0;
  for (int r = 0; r < 9; r++) for (int k = 0; k < 19; k++) for (int ch = 1; ch <= 2; ch++) { fails += check(ch, rates[r], kb[k]); n++; }
  printf("config_check: %d configurations, %d with mismatches\n", n, fails);
  printf("config_check: %d resampled configurations compared\n", resampled);
  return fails ? 1 : 0;
}
