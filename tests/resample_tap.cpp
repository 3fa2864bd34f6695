/* resample_tap.cpp -- records what the oracle's resampler (fill_buffer_resample, oracle/lj_init.cpp) writes.  Test
 * infrastructure only: tests/resample_tap.py links it with the oracle's sources, lj_init.cpp compiled with
 * -Dlj_psycho_anal_ns=tap_psycho_anal_ns, so that the frame encoder's first call into the psy model of every frame comes
 * here first.  The oracle's code and bytes are unchanged.
 *
 * Only fill_buffer_resample writes mfbuf while an encoder resamples, behind mf_size, and a frame consumes the first
 * framesize values before they are shifted out.  So the first framesize values of mfbuf at each frame, followed by
 * mfbuf[0 .. mf_size) once the caller is done, are every value it wrote, in stream order, after the 576 - 48 zeros a fresh
 * FIFO starts with. */
#include <vector>
#include "../oracle/lj_encoder.h"

static std::vector<float> g_rec[2];
static const LjEnc* g_enc = nullptr;

int tap_psycho_anal_ns(LjEnc* e, const F32* buf0, const F32* buf1, int bufPos, int gr_out, PsyRatio masking_ratio[2][2],
                       PsyRatio masking_MS_ratio[2][2], double* percep_entropy, double* percep_MS_entropy, F32* energy,
                       int* blocktype_d) {
  if (e == g_enc && gr_out == 0)
    for (int ch = 0; ch < e->channels_out; ch++)
      for (int i = 0; i < e->framesize; i++) g_rec[ch].push_back(e->mfbuf[ch][i].v);
  return lj_psycho_anal_ns(e, buf0, buf1, bufPos, gr_out, masking_ratio, masking_MS_ratio, percep_entropy, percep_MS_entropy,
                           energy, blocktype_d);
}

extern "C" {
/* start recording encoder e (one at a time) */
void tap_begin(const LjEnc* e) { g_enc = e; g_rec[0].clear(); g_rec[1].clear(); }
/* number of values recorded per channel once the values still in the FIFO are added (call when the caller is done) */
long long tap_end(const LjEnc* e) {
  for (int ch = 0; ch < e->channels_out; ch++)
    for (int i = 0; i < e->mf_size; i++) g_rec[ch].push_back(e->mfbuf[ch][i].v);
  g_enc = nullptr;
  return (long long)g_rec[0].size();
}
void tap_copy(int ch, float* out) { for (size_t i = 0; i < g_rec[ch].size(); i++) out[i] = g_rec[ch][i]; }
/* row `row` of the filter bank (33 taps; 0 past the filter's length), 0 if the encoder has not resampled yet */
int tap_filter(const LjEnc* e, int row, float* out) {
  if (!e->blackfilt) return 0;
  for (int i = 0; i < 33; i++) out[i] = e->blackfilt[row][i].v;
  return 1;
}
int tap_bpc(const LjEnc* e) { return e->rs_bpc; }
double tap_scale(const LjEnc* e) { return e->scale; }
int tap_out_samplerate(const LjEnc* e) { return e->out_samplerate; }
}
