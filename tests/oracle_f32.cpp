/* oracle_f32.cpp -- the oracle's encodeBuffer with Float32 input (lamejs's lame_encode_buffer given a Float32Array or a plain
 * Array: each value is stored into gfc.in_buffer_0/1, Float32Arrays, Lame.js:1500-1510).  Test infrastructure only:
 * tests/oracle_f32.py compiles this file, which includes the unchanged oracle/lj_init.cpp so that its file-local
 * encode_buffer_sample is reachable, with the other oracle sources into a temporary library.  lj_encode (Int16) and every
 * other entry point of the oracle are in that library unchanged, so one encoder can take both kinds of calls. */
#include "../oracle/lj_init.cpp"

extern "C" {
/* lj_encode with the store `in_buffer[i] = left[i]` of Float32 values (the caller's values rounded to Float32 once) */
int lj_encode_f32(LjEnc* e, const float* left, const float* right, int n, uint8_t* out, int cap) {
  if (!e) return -3;
  if (e->bs_fatal) return LJ_ERR_BITSTREAM;
  if (n == 0) return 0;
  if (e->channels_out == 1 || e->num_channels == 1) right = left;
  const double nsamples = (double)n;
  if (e->inb[0] == NULL || e->inb_nsamples < nsamples) {      /* update_inbuffer_size, as encode_buffer does it */
    free(e->inb[0]); free(e->inb[1]);
    e->inb[0] = (F32*)calloc(n, sizeof(F32));
    e->inb[1] = (F32*)calloc(n, sizeof(F32));
    e->inb_len = n; e->inb_nsamples = nsamples;
  }
  for (int i = 0; i < n; i++) {
    e->inb[0][i] = (double)left[i];
    if (e->num_channels > 1) e->inb[1][i] = (double)right[i];
  }
  return encode_buffer_sample(e, e->inb[0], e->inb[1], e->inb_len, nsamples, out, cap);
}
}
