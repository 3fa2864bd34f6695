/* mp3_tag.cpp -- container / metadata step after the hot path (SURVEY.md 8(f3)), host side.
 *
 * - the Xing / Info / LAME tag frame of a CBR stream: reference src/js/VBRTag.js (InitVbrTag :472-538, addVbr :149-167,
 *   xingSeekTable :169-185, setLameTagFrameHeader :281-364, getLameTagFrame :829-923, putLameVBR :558-802), read with
 *   src/main/java/mp3/VBRTag.java where the JavaScript is not runnable as shipped (integer frame size, integer bag index,
 *   character codes of "Info" / "LAME3.98r"); the seek-table arithmetic is the JavaScript's (doubles);
 * - the WAV front-end: `WavHeader.readHeader` (src/js/index.js:154-193).
 * The frame is a few hundred bytes of bookkeeping per STREAM, built once at the end from four numbers: frame count, byte
 * count, encoder padding and the music CRC.  The CRC is the part that touches every output byte; it is taken on the
 * device (k_tag.cuh) and arrives here as a 16-bit value.
 */
#include <math.h>
#include <string.h>

#include "mp3_tag.h"

namespace {

inline void put_be(uint8_t* p, int nbytes, long long v) {
  for (int i = 0; i < nbytes; i++) p[i] = (uint8_t)(v >> (8 * (nbytes - 1 - i)));
}

/* CRC-16 of the tag's own bytes (same polynomial as the music CRC; a hundred-odd bytes, done in place) */
unsigned crc16_bytes(const uint8_t* p, int n) {
  unsigned c = 0;
  for (int i = 0; i < n; i++) {
    c ^= p[i];
    for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0xA001u : c >> 1;
  }
  return c;
}

}  // namespace

void Mp3SeekBag::reset() { sum = 0; seen = 0; want = 1; pos = 0; frames = 0; }

void Mp3SeekBag::add_frames(long long n, int kbps) {
  for (long long i = 0; i < n; i++) {
    frames++;
    sum += kbps;
    if (++seen < want) continue;
    if (pos < 400) { bag[pos++] = sum; seen = 0; }
    if (pos == 400) {                          /* keep every second entry, collect twice as many frames per entry from now on */
      for (int j = 0; j < 200; j++) bag[j] = bag[2 * j + 1];
      want *= 2;
      pos = 200;
    }
  }
}

void mp3_tag_header(const Mp3TagParams& p, int mode_ext, uint8_t* h4) {
  h4[0] = 0xFF;
  h4[1] = (uint8_t)(0xE0 | (p.mpeg25 ? 0x00 : 0x10) | (p.version ? 0x0A : 0x02) | 0x01);
  h4[2] = (uint8_t)((p.bitrate_index << 4) | (p.samplerate_index << 2));
  h4[3] = (uint8_t)(((p.mono ? 3 : 0) << 6) | ((mode_ext & 3) << 4) | 0x04);
}

int mp3_tag_placeholder(const Mp3TagParams& p, uint8_t* out) {
  if (!p.fits) return 0;
  memset(out, 0, (size_t)p.frame_bytes);
  mp3_tag_header(p, 2 /* gfc.mode_ext before the first frame: MPG_MD_MS_LR (Lame.js lame_init_params) */, out);
  return p.frame_bytes;
}

int mp3_radio_gain(double title_db) { return (int)floor(title_db * 10.0 + 0.5); }

int mp3_radio_gain_field(int radio_gain) {
  if (radio_gain > 0x1FE) radio_gain = 0x1FE;
  if (radio_gain < -0x1FE) radio_gain = -0x1FE;
  return radio_gain >= 0 ? (0x2000 | 0xC00 | radio_gain) : (0x2000 | 0xC00 | 0x200 | -radio_gain);
}

int mp3_tag_frame(const Mp3TagParams& p, const Mp3SeekBag& bag, long long music_bytes, unsigned music_crc, int encoder_padding, uint8_t* out,
                  int radio_gain_field) {
  if (!p.fits || bag.pos <= 0) return 0;
  memset(out, 0, (size_t)p.frame_bytes);
  mp3_tag_header(p, 0 /* MPG_MD_LR_LR: what every encoded frame leaves in gfc.mode_ext */, out);
  uint8_t* w = out + p.sideinfo_len;
  memcpy(w, "Info", 4);                                     /* VBR == vbr_off */
  put_be(w + 4, 4, 0x1 | 0x2 | 0x4 | 0x8);                   /* frames, bytes, TOC, quality */
  put_be(w + 8, 4, bag.frames);
  const long long stream_bytes = music_bytes + p.frame_bytes;
  put_be(w + 12, 4, stream_bytes);
  uint8_t* toc = w + 16;                                     /* toc[0] stays 0 */
  for (int i = 1; i < 100; i++) {
    const double j = (double)i / 100;
    int at = (int)floor(j * bag.pos);
    if (at > bag.pos - 1) at = bag.pos - 1;
    int seek = (int)(256. * (double)bag.bag[at] / (double)bag.sum);
    toc[i] = (uint8_t)(seek > 255 ? 255 : seek);
  }
  uint8_t* q = w + 116;                                      /* the LAME extension */
  put_be(q, 4, p.quality_byte);
  memcpy(q + 4, "LAME3.98r", 9);                             /* Version.js:56-59 */
  q[13] = 1;                                                 /* tag revision 0, method 1 = CBR */
  q[14] = (uint8_t)p.lowpass_byte;
  /* q[15..18] peak amplitude: zero (it needs the decoder); q[19..20] Radio Replay Gain when analysed (0 otherwise),
   * q[21..22] Audiophile Replay Gain: zero (lamejs never sets it) */
  put_be(q + 19, 2, radio_gain_field);
  q[23] = (uint8_t)p.flags_byte;
  q[24] = (uint8_t)(p.kbps >= 255 ? 255 : p.kbps);
  const int delay = 576;                                     /* Encoder.ENCDELAY */
  q[25] = (uint8_t)(delay >> 4);
  q[26] = (uint8_t)((delay << 4) + (encoder_padding >> 8));
  q[27] = (uint8_t)encoder_padding;
  q[28] = (uint8_t)p.misc_byte;
  q[29] = 0;
  put_be(q + 30, 2, p.kbps);                                 /* gfp.preset = the bitrate (Presets.js:415) */
  put_be(q + 32, 4, stream_bytes);
  put_be(q + 36, 2, music_crc & 0xffffu);
  put_be(q + 38, 2, crc16_bytes(out, (int)(q + 38 - out)));
  return p.frame_bytes;
}

namespace {
bool rd(const uint8_t* d, long long n, long long pos, int nbytes, bool little, unsigned long long* v) {
  if (pos < 0 || pos + nbytes > n) return false;
  unsigned long long x = 0;
  for (int i = 0; i < nbytes; i++) x |= (unsigned long long)d[pos + i] << (8 * (little ? i : nbytes - 1 - i));
  *v = x;
  return true;
}
}  // namespace

int mp3_wav_read_header(const uint8_t* d, long long n, long long* data_offset, long long* data_len, int* channels, unsigned* sample_rate) {
  enum : unsigned long long { RIFF = 0x52494646ull, WAVE = 0x57415645ull, FMT = 0x666d7420ull, DATA = 0x64617461ull };
  unsigned long long id, v, fmt_len, len = 0;
  *data_offset = *data_len = 0; *channels = *sample_rate = 0;
  if (!rd(d, n, 0, 4, false, &id)) return -2;
  if (id != RIFF) return 0;
  if (!rd(d, n, 4, 4, true, &v)) return -2;                  /* RIFF length: read, not used */
  if (!rd(d, n, 8, 4, false, &v)) return -2;
  if (v != WAVE) return 0;
  if (!rd(d, n, 12, 4, false, &v)) return -2;
  if (v != FMT) return 0;                                    /* "fmt " must be the first chunk */
  if (!rd(d, n, 16, 4, true, &fmt_len)) return -2;
  if (fmt_len != 16 && fmt_len != 18) return -1;             /* 'extended fmt chunk not implemented' */
  if (!rd(d, n, 22, 2, true, &v)) return -2;
  *channels = (int)v;
  if (!rd(d, n, 24, 4, true, &v)) return -2;
  *sample_rate = (unsigned)v;
  long long pos = 20 + (long long)fmt_len;
  for (;;) {                                                 /* skip chunks until "data" */
    if (!rd(d, n, pos, 4, false, &id) || !rd(d, n, pos + 4, 4, true, &len)) return -2;
    if (id == DATA) break;
    pos += (long long)len + 8;
  }
  *data_len = (long long)len;
  *data_offset = pos + 8;
  return 1;
}

/* getVbrTag (VBRTag.js:375-470): what a decoder reads back from the first frame of a stream.  Returns 1 and fills `t`,
 * 0 when the frame carries no "Xing" / "Info" magic (the reference returns null), -2 when the buffer ends first. */
int mp3_tag_parse(const uint8_t* buf, long long n, Mp3VbrTagData* t) {
  static const int bitrates[2][16] = {{0, 8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160, -1},
                                      {0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, -1}};
  static const int rates[3][4] = {{22050, 24000, 16000, -1}, {44100, 48000, 32000, -1}, {11025, 12000, 8000, -1}};
  memset(t, 0, sizeof *t);
  if (n < 4) return -2;
  const int id = (buf[1] >> 3) & 1, sr_index = (buf[2] >> 2) & 3, mode = (buf[3] >> 6) & 3;
  const int kbps = bitrates[id][(buf[2] >> 4) & 0xf];
  t->samprate = ((buf[1] >> 4) == 0xE) ? rates[2][sr_index] : rates[id][sr_index];      /* 0xFFE sync: MPEG-2.5 */
  long long p = id ? (mode != 3 ? 32 + 4 : 17 + 4) : (mode != 3 ? 17 + 4 : 9 + 4);     /* behind the side info */
  if (p + 8 > n) return -2;
  if (memcmp(buf + p, "Xing", 4) != 0 && memcmp(buf + p, "Info", 4) != 0) return 0;
  p += 4;
  t->h_id = id;
  auto be32 = [&](long long at) { return (int)(((unsigned)buf[at] << 24) | ((unsigned)buf[at + 1] << 16) | ((unsigned)buf[at + 2] << 8) | buf[at + 3]); };
  const int flags = t->flags = be32(p);
  p += 4;
  if (flags & 1) { if (p + 4 > n) return -2; t->frames = be32(p); p += 4; }
  if (flags & 2) { if (p + 4 > n) return -2; t->bytes = be32(p); p += 4; }
  if (flags & 4) { if (p + 100 > n) return -2; memcpy(t->toc, buf + p, 100); p += 100; }
  t->vbr_scale = -1;
  if (flags & 8) { if (p + 4 > n) return -2; t->vbr_scale = be32(p); p += 4; }
  t->headersize = t->samprate > 0 ? ((id + 1) * 72000 * kbps) / t->samprate : 0;
  p += 21;
  if (p + 3 > n) return -2;
  int delay = (buf[p] << 4) + (buf[p + 1] >> 4);
  int padding = ((buf[p + 1] & 0x0F) << 8) + buf[p + 2];
  if (delay < 0 || delay > 3000) delay = -1;        /* an old Xing header without the LAME extension */
  if (padding < 0 || padding > 3000) padding = -1;
  t->enc_delay = delay; t->enc_padding = padding;
  return 1;
}

/* skipId3v2 (VBRTag.js:804-827): size of an ID3v2 tag at the head of a stream, 0 if there is none.  The port's test is
 * inverted (`if (!...startsWith("ID3"))`, VBRTag.js:811 = VBRTag.java:833: it would read a "size" out of audio bytes when
 * there is NO tag); LAME's meaning is restated. */
long long mp3_skip_id3v2(const uint8_t* s, long long n) {
  if (n < 10 || memcmp(s, "ID3", 3) != 0) return 0;
  return (((long long)(s[6] & 0x7f) << 21) | ((s[7] & 0x7f) << 14) | ((s[8] & 0x7f) << 7) | (s[9] & 0x7f)) + 10;
}
