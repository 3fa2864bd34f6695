/* mp3_tag.h -- host-side pieces of the container / metadata row (SURVEY.md 8(f3)); see mp3_tag.cpp. */
#ifndef MP3B200_TAG_H
#define MP3B200_TAG_H
#include <stdint.h>
#include "mp3_config.h"
#include "k_tag.cuh"                    /* mp3_radio_gain, mp3_radio_gain_field, mp3_tag_patch: shared with the device */

/* VBRSeekInfo (reference src/js/VBRSeekInfo.js): running bitrate sums sampled every `want` frames, at most 400 of them */
struct Mp3SeekBag {
  long long sum, frames;
  int seen, want, pos;
  long long bag[400];
  void reset();
  void add_frames(long long n, int kbps);       /* addVbrFrame n times (Encoder.js:640-641) */
};

void mp3_tag_header(const Mp3TagParams& p, int mode_ext, uint8_t* h4);
/* InitVbrTag: the all-zero frame that reserves the tag's place at the head of the stream; 0 if the tag does not fit */
int mp3_tag_placeholder(const Mp3TagParams& p, uint8_t* out);
/* getLameTagFrame: p.frame_bytes bytes, or 0 (tag off / no frame counted yet).  The data-dependent bytes are written last,
 * by mp3_tag_patch (k_tag.cuh). */
int mp3_tag_frame(const Mp3TagParams& p, const Mp3SeekBag& bag, long long music_bytes, unsigned music_crc, int encoder_padding, uint8_t* out,
                  int radio_gain_field = 0);
/* WavHeader.readHeader: 1 ok, 0 `return undefined`, -1 throws 'extended fmt chunk not implemented', -2 DataView RangeError */
int mp3_wav_read_header(const uint8_t* d, long long n, long long* data_offset, long long* data_len, int* channels, unsigned* sample_rate);
/* VBRTagData (reference src/main/java/mp3/VBRTagData.java; `new VBRTagData()` in VBRTag.js:376) */
struct Mp3VbrTagData { int h_id, samprate, flags, frames, bytes, vbr_scale, headersize, enc_delay, enc_padding; unsigned char toc[100]; };
int mp3_tag_parse(const uint8_t* buf, long long n, Mp3VbrTagData* t);
long long mp3_skip_id3v2(const uint8_t* stream, long long n);
#endif
