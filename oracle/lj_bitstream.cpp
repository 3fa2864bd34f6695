/* lj_bitstream.cpp -- frame formatting of the oracle.  TEST INFRASTRUCTURE.
 * Follows src/js/BitStream.js: putbits2 :110-138, drain_into_ancillary :175-213, writeheader :218-229,
 * encodeSideInfo2 :259-426 (MPEG-1 branch), huffman_coder_count1 :428-482, Huffmancode :487-552,
 * Short/LongHuffmancodebits :558-598, writeMainData :600-689, format_bitstream :836-901,
 * copy_buffer :912-1010.  With the reservoir disabled main_data_begin is 0, so every header is
 * emitted exactly at its frame start; the 256-entry header ring of the reference degenerates to
 * "one pending header", which is what is kept here.
 */
#include "lj_encoder.h"
#include "lj_tables.h"

extern const int lj_slen1_tab[16];
extern const int lj_slen2_tab[16];

static void putheader_bits(LjEnc* e) {
  memcpy(e->bs_buf + e->bs_byteidx, e->header[e->w_ptr].buf, e->sideinfo_len);
  e->bs_byteidx += e->sideinfo_len;
  e->bs_totbit += e->sideinfo_len * 8;
  e->w_ptr = (e->w_ptr + 1) & 255;
}

static void putbits2(LjEnc* e, int val, int j) {
  while (j > 0) {
    int k;
    if (e->bs_bitidx == 0) {
      e->bs_bitidx = 8;
      e->bs_byteidx++;
      if (e->header[e->w_ptr].write_timing == e->bs_totbit) putheader_bits(e);
      e->bs_buf[e->bs_byteidx] = 0;
    }
    k = j < e->bs_bitidx ? j : e->bs_bitidx;
    j -= k;
    e->bs_bitidx -= k;
    e->bs_buf[e->bs_byteidx] |= (uint8_t)((val >> j) << e->bs_bitidx);
    e->bs_totbit += k;
  }
}

static void drain_into_ancillary(LjEnc* e, double remainingBits) {
  if (remainingBits >= 8) { putbits2(e, 0x4c, 8); remainingBits -= 8; }
  if (remainingBits >= 8) { putbits2(e, 0x41, 8); remainingBits -= 8; }
  if (remainingBits >= 8) { putbits2(e, 0x4d, 8); remainingBits -= 8; }
  if (remainingBits >= 8) { putbits2(e, 0x45, 8); remainingBits -= 8; }
  if (remainingBits >= 32) {
    /* version.charAt(i) is a STRING operand of `>>`: "3.98.4" -> 3,NaN(0),9,8,NaN(0),4 */
    static const int version_vals[6] = {3, 0, 9, 8, 0, 4};
    for (int i = 0; i < 6 && remainingBits >= 8; ++i) {
      remainingBits -= 8;
      putbits2(e, version_vals[i], 8);
    }
  }
  for (; remainingBits >= 1; remainingBits -= 1) {
    putbits2(e, e->ancillary_flag, 1);
    e->ancillary_flag ^= (!e->disable_reservoir ? 1 : 0);
  }
}

static void writeheader(LjEnc* e, int val, int j) {
  int ptr = e->header[e->h_ptr].ptr;
  while (j > 0) {
    int k = j < 8 - (ptr & 7) ? j : 8 - (ptr & 7);
    j -= k;
    e->header[e->h_ptr].buf[ptr >> 3] |= (uint8_t)(((val >> j)) << (8 - (ptr & 7) - k));
    ptr += k;
  }
  e->header[e->h_ptr].ptr = ptr;
}

static void encodeSideInfo2(LjEnc* e, int bitsPerFrame) {
  e->header[e->h_ptr].ptr = 0;
  memset(e->header[e->h_ptr].buf, 0, e->sideinfo_len);
  writeheader(e, e->out_samplerate < 16000 ? 0xffe : 0xfff, 12);   /* MPEG-2.5 sync word */
  writeheader(e, e->version, 1);
  writeheader(e, 4 - 3, 2);
  writeheader(e, 1, 1);                        /* !error_protection */
  writeheader(e, e->bitrate_index, 4);
  writeheader(e, e->samplerate_index, 2);
  writeheader(e, e->padding, 1);
  writeheader(e, 0, 1);                        /* extension */
  writeheader(e, e->mode_mono ? 3 : (e->mode_joint ? 1 : 0), 2);     /* MPEGMode ordinal: STEREO 0, JOINT_STEREO 1, MONO 3 */
  writeheader(e, e->mode_ext, 2);
  writeheader(e, 0, 1);                        /* copyright */
  writeheader(e, 1, 1);                        /* original */
  writeheader(e, 0, 2);                        /* emphasis */
  if (e->version == 1) {
  writeheader(e, js_toint32(e->main_data_begin), 9);        /* `val >> j` on a JS number: ToInt32 */
  if (e->channels_out == 2) writeheader(e, 0, 3);
  else writeheader(e, 0, 5);
  for (int ch = 0; ch < e->channels_out; ch++)
    for (int band = 0; band < 4; band++) writeheader(e, e->scfsi[ch][band], 1);
  for (int gr = 0; gr < 2; gr++) {
    for (int ch = 0; ch < e->channels_out; ch++) {
      GrInfo* gi = &e->tt[gr][ch];
      writeheader(e, gi->part2_3_length + gi->part2_length, 12);
      writeheader(e, gi->big_values / 2, 9);
      writeheader(e, gi->global_gain, 8);
      writeheader(e, gi->scalefac_compress, 4);
      if (gi->block_type != NORM_TYPE) {
        writeheader(e, 1, 1);
        writeheader(e, gi->block_type, 2);
        writeheader(e, gi->mixed_block_flag, 1);
        if (gi->table_select[0] == 14) gi->table_select[0] = 16;
        writeheader(e, gi->table_select[0], 5);
        if (gi->table_select[1] == 14) gi->table_select[1] = 16;
        writeheader(e, gi->table_select[1], 5);
        writeheader(e, gi->subblock_gain[0], 3);
        writeheader(e, gi->subblock_gain[1], 3);
        writeheader(e, gi->subblock_gain[2], 3);
      } else {
        writeheader(e, 0, 1);
        if (gi->table_select[0] == 14) gi->table_select[0] = 16;
        writeheader(e, gi->table_select[0], 5);
        if (gi->table_select[1] == 14) gi->table_select[1] = 16;
        writeheader(e, gi->table_select[1], 5);
        if (gi->table_select[2] == 14) gi->table_select[2] = 16;
        writeheader(e, gi->table_select[2], 5);
        writeheader(e, gi->region0_count, 4);
        writeheader(e, gi->region1_count, 3);
      }
      writeheader(e, gi->preflag, 1);
      writeheader(e, gi->scalefac_scale, 1);
      writeheader(e, gi->count1table_select, 1);
    }
  }
  } else {
    /* MPEG-2 / 2.5 (BitStream.js:352-404): one granule, 9-bit scalefac_compress, no preflag bit, no scfsi */
    writeheader(e, js_toint32(e->main_data_begin), 8);
    writeheader(e, 0, e->channels_out);          /* private_bits */
    for (int ch = 0; ch < e->channels_out; ch++) {
      GrInfo* gi = &e->tt[0][ch];
      writeheader(e, gi->part2_3_length + gi->part2_length, 12);
      writeheader(e, gi->big_values / 2, 9);
      writeheader(e, gi->global_gain, 8);
      writeheader(e, gi->scalefac_compress, 9);
      if (gi->block_type != NORM_TYPE) {
        writeheader(e, 1, 1);
        writeheader(e, gi->block_type, 2);
        writeheader(e, gi->mixed_block_flag, 1);
        if (gi->table_select[0] == 14) gi->table_select[0] = 16;
        writeheader(e, gi->table_select[0], 5);
        if (gi->table_select[1] == 14) gi->table_select[1] = 16;
        writeheader(e, gi->table_select[1], 5);
        writeheader(e, gi->subblock_gain[0], 3);
        writeheader(e, gi->subblock_gain[1], 3);
        writeheader(e, gi->subblock_gain[2], 3);
      } else {
        writeheader(e, 0, 1);
        if (gi->table_select[0] == 14) gi->table_select[0] = 16;
        writeheader(e, gi->table_select[0], 5);
        if (gi->table_select[1] == 14) gi->table_select[1] = 16;
        writeheader(e, gi->table_select[1], 5);
        if (gi->table_select[2] == 14) gi->table_select[2] = 16;
        writeheader(e, gi->table_select[2], 5);
        writeheader(e, gi->region0_count, 4);
        writeheader(e, gi->region1_count, 3);
      }
      writeheader(e, gi->scalefac_scale, 1);
      writeheader(e, gi->count1table_select, 1);
    }
  }
  {
    int old = e->h_ptr;
    e->h_ptr = (old + 1) & 255;
    e->header[e->h_ptr].write_timing = e->header[old].write_timing + bitsPerFrame;
  }
}

static int huffman_coder_count1(LjEnc* e, const GrInfo* gi) {
  const int t = gi->count1table_select + 32;
  int bits = 0;
  int ix = gi->big_values;
  int xr = gi->big_values;
  for (int i = (gi->count1 - gi->big_values) / 4; i > 0; --i) {
    int huffbits = 0;
    int p = 0, v;
    v = gi->l3_enc[ix + 0];
    if (v != 0) { p += 8; if (gi->xr[xr + 0] < 0) huffbits++; }
    v = gi->l3_enc[ix + 1];
    if (v != 0) { p += 4; huffbits *= 2; if (gi->xr[xr + 1] < 0) huffbits++; }
    v = gi->l3_enc[ix + 2];
    if (v != 0) { p += 2; huffbits *= 2; if (gi->xr[xr + 2] < 0) huffbits++; }
    v = gi->l3_enc[ix + 3];
    if (v != 0) { p++; huffbits *= 2; if (gi->xr[xr + 3] < 0) huffbits++; }
    ix += 4;
    xr += 4;
    putbits2(e, huffbits + LJ_HUFF_CODE[LJ_HUFF_OFF[t] + p], LJ_HUFF_LEN[LJ_HUFF_OFF[t] + p]);
    bits += LJ_HUFF_LEN[LJ_HUFF_OFF[t] + p];
  }
  return bits;
}

static int Huffmancode(LjEnc* e, int tableindex, int start, int end, const GrInfo* gi) {
  int bits = 0;
  if (0 == tableindex) return bits;
  const int hxlen = LJ_HUFF_XLEN[tableindex];
  const int off = LJ_HUFF_OFF[tableindex];
  for (int i = start; i < end; i += 2) {
    int cbits = 0;
    int xbits = 0;
    int linbits = hxlen;
    int xlen = hxlen;
    int ext = 0;
    int x1 = gi->l3_enc[i];
    int x2 = gi->l3_enc[i + 1];
    if (x1 != 0) { if (gi->xr[i] < 0) ext++; cbits--; }
    if (tableindex > 15) {
      if (x1 > 14) { int linbits_x1 = x1 - 15; ext |= linbits_x1 << 1; xbits = linbits; x1 = 15; }
      if (x2 > 14) { int linbits_x2 = x2 - 15; ext <<= linbits; ext |= linbits_x2; xbits += linbits; x2 = 15; }
      xlen = 16;
    }
    if (x2 != 0) { ext <<= 1; if (gi->xr[i + 1] < 0) ext++; cbits--; }
    x1 = x1 * xlen + x2;
    xbits -= cbits;
    cbits += LJ_HUFF_LEN[off + x1];
    putbits2(e, LJ_HUFF_CODE[off + x1], cbits);
    putbits2(e, ext, xbits);
    bits += cbits + xbits;
  }
  return bits;
}

static int ShortHuffmancodebits(LjEnc* e, const GrInfo* gi) {
  int region1Start = 3 * e->sfb_s[3];
  if (region1Start > gi->big_values) region1Start = gi->big_values;
  int bits = Huffmancode(e, gi->table_select[0], 0, region1Start, gi);
  bits += Huffmancode(e, gi->table_select[1], region1Start, gi->big_values, gi);
  return bits;
}

static int LongHuffmancodebits(LjEnc* e, const GrInfo* gi) {
  int bigvalues = gi->big_values, bits;
  int region1Start, region2Start;
  int i = gi->region0_count + 1;
  region1Start = e->sfb_l[i];
  i += gi->region1_count + 1;
  region2Start = e->sfb_l[i];
  if (region1Start > bigvalues) region1Start = bigvalues;
  if (region2Start > bigvalues) region2Start = bigvalues;
  bits = Huffmancode(e, gi->table_select[0], 0, region1Start, gi);
  bits += Huffmancode(e, gi->table_select[1], region1Start, region2Start, gi);
  bits += Huffmancode(e, gi->table_select[2], region2Start, bigvalues, gi);
  return bits;
}

static int writeMainData(LjEnc* e) {
  int tot_bits = 0;
  if (e->version != 1) {   /* MPEG-2 / 2.5 (BitStream.js:641-687) */
    for (int ch = 0; ch < e->channels_out; ch++) {
      const GrInfo* gi = &e->tt[0][ch];
      int data_bits = 0, scale_bits = 0, sfb = 0;
      if (gi->block_type == SHORT_TYPE) {
        for (int part = 0; part < 4; part++) {
          const int sfbs = gi->sfb_partition_table[part] / 3, slen = gi->slen[part];
          for (int i = 0; i < sfbs; i++, sfb++) {
            putbits2(e, gi->scalefac[sfb * 3 + 0] > 0 ? gi->scalefac[sfb * 3 + 0] : 0, slen);
            putbits2(e, gi->scalefac[sfb * 3 + 1] > 0 ? gi->scalefac[sfb * 3 + 1] : 0, slen);
            putbits2(e, gi->scalefac[sfb * 3 + 2] > 0 ? gi->scalefac[sfb * 3 + 2] : 0, slen);
            scale_bits += 3 * slen;
          }
        }
        data_bits += ShortHuffmancodebits(e, gi);
      } else {
        for (int part = 0; part < 4; part++) {
          const int sfbs = gi->sfb_partition_table[part], slen = gi->slen[part];
          for (int i = 0; i < sfbs; i++, sfb++) {
            putbits2(e, gi->scalefac[sfb] > 0 ? gi->scalefac[sfb] : 0, slen);
            scale_bits += slen;
          }
        }
        data_bits += LongHuffmancodebits(e, gi);
      }
      data_bits += huffman_coder_count1(e, gi);
      tot_bits += scale_bits + data_bits;
    }
    return tot_bits;
  }
  for (int gr = 0; gr < 2; gr++) {
    for (int ch = 0; ch < e->channels_out; ch++) {
      const GrInfo* gi = &e->tt[gr][ch];
      int slen1 = lj_slen1_tab[gi->scalefac_compress];
      int slen2 = lj_slen2_tab[gi->scalefac_compress];
      int data_bits = 0;
      int sfb;
      for (sfb = 0; sfb < gi->sfbdivide; sfb++) {
        if (gi->scalefac[sfb] == -1) continue;
        putbits2(e, gi->scalefac[sfb], slen1);
        data_bits += slen1;
      }
      for (; sfb < gi->sfbmax; sfb++) {
        if (gi->scalefac[sfb] == -1) continue;
        putbits2(e, gi->scalefac[sfb], slen2);
        data_bits += slen2;
      }
      if (gi->block_type == SHORT_TYPE) data_bits += ShortHuffmancodebits(e, gi);
      else data_bits += LongHuffmancodebits(e, gi);
      data_bits += huffman_coder_count1(e, gi);
      tot_bits += data_bits;
    }
  }
  return tot_bits;
}

/* BitStream.js:708-755 */
static double compute_flushbits(LjEnc* e) {
  int first_ptr = e->w_ptr, last_ptr = e->h_ptr - 1;
  if (last_ptr == -1) last_ptr = 255;
  double flushbits = e->header[last_ptr].write_timing - e->bs_totbit;
  if (flushbits >= 0) {
    int remaining_headers = 1 + last_ptr - first_ptr;
    if (last_ptr < first_ptr) remaining_headers = 1 + last_ptr - first_ptr + 256;
    flushbits -= remaining_headers * 8 * e->sideinfo_len;
  }
  flushbits += lj_getframebits(e);
  return flushbits;
}

/* BitStream.js:757-776 (ReplayGain / peak parts are off) */
void lj_flush_bitstream(LjEnc* e) {
  double flushbits = compute_flushbits(e);
  if (flushbits < 0) return;
  drain_into_ancillary(e, flushbits);
  e->ResvSize = 0;
  e->main_data_begin = 0;
}

void lj_format_bitstream(LjEnc* e) {
  int bitsPerFrame = lj_getframebits(e);
  drain_into_ancillary(e, e->resvDrain_pre);
  encodeSideInfo2(e, bitsPerFrame);
  double bits = 8 * e->sideinfo_len;
  bits += writeMainData(e);
  drain_into_ancillary(e, e->resvDrain_post);
  bits += e->resvDrain_post;
  e->main_data_begin += (bitsPerFrame - bits) / 8;
  /* BitStream.js:851-884: consistency checks.  Both report through System.err, which lamejs's common.js does not define:
   * a failing check throws a TypeError out of lame_encode_buffer / lame_encode_flush.  That happens when a frame's bits
   * do not fit its slot (loud Float32 input), and the encoder is left unusable.  Java's LAME prints and re-bases ResvSize;
   * the integer-quotient reservoir switch (not lamejs either) keeps that. */
  if (e->java_int_div) {
    if ((e->main_data_begin * 8) != e->ResvSize) e->ResvSize = e->main_data_begin * 8;
  } else if (compute_flushbits(e) != e->ResvSize || (e->main_data_begin * 8) != e->ResvSize) {
    e->bs_fatal = 1;
    return;
  }
  if (e->bs_totbit > 1000000000) {
    for (int i = 0; i < 256; ++i) e->header[i].write_timing -= e->bs_totbit;
    e->bs_totbit = 0;
  }
}

int lj_copy_buffer(LjEnc* e, uint8_t* out, int cap, int mp3data) {
  int minimum = e->bs_byteidx + 1;
  if (minimum <= 0) return 0;
  if (cap != 0 && minimum > cap) return -1;
  memcpy(out, e->bs_buf, minimum);
  e->bs_byteidx = -1;
  e->bs_bitidx = 0;
  if (mp3data != 0) {              /* BitStream.js:924-935: music CRC and byte count of real frame data */
    lj_update_music_crc(e, out, minimum);
    if (minimum > 0) e->nBytesWritten += minimum;
  }
  return minimum;
}
