/* k_tag.cuh -- the music CRC of the Xing / LAME tag on the GPU (SURVEY.md 8(f3)), the placement of the tag frames of
 * device-resident streams (k_tag_scatter), and the frames an encode session finishes on the device (k_tag_finish).
 *
 * lamejs keeps gfc.nMusicCRC by pushing every byte copy_buffer hands out through a table-driven CRC-16 (polynomial
 * x^16 + x^15 + x^2 + 1, reflected, start 0; reference src/js/VBRTag.js:547-556, BitStream.js:924-928): one dependent table
 * look-up per byte, 4 MB per 10 000 frames.  The bytes are in HBM when the packer has run, so the CRC is taken there,
 * in parallel, before they leave the device:
 *
 *   a CRC with start value 0 is linear over GF(2):  crc(A || B) = shift(crc(A), |B|)  xor  crc(B),
 *   where shift(c, n) advances the register through n zero bytes, i.e. multiplies by x^(8n) modulo the polynomial.
 *
 * The byte range of a stream is cut into 512-byte pieces, one warp per piece, 16 bytes per lane.  A lane runs the table
 * CRC over its bytes, shifts the result by the bytes that follow it inside the piece, the warp xors the 32 values, lane 0
 * shifts the piece by the bytes that follow it in the stream and xors it into the stream's accumulator (xor commutes:
 * the atomics need no order).  shift() is a product of the 16 x 16 bit matrices Z^(2^k) (Z = one zero byte), picked by
 * the set bits of n; the matrices and the byte table are built on the host (crc_host_tables) and staged in shared memory.
 *
 * Everything that decides a bit is in the __host__ __device__ functions below; tests/crc_emul.cpp compiles this header with
 * g++ and replays the kernel's lane / piece decomposition on the CPU against the serial definition.
 * Algorithmic traffic: 1 byte read per output byte (L2-resident right after the packer); 4 bytes written per stream.
 */
#ifndef MP3B200_K_TAG_CUH
#define MP3B200_K_TAG_CUH
#include <math.h>
#include <stdint.h>
#include "mp3_config.h"

#ifndef __CUDACC__
#define MP3_HD inline
#else
#define MP3_HD __host__ __device__ __forceinline__
#endif

enum { CRC_POW_LEVELS = 40, CRC_LANE_BYTES = 16, CRC_PIECE_BYTES = 32 * CRC_LANE_BYTES, CRC_WARPS = 8 };

struct CrcTables {
  unsigned short byte_table[256];                 /* crc16Lookup (VBRTag.js:113-145) */
  unsigned short pow[CRC_POW_LEVELS][16];         /* pow[k][b] = image of bit b under Z^(2^k), Z = "one zero byte" */
};

/* one byte through the register (crcUpdateLookup, VBRTag.js:547-551) */
MP3_HD unsigned crc_step(unsigned crc, unsigned byte, const unsigned short* byte_table) {
  return (crc >> 8) ^ byte_table[(crc ^ byte) & 0xffu];
}

/* register advanced through `nbytes` zero bytes */
MP3_HD unsigned crc_shift(unsigned crc, unsigned long long nbytes, const unsigned short (*pow)[16]) {
  for (int k = 0; nbytes != 0 && k < CRC_POW_LEVELS; k++, nbytes >>= 1) {
    if (!(nbytes & 1ull)) continue;
    unsigned r = 0;
    for (int b = 0; b < 16; b++)
      if ((crc >> b) & 1u) r ^= pow[k][b];
    crc = r;
  }
  return crc;
}

/* what lane `lane` of the warp working on piece `piece` of a `len`-byte range does: its bytes [lo, lo + n), the bytes
 * that follow them inside the piece, and (for lane 0's final step) the bytes that follow the piece in the range */
struct CrcLanePlan { long long lo; int n; int after_in_piece; long long after_piece; };
MP3_HD CrcLanePlan crc_plan(long long len, long long piece, int lane) {
  CrcLanePlan p;
  const long long p_lo = piece * CRC_PIECE_BYTES;
  long long p_hi = p_lo + CRC_PIECE_BYTES;
  if (p_hi > len) p_hi = len;
  long long lo = p_lo + (long long)lane * CRC_LANE_BYTES, hi = lo + CRC_LANE_BYTES;
  if (lo > p_hi) lo = p_hi;
  if (hi > p_hi) hi = p_hi;
  p.lo = lo; p.n = (int)(hi - lo);
  p.after_in_piece = (int)(p_hi - hi);
  p.after_piece = len - p_hi;
  return p;
}

/* a lane's share: table CRC of its bytes, moved to the end of the piece */
MP3_HD unsigned crc_lane(const uint8_t* range, const CrcLanePlan& p, const unsigned short* byte_table, const unsigned short (*pow)[16]) {
  unsigned c = 0;
  for (int i = 0; i < p.n; i++) c = crc_step(c, range[p.lo + i], byte_table);
  return crc_shift(c, (unsigned long long)p.after_in_piece, pow);
}

/* combination rule of a streaming handle: the register after `nbytes` more bytes whose own CRC (start 0) is `crc_new` */
MP3_HD unsigned crc_append(unsigned crc_old, unsigned crc_new, unsigned long long nbytes, const unsigned short (*pow)[16]) {
  return crc_shift(crc_old, nbytes, pow) ^ crc_new;
}

/* host: the byte table from the polynomial, Z from the byte table, the powers by squaring */
inline void crc_host_tables(CrcTables* t) {
  for (int i = 0; i < 256; i++) {
    unsigned c = (unsigned)i;
    for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0xA001u : c >> 1;
    t->byte_table[i] = (unsigned short)c;
  }
  for (int b = 0; b < 16; b++) t->pow[0][b] = (unsigned short)crc_step(1u << b, 0, t->byte_table);
  for (int k = 1; k < CRC_POW_LEVELS; k++)
    for (int b = 0; b < 16; b++) {
      unsigned v = t->pow[k - 1][b], r = 0;
      for (int j = 0; j < 16; j++)
        if ((v >> j) & 1u) r ^= t->pow[k - 1][j];
      t->pow[k][b] = (unsigned short)r;
    }
}

/* ---- the bytes of a tag frame that depend on the encoded data (mp3_tag_frame, mp3_tag.cpp; k_tag_finish below) ----
 * Everything else in the frame follows from the configuration and the stream's length.  One definition for the host and
 * the device; tests/tag_patch_emul.cpp compiles it with g++. */

/* gfc.RadioGain = Math.floor(title gain * 10 + 0.5) | 0 (BitStream.js:785) */
MP3_HD int mp3_radio_gain(double title_db) { return (int)floor(title_db * 10.0 + 0.5); }

/* the tag's Radio Replay Gain field (VBRTag.js:640-661): name code 1, originator 3 (determined automatically), sign bit,
 * |RadioGain| clamped to 0x1FE */
MP3_HD int mp3_radio_gain_field(int radio_gain) {
  if (radio_gain > 0x1FE) radio_gain = 0x1FE;
  if (radio_gain < -0x1FE) radio_gain = -0x1FE;
  return radio_gain >= 0 ? (0x2000 | 0xC00 | radio_gain) : (0x2000 | 0xC00 | 0x200 | -radio_gain);
}

/* CRC-16 of the tag's own bytes (the music CRC's polynomial; under two hundred bytes, bit by bit) */
MP3_HD unsigned mp3_tag_crc16(const uint8_t* p, int n) {
  unsigned c = 0;
  for (int i = 0; i < n; i++) {
    c ^= p[i];
    for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0xA001u : c >> 1;
  }
  return c;
}

/* offset of the LAME extension in a tag frame, and the bytes of the frame up to and including its CRC */
MP3_HD int mp3_tag_lame_at(const Mp3TagParams& p) { return p.sideinfo_len + 116; }
MP3_HD int mp3_tag_head_bytes(const Mp3TagParams& p) { return mp3_tag_lame_at(p) + 40; }

/* Completes a frame whose other bytes are in place: the Radio Replay Gain field (0: nobody analysed), the music CRC, and
 * then the frame's own CRC over everything in front of it. */
MP3_HD void mp3_tag_patch(uint8_t* frame, const Mp3TagParams& p, unsigned music_crc, int radio_gain_field) {
  uint8_t* q = frame + mp3_tag_lame_at(p);
  q[19] = (uint8_t)(radio_gain_field >> 8); q[20] = (uint8_t)radio_gain_field;
  q[36] = (uint8_t)(music_crc >> 8); q[37] = (uint8_t)music_crc;
  const unsigned own = mp3_tag_crc16(frame, mp3_tag_lame_at(p) + 38);
  q[38] = (uint8_t)(own >> 8); q[39] = (uint8_t)own;
}

#ifdef __CUDACC__
/* grid (pieces of the longest range / CRC_WARPS, ranges); crc_out[r] must be zero before the launch.
 * off[r] / len[r]: byte range r inside `buf`. */
__global__ void __launch_bounds__(CRC_WARPS * 32)
k_music_crc(const uint8_t* __restrict__ buf, const long long* __restrict__ off, const long long* __restrict__ len, const CrcTables* __restrict__ tables,
            unsigned* __restrict__ crc_out) {
  __shared__ CrcTables s_t;
  {
    const unsigned* src = reinterpret_cast<const unsigned*>(tables);
    unsigned* dst = reinterpret_cast<unsigned*>(&s_t);
    for (int i = threadIdx.x; i < (int)(sizeof(CrcTables) / sizeof(unsigned)); i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const int r = blockIdx.y, lane = threadIdx.x & 31;
  const long long n = len[r];
  const long long piece = (long long)blockIdx.x * CRC_WARPS + (threadIdx.x >> 5);
  if (piece * CRC_PIECE_BYTES >= n) return;             /* whole warp */
  const CrcLanePlan p = crc_plan(n, piece, lane);
  unsigned c = crc_lane(buf + off[r], p, s_t.byte_table, s_t.pow);
  c ^= __shfl_xor_sync(0xffffffffu, c, 16);
  c ^= __shfl_xor_sync(0xffffffffu, c, 8);
  c ^= __shfl_xor_sync(0xffffffffu, c, 4);
  c ^= __shfl_xor_sync(0xffffffffu, c, 2);
  c ^= __shfl_xor_sync(0xffffffffu, c, 1);
  if (lane == 0) atomicXor(&crc_out[r], crc_shift(c, (unsigned long long)p.after_piece, s_t.pow));
}

/* The tag frames of a batch of device-resident streams, built on the host (mp3_tag_frame) and uploaded in one copy, put in
 * front of their streams: grid (frames), frame i is frame_bytes bytes at frames + i * frame_bytes and goes to out + dst[i].
 * One block per frame, so a batch of any size is one launch. */
enum { TAG_SCATTER_THREADS = 128 };
__global__ void __launch_bounds__(TAG_SCATTER_THREADS)
k_tag_scatter(const long long* __restrict__ dst, const uint8_t* __restrict__ frames, int frame_bytes, uint8_t* __restrict__ out) {
  const uint8_t* src = frames + (size_t)blockIdx.x * frame_bytes;
  uint8_t* d = out + dst[blockIdx.x];
  for (int i = threadIdx.x; i < frame_bytes; i += TAG_SCATTER_THREADS) d[i] = src[i];
}

/* The tag frames an encode session finishes without the host: grid (frames), one block per frame.  templates + i *
 * p.frame_bytes is mp3_tag_frame with music CRC 0 and gain field 0, built on the host before anything ran; it goes to
 * dst[i].at, completed by mp3_tag_patch with the music CRC k_music_crc left in crc[dst[i].stream] and, when the call analysed
 * (gain != NULL), the field of gain[dst[i].stream].  The patched head is staged in shared memory, so the frame's own CRC reads
 * no global memory. */
struct TagDest { uint8_t* at; long long stream; };
enum { TAG_FINISH_THREADS = 128, TAG_HEAD_MAX = 4 + 32 + 116 + 40 };      /* the longest side info: MPEG-1 stereo */
__global__ void __launch_bounds__(TAG_FINISH_THREADS)
k_tag_finish(const TagDest* __restrict__ dst, const uint8_t* __restrict__ templates, Mp3TagParams p, const unsigned* __restrict__ crc,
             const double* __restrict__ gain) {
  __shared__ uint8_t head[TAG_HEAD_MAX];
  const TagDest d = dst[blockIdx.x];
  const uint8_t* src = templates + (size_t)blockIdx.x * p.frame_bytes;
  const int nhead = mp3_tag_head_bytes(p);
  for (int i = threadIdx.x; i < nhead; i += TAG_FINISH_THREADS) head[i] = src[i];
  for (int i = nhead + threadIdx.x; i < p.frame_bytes; i += TAG_FINISH_THREADS) d.at[i] = src[i];
  __syncthreads();
  if (threadIdx.x == 0)
    mp3_tag_patch(head, p, crc[d.stream] & 0xffffu, gain ? mp3_radio_gain_field(mp3_radio_gain(gain[d.stream])) : 0);
  __syncthreads();
  for (int i = threadIdx.x; i < nhead; i += TAG_FINISH_THREADS) d.at[i] = head[i];
}
#endif

#endif
