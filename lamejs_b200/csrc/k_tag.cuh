/* k_tag.cuh -- the music CRC of the Xing / LAME tag on the GPU (SURVEY.md 8(f3)), and the placement of the tag frames of
 * device-resident streams (k_tag_scatter).
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
#include <stdint.h>

#ifndef __CUDACC__
#define MP3_HD
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
#endif

#endif
