/* k_quant.cuh -- K4/K5: bit allocation, noise-shaping loop, quantizer, Huffman bit counting, bit packing.
 *
 * Replaces lamejs CBRNewIterationLoop.iteration_loop (reference src/js/CBRNewIterationLoop.js:25-90) with
 * everything it calls -- Reservoir.js (bit budget), QuantizePVT.js (on_pe :421, calc_xmin :569, calc_noise :725),
 * Quantize.js (init_outer_loop :204, init_xrpow :105, bin_search_StepSize :322, outer_loop :871, balance_noise,
 * amp_scalefac_bands, inc_scalefac_scale, inc_subblock_gain, iteration_finish_one :1059), Takehiro.js
 * (quantize_xrpow :171, noquant_count_bits :521, choose_table :465, best_huffman_divide :727, best_scalefac_store
 * :809, scale_bitcount :980) -- and BitStream.format_bitstream (src/js/BitStream.js:836-901).
 *
 * Mapping: one CUDA block per frame, one warp per channel (a granule-channel is "gc").  All control decisions are
 * warp-uniform: scalars live in shared memory, lane 0 writes, __syncwarp publishes.  The 576 spectral lines are
 * spread 18 per lane; Huffman bit counts, maxima and region scans are warp reductions over table look-ups
 * (integer sums are order-free); floating-point sums whose order matters (calc_xmin energies, calc_noise) run one
 * scalefactor band per lane in the reference's line order.  gr1 needs the bits both channels spent in gr0
 * (Reservoir.ResvMaxBits), so the two warps meet at a block barrier between granules.
 *
 * Cross-frame recurrence: bin_search_StepSize starts from gfc.OldValue/CurrentStep left by the previous frame.
 * Frames are encoded in parallel from a speculated in-state, the out-states are compared with the successor's
 * assumption and mismatching frames are redone (a device loop in quant_run) until a fixed point -- byte-identical to
 * the sequential order.
 */
#ifndef MP3B200_K_QUANT_CUH
#define MP3B200_K_QUANT_CUH
#include <stddef.h>
#include "mp3_device.cuh"
#include "mp3_tables.h"
#include "k_psy.cuh"

#define Q_LARGE_BITS 100000
#define Q_IXMAX 8206
#define Q_FULL 0xffffffffu

struct GranuleInfoDev {
  int global_gain, part2_3_length, part2_length, big_values, count1, scalefac_compress;
  int table_select[3], region0_count, region1_count, preflag, scalefac_scale, count1table_select, block_type;
  int subblock_gain[4];
  int count1bits, sfbmax, sfbdivide, sfb_lmax, psymax, psy_lmax, sfb_smin, max_nonzero_coeff;
  int scalefac[MP3_SFBMAX];
  int slen[4];                      /* MPEG-2 / 2.5 (LSF): scalefactor bit widths of the four partitions (scale_bitcount_lsf) */
  int part_row;                     /* LSF: row of nr_of_sfb_block[0]: 0 long {6,5,5,5}, 1 short {9,9,9,9} */
  int pad_;
  double xrpow_max;
};
struct QuantFrameState {
  int stream, rel_frame;
  int in_old[2], in_step[2];        /* assumed gfc.OldValue / CurrentStep at frame start */
  int out_old[2], out_step[2];      /* state after the frame */
  int bs_gain0[2], bs_step0[2];     /* state right after gr0's bin search (re-validation shortcut) */
  int used0[2];                     /* bits gr0 spent per channel (part2_3_length + part2_length) */
  unsigned long long bs_hash[2][2]; /* [gr][ch] fingerprint of cod_info right after the bin search: stale fields such as
                                       table_select[] of an empty region depend on the gains the search visited */
  int scfsi[2][4];                  /* [ch][band group], decided while gr1 is finished */
  int redo;                         /* re-validation pass: Q_R0(ch) gr0 rate loop must be redone, Q_R1S(ch) gr1 search must be
                                       re-run (start step changed), Q_R1(ch) gr1 rate loop must be redone */
  int valid;
};
#define Q_R0(ch) (1 << (ch))
#define Q_R1S(ch) (4 << (ch))
#define Q_R1(ch) (16 << (ch))
#define Q_R0_ANY 3
#define Q_R1_ANY 48
#define Q_R1S_ANY 12
/* what the prepare kernel hands to the search / rate-loop kernels besides the xr and xrpow rows */
struct GcPrep { float xmin[MP3_SFBMAX]; int have, mnz, block_type; double xrpow_max; };

/* tables indexed by data (different index per lane) live in global memory and are read through the read-only
 * cache (__ldg): divergent __constant__ reads would serialise 32-fold */
__device__ unsigned short g_huff_code[1666];
__device__ unsigned char g_huff_len[1666];
__constant__ int c_huff_off[34];
__constant__ int c_huff_xlen[34];
__device__ int g_t32l[16];
__device__ int g_t33l[16];
__constant__ int c_slen1_n[16];
__constant__ int c_slen2_n[16];
__device__ int g_slen_n[2][16];                  /* slen1_n / slen2_n, read with one index per lane */
__device__ int g_scale_tab[2][16];               /* scale_long / scale_short */
/* Code lengths of a pair (x, y), both clamped to 15, at index x * 16 + y, for the table family of each "largest
 * value" class -- three candidate tables packed 11:11:10 (a | b << 11 | c << 22; families with fewer tables repeat
 * the last one, which never wins a strict comparison):
 *   0: max 1 -> table 1          1: max 2 -> 2, 3        2: max 3 -> 5, 6       3: max 4-5 -> 7, 8, 9
 *   4: max 6-7 -> 10, 11, 12     5: max 8-15 -> 13, 14, 15                      6: escape tables 16.. / 24.. (largetbl)
 *   7: all zero (region without non-zero lines) */
__device__ unsigned int g_cat_tab[8][256];
__constant__ int c_slen1_tab[16];
__constant__ int c_slen2_tab[16];
__constant__ int c_huf_noesc[15];

static int quant_upload_constants() {
  static const int t32l[16] = {1, 5, 5, 7, 5, 8, 7, 9, 5, 7, 7, 9, 7, 9, 9, 10};
  static const int t33l[16] = {4, 5, 5, 6, 5, 6, 6, 7, 5, 6, 6, 7, 6, 7, 7, 8};
  static const int s1n[16] = {1, 1, 1, 1, 8, 2, 2, 2, 4, 4, 4, 8, 8, 8, 16, 16};
  static const int s2n[16] = {1, 2, 4, 8, 1, 2, 4, 8, 2, 4, 8, 2, 4, 8, 4, 8};
  static const int s1t[16] = {0, 0, 0, 0, 3, 1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4};
  static const int s2t[16] = {0, 1, 2, 3, 0, 1, 2, 3, 1, 2, 3, 1, 2, 3, 2, 3};
  static const int ss[16] = {0, 18, 36, 54, 54, 36, 54, 72, 54, 72, 90, 72, 90, 108, 108, 126};
  static const int sl[16] = {0, 10, 20, 30, 33, 21, 31, 41, 32, 42, 52, 43, 53, 63, 64, 74};
  static const int hn[15] = {1, 2, 5, 7, 7, 10, 10, 13, 13, 13, 13, 13, 13, 13, 13};
#define UP(sym, src) if (cudaMemcpyToSymbol(sym, src, sizeof(src)) != cudaSuccess) return -100
  UP(g_huff_code, MP3_HUFF_CODE); UP(g_huff_len, MP3_HUFF_LEN); UP(c_huff_off, MP3_HUFF_OFF);
  UP(c_huff_xlen, MP3_HUFF_XLEN);
  UP(g_t32l, t32l); UP(g_t33l, t33l); UP(c_slen1_n, s1n); UP(c_slen2_n, s2n);
  UP(c_slen1_tab, s1t); UP(c_slen2_tab, s2t); UP(c_huf_noesc, hn);
  {
    static int sn[2][16], st[2][16];
    static unsigned int ct[8][256];
    for (int k = 0; k < 16; k++) { sn[0][k] = s1n[k]; sn[1][k] = s2n[k]; st[0][k] = sl[k]; st[1][k] = ss[k]; }
    static const int fam[6] = {1, 2, 5, 7, 10, 13};
    for (int x = 0; x < 16; x++) for (int y = 0; y < 16; y++) {
      const int q = x * 16 + y;
      for (int c = 0; c < 6; c++) {
        const int t1 = fam[c], xl = MP3_HUFF_XLEN[t1];
        unsigned a = 0, b = 0, d = 0;
        if (x < xl && y < xl) {
          const int i = x * xl + y;
          if (c == 0) a = b = d = MP3_HUFF_LEN[MP3_HUFF_OFF[1] + i];
          else if (c == 1) { a = MP3_HUFF_TABLE23[i] >> 16; b = d = MP3_HUFF_TABLE23[i] & 0xffff; }       /* count_bit_noESC_from2 */
          else if (c == 2) { a = MP3_HUFF_TABLE56[i] >> 16; b = d = MP3_HUFF_TABLE56[i] & 0xffff; }
          else { a = MP3_HUFF_LEN[MP3_HUFF_OFF[t1] + i]; b = MP3_HUFF_LEN[MP3_HUFF_OFF[t1 + 1] + i]; d = MP3_HUFF_LEN[MP3_HUFF_OFF[t1 + 2] + i]; }
        }
        ct[c][q] = a | (b << 11) | (d << 22);
      }
      { const unsigned a = MP3_HUFF_LARGETBL[q] >> 16, b = MP3_HUFF_LARGETBL[q] & 0xffff; ct[6][q] = a | (b << 11) | (b << 22); }
      ct[7][q] = 0;
    }
    UP(g_slen_n, sn); UP(g_scale_tab, st); UP(g_cat_tab, ct);
  }
#undef UP
  return 0;
}

/* ---- per-warp working set (shared memory) ---------------------------------------------------------------- */
struct __align__(16) GcWork {
  float xrpow[576];
  short ixw[576];                /* the one quantised-line buffer: cod_info_w.l3_enc; cod_info.l3_enc (best so far) is
                                    either this buffer (best_here) or parked in global memory at ixg */
  short* ixg;                    /* this gc's row of the l3_enc array in HBM */
  GranuleInfoDev w, b;           /* cod_info_w / cod_info */
  const Mp3Geo* geo;             /* band geometry of this block type (constant table in HBM, L1-resident) */
  float xmin[MP3_SFBMAX], distort[MP3_SFBMAX];
  int pn_step[MP3_SFBMAX]; float pn_noise[MP3_SFBMAX], pn_noise_log[MP3_SFBMAX];
  int pn_global_gain, pn_sfb_count1;
  unsigned char mode[MP3_SFBMAX + 1];
  short nstart[MP3_SFBMAX], nlen[MP3_SFBMAX];
  int scratch[8];
  double dscratch[4];
  __align__(16) float xr[576];   /* gi.xr after short-block reorder and analog-silence zeroing.  LAST member: the search and
                                    finish kernels never touch it and leave it out of their shared-memory footprint */
};
/* everything one warp (= one granule-channel task) keeps in shared memory */
struct __align__(16) WarpShared {
  double ath[6];                  /* analog-silence thresholds of the pseudo bands (psfb21 or psfb12) of this gc */
  int scfsi[4];
  GcWork wk;                      /* last, so that wk.xr is the tail of the struct */
};
/* per-warp stride of the kernels that do not use wk.xr */
#define Q_STRIDE_NOXR ((int)((offsetof(WarpShared, wk) + offsetof(GcWork, xr) + 15) & ~(size_t)15))
static_assert((offsetof(WarpShared, wk) + offsetof(GcWork, xr)) % 16 == 0 && (offsetof(WarpShared, wk) + offsetof(GcWork, xrpow)) % 16 == 0 &&
              (offsetof(WarpShared, wk) + offsetof(GcWork, ixw)) % 16 == 0 && sizeof(WarpShared) % 16 == 0, "rows are moved as 16-byte vectors");
#ifndef Q_SLIM_BLOCKS
#define Q_SLIM_BLOCKS 9           /* blocks per SM of the slim kernels (shared memory allows 10) */
#endif

#define LANE (threadIdx.x & 31)
#ifdef Q_TASKSTAT
/* tuning builds: per rate-loop task {clocks >> 6, gr, max_nonzero_coeff, block type, gain in, bits in, target bits, gain out} */
__device__ int g_taskstat[1 << 16][8];
#endif
/* -DQ_STATS: call counters for tuning (tools/profile_run.py prints them); absent from the product build */
#ifdef Q_STATS
__device__ unsigned long long g_qstats[16];
#define QSTAT(i) do { if (LANE == 0) atomicAdd(&g_qstats[i], 1ull); } while (0)
#else
#define QSTAT(i) do { } while (0)
#endif
/* tuning knobs (tools/build_variants.py) */
#define Q_PRAGMA(x) _Pragma(#x)
#define Q_UNROLL(n) Q_PRAGMA(unroll n)
#ifndef Q_RT_UNROLL
#define Q_RT_UNROLL 1
#endif
#ifndef Q_CB_UNROLL
#define Q_CB_UNROLL 1
#endif
#ifndef Q_CN_UNROLL
#define Q_CN_UNROLL 2          /* calc_noise band chain: unroll 1 / 2 -> C2 step 5.16 / 5.13 ms (H100 SXM, 400 W) */
#endif
#ifndef Q_HELPER
#define Q_HELPER __forceinline__
#endif
#ifndef Q_SPEC_START
#define Q_SPEC_START 180
#endif
#ifndef Q_SPEC_STEP
#define Q_SPEC_STEP 32
#endif
#ifndef Q_SPEC_GR1_STEP
#define Q_SPEC_GR1_STEP 2      /* the start step a speculated MPEG-1 frame hands its gr1 search (k_q_search) */
#endif
#ifndef Q_SPEC_FOLD
#define Q_SPEC_FOLD 1          /* 0: no re-validation / repair inside the first pass; the fixed-point loop does all of it */
#endif
#ifndef Q_MIN_BLOCKS
#define Q_MIN_BLOCKS 14
#endif
/* one copy of the fdlibm routines per kernel instead of one per call site (instruction-cache footprint) */
__device__ __noinline__ double q_log10(double x) { return m3_log10(x); }
__device__ __noinline__ double q_pow(double x, double y) { return m3_pow(x, y); }
__device__ __forceinline__ int wmax(int v) { return __reduce_max_sync(Q_FULL, v); }
__device__ __forceinline__ int wsum(int v) { return __reduce_add_sync(Q_FULL, v); }
__device__ __forceinline__ unsigned wsumu(unsigned v) { return __reduce_add_sync(Q_FULL, v); }

/* ---- choose_table (Takehiro.js:465-516) with its count_bit_* callees, table-driven ------------------------------
 * A region is classified by its largest value (RegionClass); one pass then adds, for every pair, the packed code
 * lengths of the class's candidate tables (g_cat_tab) -- the same loop for every class, so a warp can sum several
 * regions of different classes in one sweep.  A pair is one 32-bit shared-memory word (x | y << 16). */
struct RegionClass { int cat; unsigned lin; int t1, t2; };   /* lin: linbits of (t1, t2, t2) packed like the table */
__device__ Q_HELPER RegionClass region_class(int mx) {
  RegionClass rc;
  rc.lin = 0; rc.t2 = 0;
  if (mx == 0) { rc.cat = 7; rc.t1 = 0; }
  else if (mx <= 15) {
    rc.t1 = c_huf_noesc[mx - 1];
    rc.cat = mx <= 3 ? mx - 1 : (mx <= 5 ? 3 : (mx <= 7 ? 4 : 5));
  } else {
    /* first table of 24..31, then first of (t2 - 8)..23, whose linmax covers mx - 15: linmax is
     * {1,3,7,15,63,255,1023,8191} for 16..23 and {15,31,63,127,255,511,2047,8191} for 24..31 (Tables.js ht[]) */
    /* both counts depend only on the bit length n of v = mx - 15 (all thresholds are 2^k - 1): nibble n of the literals */
    const int n = 32 - __clz(mx - 15);
    rc.t2 = 24 + (int)((0x7777665432100000ull >> (4 * n)) & 15ull);
    rc.t1 = max(rc.t2 - 8, 16 + (int)((0x7777766554432100ull >> (4 * n)) & 15ull));
    const unsigned la = (unsigned)c_huff_xlen[rc.t1], lb = (unsigned)c_huff_xlen[rc.t2];
    rc.lin = la | (lb << 11) | (lb << 22);
    rc.cat = 6;
  }
  return rc;
}
/* packed lengths of one pair under class (cat, lin) */
__device__ __forceinline__ unsigned pair_bits(unsigned w, int cat, unsigned lin) {
  const unsigned x = w & 0xffffu, y = w >> 16;
  const unsigned xe = min(x, 15u), ye = min(y, 15u);
  return __ldg(&g_cat_tab[cat][xe * 16 + ye]) + ((x > 14u) + (y > 14u)) * lin;
}
/* table and bits of a region from the warp totals (a, b, c) of its three packed sums */
__device__ Q_HELPER int region_pick(int mx, const RegionClass& rc, int a, int b, int c, int* bits) {
  DOMAIN_MISS(DOM_REGION_MX, mx > Q_IXMAX);
  if (mx > Q_IXMAX) { *bits = Q_LARGE_BITS; return -1; }
  if (mx == 0) return 0;
  int t = rc.t1;
  if (mx <= 15) {
    if (a > b) { a = b; t++; }
    if (a > c) { a = c; t = rc.t1 + 2; }
  } else if (a > b) { a = b; t = rc.t2; }
  *bits += a;
  return t;
}

/* Huffman table and bits of the pairs [begin, end) (even bounds) */
__device__ __forceinline__ int region_table_w(const short* ix, int begin, int end, int* bits) {
  const int lane = LANE;
  const unsigned* w32 = reinterpret_cast<const unsigned*>(ix);
  const int p0 = (begin >> 1) + lane, p1 = end >> 1;
  unsigned m = 0;
Q_UNROLL(Q_RT_UNROLL)
  for (int p = p0; p < p1; p += 32) m = __vmaxu2(m, w32[p]);        /* both 16-bit halves at once */
  const int mx = (int)__reduce_max_sync(Q_FULL, max(m & 0xffffu, m >> 16));
  if (mx == 0) return 0;
  const RegionClass rc = region_class(mx);
  unsigned s = 0;                                  /* a lane adds <= 9 pairs x <= 45 bits per field */
  if (rc.cat == 6) {
Q_UNROLL(Q_RT_UNROLL)
    for (int p = p0; p < p1; p += 32) s += pair_bits(w32[p], 6, rc.lin);
  } else {                                         /* no value above 15: the pair is its own table index */
    const unsigned int* tab = g_cat_tab[rc.cat];
Q_UNROLL(Q_RT_UNROLL)
    for (int p = p0; p < p1; p += 32) { const unsigned w = w32[p]; s += __ldg(&tab[((w & 0xfu) << 4) | (w >> 16)]); }
  }
#ifdef MP3_DOMAIN_CHECK
  {   /* the same sums field by field, unpacked: a field that carried into its neighbour differs */
    unsigned fa = 0, fb = 0, fc = 0;
    for (int p = p0; p < p1; p += 32) {
      const unsigned v = rc.cat == 6 ? pair_bits(w32[p], 6, rc.lin) : __ldg(&g_cat_tab[rc.cat][((w32[p] & 0xfu) << 4) | (w32[p] >> 16)]);
      fa += v & 0x7ffu; fb += (v >> 11) & 0x7ffu; fc += v >> 22;
    }
    DOMAIN_MISS(DOM_BITSUM_FIELD, fa > 0x7ffu || fb > 0x7ffu || fc > 0x3ffu || wsumu(fa) > 0xffffu || wsumu(fb) > 0xffffu);
  }
#endif
  /* warp totals need up to 14 bits: reduce (a, b) as two 16-bit fields, c alone */
  const unsigned ab = wsumu((s & 0x7ffu) | (((s >> 11) & 0x7ffu) << 16));
  const int c = wsum((int)(s >> 22));
  return region_pick(mx, rc, (int)(ab & 0xffffu), (int)(ab >> 16), c, bits);
}

/* noquant_count_bits (Takehiro.js:521-628).  gi scalars are updated by lane 0. */
/* `top`: per lane, end (2p + 2) of its last non-zero pair below i0 = min(576, (max_nonzero_coeff + 2) & ~1), found by
 * the quantising loop of the caller while it had the pair in a register */
__device__ __forceinline__ int noquant_count_bits_w(const Mp3Tables* T, const short* ix, GranuleInfoDev* gi, GcWork* wk, bool use_prev, int top) {
  const int lane = LANE;
  const unsigned* w32 = reinterpret_cast<const unsigned*>(ix);
  /* count1 = end of the last non-zero pair below i0 */
  const int count1 = wmax(top);
  /* quadruples of |x| <= 1 counted down from count1 (values are >= 0: "<= 1" == no bit above bit 0 in either half) */
  int a1 = 0, a2 = 0, nq = 0;
  const int qmax = count1 >> 2;
  bool stop = false;
#pragma unroll 1
  for (int q0 = 0; q0 < qmax && !stop; q0 += 32) {
    const int q = q0 + lane;
    int bad = 1, v1 = 0, v2 = 0;
    if (q < qmax) {
      const int i = count1 - 4 * q;
      const unsigned wa = w32[(i - 4) >> 1], wb = w32[(i - 2) >> 1];
      if (((wa | wb) & 0xfffefffeu) == 0) {
        bad = 0;
        const int p = (int)(((wa & 1u) << 3) | ((wa >> 16) << 2) | ((wb & 1u) << 1) | (wb >> 16));
        v1 = __ldg(&g_t32l[p]); v2 = __ldg(&g_t33l[p]);
      }
    }
    const unsigned m = __ballot_sync(Q_FULL, bad);
    const int first_bad = m ? __ffs(m) - 1 : 32;
    if (lane >= first_bad) { v1 = 0; v2 = 0; }
    a1 += wsum(v1); a2 += wsum(v2);
    nq += first_bad;
    if (first_bad < 32) stop = true;
  }
  if (nq > qmax) nq = qmax;
  const int bigv = count1 - 4 * nq;
  int bits = a1, c1sel = 0;
  if (a1 > a2) { bits = a2; c1sel = 1; }
  const int count1bits = bits;
  int r0 = gi->region0_count, r1 = gi->region1_count;
  int ts0 = gi->table_select[0], ts1 = gi->table_select[1], ts2 = gi->table_select[2];
  if (bigv != 0) {
    int b1, b2;
    const int bt = gi->block_type;
    if (bt == BT_SHORT) {
      b1 = 3 * T->sfb_s[3];
      b2 = bigv;
    } else if (bt == BT_NORM) {
      b1 = r0 = T->bv_scf[bigv - 2];
      b2 = r1 = T->bv_scf[bigv - 1];
      b2 = T->sfb_l[b1 + b2 + 2];
      b1 = T->sfb_l[b1 + 1];
    } else {
      r0 = 7; r1 = 22 - 1 - 7 - 1;
      b1 = T->sfb_l[7 + 1];
      b2 = bigv;
    }
    b1 = min(b1, bigv);
    b2 = min(b2, bigv);
    /* same order as the reference: region 2 (long blocks only), then 0, then 1; empty regions keep their table.
     * One small routine inlined at three call sites: calls and their stack frame cost more than the code size (DESIGN.md §6). */
    if (bt == BT_NORM && b2 < bigv) { QSTAT(15); ts2 = region_table_w(ix, b2, bigv, &bits); }
    if (0 < b1) { QSTAT(15); ts0 = region_table_w(ix, 0, b1, &bits); }
    if (b1 < b2) { QSTAT(15); ts1 = region_table_w(ix, b1, b2, &bits); }
  }
  __syncwarp();
  if (lane == 0) {
    gi->count1 = count1; gi->count1table_select = c1sel; gi->count1bits = count1bits; gi->big_values = bigv;
    gi->region0_count = r0; gi->region1_count = r1;
    gi->table_select[0] = ts0; gi->table_select[1] = ts1; gi->table_select[2] = ts2;
    if (use_prev) {
      int sc = 0;                                  /* first band edge at or above big_values */
      if (bigv != 0 && gi->block_type == BT_NORM) {
        if (bigv >= 576) sc = 22;
        else { sc = T->geo[0].sfb_of_line[bigv]; if (T->sfb_l[sc] != bigv) sc++; }
      }
      wk->pn_sfb_count1 = sc;
    }
  }
  __syncwarp();
  return bits;
}

/* pretab[sfb] (0 beyond band 20) from a packed literal: each lane asks for a different band */
__device__ __forceinline__ int pretab_of(int sfb) { return sfb < 22 ? (int)((0x2fe95400000ull >> (2 * sfb)) & 3ull) : 0; }

/* step of scalefactor band sfb (Takehiro.js:205-209 / QuantizePVT.js:744-747) */
__device__ __forceinline__ int sfb_step(const GranuleInfoDev* gi, const GcWork* wk, int sfb) {
  return gi->global_gain - ((gi->scalefac[sfb] + (gi->preflag != 0 ? pretab_of(sfb) : 0)) << (gi->scalefac_scale + 1)) -
         gi->subblock_gain[wk->geo->window[sfb]] * 8;
}

/* count_bits (Takehiro.js:630-660) = range check + quantize_xrpow (:171-314) + noquant_count_bits */
template <bool use_prev>
__device__ __forceinline__ int count_bits_w(const Mp3Tables* T, GcWork* wk, GranuleInfoDev* gi, short* ix) {
  const int lane = LANE;
  const double istep = (double)T->ipow20[gi->global_gain];
  if (gi->xrpow_max > T->ixmax_over_istep[gi->global_gain]) return Q_LARGE_BITS;
  const int sfbmax = gi->block_type == BT_SHORT ? 38 : 21;
  const int mnz = gi->max_nonzero_coeff;
  unsigned* iw32 = reinterpret_cast<unsigned*>(ix);
  const int i0h = min(576, ((mnz + 2) >> 1) << 1) >> 1;    /* noquant_count_bits looks for count1 below this pair index */
  if (!use_prev) {
    /* bin_search_StepSize path (prevNoise == null): no band is cached and none uses the 0/1 quantizer, so the band
     * walk of quantize_xrpow reduces to: full quantizer below the truncation point, zeros from max_nonzero_coeff on.
     * Band starts are even, hence the quantised range ends at (mnz + 1) & ~1 (an odd tail length drops its last line). */
    const int qend = (mnz + 1) & ~1;
    int top = 0;
Q_UNROLL(Q_CB_UNROLL)
    for (int p = lane; p < 288; p += 32) {            /* two lines per step: one 64-bit load, one 32-bit store */
      unsigned v = 0;
      if (2 * p < qend) {
        const float2 xp = *reinterpret_cast<const float2*>(&wk->xrpow[2 * p]);
        double x0 = (double)xp.x * istep, x1 = (double)xp.y * istep;
        x0 += (double)__ldg(&T->adj43[js_trunc<DOM_TRUNC_QUANT>(x0)]);
        x1 += (double)__ldg(&T->adj43[js_trunc<DOM_TRUNC_QUANT>(x1)]);
        v = (unsigned)js_trunc<DOM_TRUNC_QUANT>(x0) | ((unsigned)js_trunc<DOM_TRUNC_QUANT>(x1) << 16);
        DOMAIN_MISS(DOM_PACK_SEARCH, x0 >= 32768.0 || x1 >= 32768.0);
        if (v != 0 && p < i0h) top = 2 * p + 2;
      }
      iw32[p] = v;
    }
    __syncwarp();
    return noquant_count_bits_w(T, ix, gi, wk, false, top);
  }
  const bool prev_data_use = use_prev && (gi->global_gain == wk->pn_global_gain);
  const bool calc_step = prev_data_use || gi->block_type == BT_NORM;
  /* per-band decision: 0 skip (cached), 1 full quantizer, 2 zero/one quantizer; term = first non-cached band that
   * crosses max_nonzero_coeff (the reference zero-fills the tail there and stops) */
  int term = sfbmax + 1;
#pragma unroll 1
  for (int s0 = 0; s0 <= sfbmax; s0 += 32) {
    const int sfb = s0 + lane;
    int md = 0, trunc_here = 0;
    if (sfb <= sfbmax) {
      const int jst = wk->geo->start[sfb];
      const int step = calc_step ? sfb_step(gi, wk, sfb) : -1;
      if (prev_data_use && wk->pn_step[sfb] == step) md = 0;
      else {
        if (jst + wk->geo->width[sfb] > mnz) trunc_here = 1;
        md = (use_prev && wk->pn_sfb_count1 > 0 && sfb >= wk->pn_sfb_count1 && wk->pn_step[sfb] > 0 && step >= wk->pn_step[sfb]) ? 2 : 1;
      }
      wk->mode[sfb] = (unsigned char)md;
      wk->nstart[sfb] = jst;
    }
    const unsigned m = __ballot_sync(Q_FULL, trunc_here);
    if (m && term == sfbmax + 1) term = s0 + __ffs(m) - 1;
  }
  __syncwarp();
  /* lines >= zero_from are zero-filled (Arrays.fill(pi, max_nonzero_coeff, 576, 0) happens when the walk reaches the
   * truncating band); the truncating band itself quantises an even number of lines in full mode */
  int zero_from = 576;
  if (term <= sfbmax) {
    const int term_len = mnz - wk->nstart[term] + 1;
    zero_from = term_len > 0 ? ((term_len & 1) ? mnz : mnz + 1) : mnz;
    if (lane == 0) wk->mode[term] = 1;
  }
  __syncwarp();
  const double compare01 = T->cmp01_over_istep[gi->global_gain];
  int top = 0;
Q_UNROLL(Q_CB_UNROLL)
  for (int p = lane; p < 288; p += 32) {              /* pairs never straddle a band: band starts and widths are even */
    const int i = 2 * p;
    unsigned v;
    if (i >= zero_from) { v = 0; iw32[p] = 0; }
    else {
      const int md = wk->mode[wk->geo->sfb_of_line[i]];
      const bool z1 = (i + 1) >= zero_from;           /* zero_from may be odd: only the pair's second line is cleared */
      if (md == 0) {
        v = iw32[p];
        if (z1) { v &= 0xffffu; iw32[p] = v; }
      } else {
        const float2 xp = *reinterpret_cast<const float2*>(&wk->xrpow[i]);
        unsigned v0, v1;
        if (md == 2) { v0 = (compare01 > (double)xp.x) ? 0u : 1u; v1 = (compare01 > (double)xp.y) ? 0u : 1u; }
        else {
          double x0 = (double)xp.x * istep, x1 = (double)xp.y * istep;
          x0 += (double)__ldg(&T->adj43[js_trunc<DOM_TRUNC_QUANT>(x0)]);
          x1 += (double)__ldg(&T->adj43[js_trunc<DOM_TRUNC_QUANT>(x1)]);
          v0 = (unsigned)js_trunc<DOM_TRUNC_QUANT>(x0); v1 = (unsigned)js_trunc<DOM_TRUNC_QUANT>(x1);
          DOMAIN_MISS(DOM_PACK_OUTER, x0 >= 32768.0 || x1 >= 32768.0);
        }
        if (z1) v1 = 0;
        v = v0 | (v1 << 16);
        iw32[p] = v;
      }
    }
    if (v != 0 && p < i0h) top = 2 * p + 2;
  }
  __syncwarp();
  return noquant_count_bits_w(T, ix, gi, wk, use_prev, top);
}

/* calc_noise (QuantizePVT.js:725-878) for quant_comp 9: over_count, over_SSD, max_noise (+ distort[]) */
struct NoiseRes { int over_count; double over_SSD, max_noise; int bits; };
__device__ __forceinline__ void calc_noise_w(const Mp3Tables* T, GcWork* wk, const GranuleInfoDev* gi, const short* ix, NoiseRes* res) {
  const int lane = LANE;
  const int psymax = gi->psymax, mnz = gi->max_nonzero_coeff;
  /* Line cursor: a band starts where the previous one stopped.  Cached bands and bands that end at or below
   * max_nonzero_coeff advance by their full (even) width, so up to the first non-cached band that crosses the truncation
   * point every band starts at its nominal offset; from there on the walk is sequential (lane 0, usually 1-2 bands). */
  int first_trunc = psymax;
#pragma unroll 1
  for (int s0 = 0; s0 < psymax; s0 += 32) {
    const int sfb = s0 + lane;
    int crosses = 0;
    if (sfb < psymax) {
      const int j = wk->geo->start[sfb], w = wk->geo->width[sfb];
      if (wk->pn_step[sfb] == sfb_step(gi, wk, sfb)) wk->nlen[sfb] = -1;
      else { wk->nstart[sfb] = (short)j; wk->nlen[sfb] = (short)(w >> 1); crosses = (j + w) > mnz; }
    }
    const unsigned m = __ballot_sync(Q_FULL, crosses);
    if (m && first_trunc == psymax) first_trunc = s0 + __ffs(m) - 1;
  }
  __syncwarp();
  if (lane == 0 && first_trunc < psymax) {
    int j = wk->geo->start[first_trunc];
#pragma unroll 1
    for (int sfb = first_trunc; sfb < psymax; sfb++) {
      const int w = wk->geo->width[sfb];
      if (wk->nlen[sfb] < 0) { j += w; continue; }
      int l = w >> 1;
      if ((j + w) > mnz) { const int us = mnz - j + 1; l = us > 0 ? us >> 1 : 0; }
      wk->nstart[sfb] = (short)j; wk->nlen[sfb] = (short)l;
      j += 2 * l;
    }
  }
  __syncwarp();
  int over = 0, ssd = 0; double mxn = -20.0;
#pragma unroll 1
  for (int s0 = 0; s0 < psymax; s0 += 32) {
    const int sfb = s0 + lane;
    if (sfb < psymax) {
      const int s = sfb_step(gi, wk, sfb);
      const bool cached = wk->nlen[sfb] < 0;
      double noise;
      if (cached) noise = (double)wk->pn_noise[sfb];
      else {
        const double step = (double)T->pow20[s + MP3_QMAX2];
        int j = wk->nstart[sfb];
        noise = 0;
Q_UNROLL(Q_CN_UNROLL)
        for (int l = wk->nlen[sfb]; l > 0; l--, j += 2) {          /* j is even: one 64-bit and one 32-bit load per pair */
          const float2 x = *reinterpret_cast<const float2*>(&wk->xr[j]);
          const unsigned q0 = reinterpret_cast<const unsigned short*>(ix)[j], q1 = reinterpret_cast<const unsigned short*>(ix)[j + 1];
          double temp;                             /* (two 16-bit loads: the index is ready without shift / mask / 64-bit add) */
          temp = fabs((double)x.x) - (double)__ldg(&T->pow43[q0]) * step; noise += temp * temp;
          temp = fabs((double)x.y) - (double)__ldg(&T->pow43[q1]) * step; noise += temp * temp;
        }
        wk->pn_step[sfb] = s;
        { f32s t; t = noise; wk->pn_noise[sfb] = t.v; }
      }
      noise = noise / (double)wk->xmin[sfb];       /* distort = noise / xmin from the cached or the fresh noise */
      { f32s t; t = noise; wk->distort[sfb] = t.v; }
      if (cached) noise = (double)wk->pn_noise_log[sfb];
      else {
        noise = q_log10(js_dmax(noise, 1E-20));
        { f32s t; t = noise; wk->pn_noise_log[sfb] = t.v; }
      }
      if (noise > 0.0) {
        int tmp = js_trunc<DOM_TRUNC_NOISE>(noise * 10 + .5);
        if (tmp < 1) tmp = 1;
        ssd += tmp * tmp;
        over++;
      }
      mxn = js_dmax(mxn, noise);
    }
  }
  /* over_SSD is a sum of small squared integers (exact in a double in any order): integer warp sum */
#pragma unroll 1
  for (int o = 16; o > 0; o >>= 1) {
    const double other = __shfl_xor_sync(Q_FULL, mxn, o);
    mxn = js_dmax(mxn, other);
  }
  over = wsum(over);
  if (lane == 0) wk->pn_global_gain = gi->global_gain;
  __syncwarp();
  res->over_count = over; res->over_SSD = (double)wsum(ssd); res->max_noise = mxn;
}

/* scale_bitcount (Takehiro.js:980-1030), MPEG-1, all lanes; returns true when no legal scalefac_compress exists */
__device__ __forceinline__ bool scale_bitcount_w(GranuleInfoDev* gi) {
  const int lane = LANE;
  int* scalefac = gi->scalefac;
  const bool is_short = gi->block_type == BT_SHORT;
  const int sfbmax = gi->sfbmax, sfbdivide = gi->sfbdivide;
  __syncwarp();
  if (!is_short && 0 == gi->preflag) {
    const bool in = lane >= 11 && lane < 21;
    const int pt = pretab_of(lane);
    const bool ok = !in || scalefac[lane] >= pt;
    if (__all_sync(Q_FULL, ok)) {
      __syncwarp();
      if (in) scalefac[lane] -= pt;
      if (lane == 0) gi->preflag = 1;
      __syncwarp();
    }
  }
  int m1 = 0, m2 = 0;
#pragma unroll 1
  for (int sfb = lane; sfb < sfbmax; sfb += 32) {
    const int v = scalefac[sfb];
    if (sfb < sfbdivide) m1 = max(m1, v); else m2 = max(m2, v);
  }
  m1 = wmax(m1); m2 = wmax(m2);
  /* first k with the smallest table value among the legal ones: min over (value, k) */
  int key = Q_LARGE_BITS * 16 + 15;
  if (lane < 16 && m1 < __ldg(&g_slen_n[0][lane]) && m2 < __ldg(&g_slen_n[1][lane])) key = __ldg(&g_scale_tab[is_short ? 1 : 0][lane]) * 16 + lane;
  key = __reduce_min_sync(Q_FULL, key);
  const int p2 = key >> 4;
  if (lane == 0) { gi->part2_length = p2; if (p2 != Q_LARGE_BITS) gi->scalefac_compress = key & 15; }
  __syncwarp();
  return p2 == Q_LARGE_BITS;
}

/* scale_bitcount_lsf (Takehiro.js:1036-1132), MPEG-2 / 2.5, all lanes; returns true when a partition's largest scalefactor
 * exceeds its range (the side info fields are then left as they were, like the reference).  preflag is never set on the LSF
 * path (scale_bitcount and the pre-emphasis step of best_scalefac_store are MPEG-1 only; inc_scalefac_scale clears it), so
 * only partition table 0 occurs: long {6,5,5,5}, short {9,9,9,9} bands, ranges {15,15,7,7}. */
__device__ __forceinline__ bool scale_bitcount_lsf_w(GranuleInfoDev* gi) {
  const int lane = LANE;
  const bool is_short = gi->block_type == BT_SHORT;
  __syncwarp();
  /* partition of scalefactor index i: long bands 0-5 | 6-10 | 11-15 | 16-20; short: 9 consecutive (band, window) entries each */
  int m0 = 0, m1 = 0, m2 = 0, m3 = 0;
  const int n = is_short ? 36 : 21;
#pragma unroll 1
  for (int i = lane; i < n; i += 32) {
    const int v = gi->scalefac[i];
    const int p = is_short ? i / 9 : (i < 6 ? 0 : (i - 6) / 5 + 1);
    if (p == 0) m0 = max(m0, v); else if (p == 1) m1 = max(m1, v); else if (p == 2) m2 = max(m2, v); else m3 = max(m3, v);
  }
  m0 = wmax(m0); m1 = wmax(m1); m2 = wmax(m2); m3 = wmax(m3);
  const bool over = m0 > 15 || m1 > 15 || m2 > 7 || m3 > 7;
  if (!over && lane == 0) {
    /* log2tab (Takehiro.js:1138): bits needed for 0..15 */
    const int s1 = m0 ? 32 - __clz(m0) : 0, s2 = m1 ? 32 - __clz(m1) : 0, s3 = m2 ? 32 - __clz(m2) : 0, s4 = m3 ? 32 - __clz(m3) : 0;
    gi->slen[0] = s1; gi->slen[1] = s2; gi->slen[2] = s3; gi->slen[3] = s4;
    gi->part_row = is_short ? 1 : 0;
    gi->scalefac_compress = (((s1 * 5) + s2) << 4) + (s3 << 2) + s4;
    gi->part2_length = is_short ? 9 * (s1 + s2 + s3 + s4) : 6 * s1 + 5 * (s2 + s3 + s4);
  }
  __syncwarp();
  return over;
}
/* scale_bitcount of the stream's MPEG version (Quantize.js:814-817,840-843; Takehiro.js:937-941) */
__device__ __forceinline__ bool scale_bitcount_any_w(GranuleInfoDev* gi, int mode_gr) {
  return mode_gr == 2 ? scale_bitcount_w(gi) : scale_bitcount_lsf_w(gi);
}

/* loop_break (Quantize.js:584-594): true when every band is amplified */
__device__ __forceinline__ bool loop_break_w(const GranuleInfoDev* gi, const GcWork* wk) {
  bool nz = true;
#pragma unroll 1
  for (int sfb = LANE; sfb < gi->sfbmax; sfb += 32)
    if (gi->scalefac[sfb] + gi->subblock_gain[wk->geo->window[sfb]] == 0) nz = false;
  return __all_sync(Q_FULL, nz);
}

/* multiply xrpow of the bands flagged in wk->mode[] by `factor[band]` (amp_scalefac_bands / inc_scalefac_scale
 * line loops, Quantize.js:650-655,690-695) and fold the new values into xrpow_max */
__device__ __forceinline__ void scale_xrpow_w(GcWork* wk, GranuleInfoDev* gi, double f34) {
  const int lane = LANE;
  const int sfbmax = gi->sfbmax;
  float mx = 0.0f;
#pragma unroll 1
  for (int p = lane; p < 288; p += 32) {              /* a pair of lines lies in one band */
    const int sfb = wk->geo->sfb_of_line[2 * p];
    if (sfb < sfbmax && wk->mode[sfb]) {
      float2* xp = reinterpret_cast<float2*>(&wk->xrpow[2 * p]);
      float2 x = *xp;
      f32s v0, v1; v0.v = x.x; v1.v = x.y;
      v0 *= f34; v1 *= f34;
      x.x = v0.v; x.y = v1.v;
      *xp = x;
      mx = fmaxf(mx, fmaxf(v0.v, v1.v));
    }
  }
#pragma unroll 1
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(Q_FULL, mx, o));
  if (lane == 0 && (double)mx > gi->xrpow_max) gi->xrpow_max = (double)mx;
  __syncwarp();
}

/* second half of balance_noise: the scalefactors no longer fit -- switch to scalefac_scale 1 or raise a
 * subblock_gain (rare; kept out of the hot function's instruction footprint) */
__device__ __noinline__ bool balance_escalate_w(const Mp3Tables* T, GcWork* wk) {
  const int lane = LANE;
  GranuleInfoDev* gi = &wk->w;
  int* flag = &wk->scratch[0];
  bool status = true;
  const int scale_now = gi->scalefac_scale, is_short_blk = gi->block_type == BT_SHORT;
  __syncwarp();                                    /* all lanes hold the decision inputs before lane 0 edits gi */
  if (T->noise_shaping > 1) {
    if (0 == scale_now) {
      /* inc_scalefac_scale (Quantize.js:676-699) */
      {
        const int sfbmax = gi->sfbmax, pre = gi->preflag;
#pragma unroll 1
        for (int sfb = lane; sfb < sfbmax; sfb += 32) {
          int s = gi->scalefac[sfb];
          if (pre != 0) s += pretab_of(sfb);
          const int odd = (s & 1) != 0;
          if (odd) s++;
          wk->mode[sfb] = (unsigned char)odd;
          gi->scalefac[sfb] = s >> 1;
        }
        __syncwarp();
        if (lane == 0) { gi->preflag = 0; gi->scalefac_scale = 1; }
      }
      __syncwarp();
      scale_xrpow_w(wk, gi, 1.29683955465100964055);
      status = false;
    } else if (is_short_blk) {                    /* gfc.subblock_gain == 1 */
      /* inc_subblock_gain (Quantize.js:705-781): lane 0 decides, all lanes rescale the touched windows */
      if (lane == 0) {
        int ret = 0;
        int* scalefac = gi->scalefac;
#pragma unroll 1
        for (int i = 0; i < MP3_SFBMAX; i++) wk->nlen[i] = -1;      /* per-band amp index: -1 none, else ipow20 index */
#pragma unroll 1
        for (int window = 0; window < 3 && !ret; window++) {
          int s1 = 0, s2 = 0, sfb;
#pragma unroll 1
          for (sfb = gi->sfb_lmax + window; sfb < gi->sfbdivide; sfb += 3) if (s1 < scalefac[sfb]) s1 = scalefac[sfb];
#pragma unroll 1
          for (; sfb < gi->sfbmax; sfb += 3) if (s2 < scalefac[sfb]) s2 = scalefac[sfb];
          if (s1 < 16 && s2 < 8) continue;
          if (gi->subblock_gain[window] >= 7) { ret = 1; break; }
          gi->subblock_gain[window]++;
#pragma unroll 1
          for (sfb = gi->sfb_lmax + window; sfb < gi->sfbmax; sfb += 3) {
            int s = scalefac[sfb];
            s = s - (4 >> gi->scalefac_scale);
            if (s >= 0) { scalefac[sfb] = s; continue; }
            scalefac[sfb] = 0;
            wk->nlen[sfb] = 210 + s * (1 << (gi->scalefac_scale + 1));
          }
          wk->nlen[sfb] = 202;                      /* sfb12 window `window`: sfb == sfbmax + window */
        }
        *flag = ret;
      }
      __syncwarp();
      /* NOTE: when inc_subblock_gain bails out with `true` mid-way the windows already processed stay modified,
       * exactly like the reference (it returns without undoing). */
      {
        float mx = 0.0f;
#pragma unroll 1
        for (int i = lane; i < 576; i += 32) {
          const int sfb = wk->geo->sfb_of_line[i];
          if (sfb < MP3_SFBMAX && wk->nlen[sfb] >= 0) {
            f32s v; v.v = wk->xrpow[i];
            v *= (double)T->ipow20[wk->nlen[sfb]];
            wk->xrpow[i] = v.v;
            mx = fmaxf(mx, v.v);
          }
        }
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(Q_FULL, mx, o));
        if (lane == 0 && (double)mx > gi->xrpow_max) gi->xrpow_max = (double)mx;
        __syncwarp();
      }
      {
        const int bailed = *flag;
        __syncwarp();
        status = bailed != 0 || loop_break_w(gi, wk);
      }
    }
  }
  if (!status) status = scale_bitcount_any_w(gi, T->mode_gr);
  return !status;
}


/* balance_noise (Quantize.js:783-846) on cod_info_w.  Returns true when a new scalefactor combination exists. */
__device__ __forceinline__ bool balance_noise_w(const Mp3Tables* T, GcWork* wk) {
  const int lane = LANE;
  GranuleInfoDev* gi = &wk->w;
  /* ---- amp_scalefac_bands, noise_shaping_amp == 1 (Quantize.js:597-660) ---- */
  const double ifq = gi->scalefac_scale == 0 ? 1.29683955465100964055 : 1.68179283050742922612;
  {
    const int sfbmax = gi->sfbmax;
    double trigger = 0;
#pragma unroll 1
    for (int sfb = lane; sfb < sfbmax; sfb += 32) if (trigger < (double)wk->distort[sfb]) trigger = (double)wk->distort[sfb];
    for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_xor_sync(Q_FULL, trigger, o); if (trigger < t) trigger = t; }
    if (trigger > 1.0) trigger = sqrt(trigger);     /* Math.pow(trigger, .5): fdlibm returns sqrt(x) for y == 0.5 */
    else trigger *= .95;
#pragma unroll 1
    for (int sfb = lane; sfb < sfbmax; sfb += 32) {
      const int amp = !((double)wk->distort[sfb] < trigger);
      wk->mode[sfb] = (unsigned char)amp;
      if (amp) gi->scalefac[sfb]++;
    }
  }
  __syncwarp();
  scale_xrpow_w(wk, gi, ifq);
  /* ---- rest of balance_noise ---- */
  int r;
  if (loop_break_w(gi, wk)) r = 0;                 /* all bands amplified */
  else r = scale_bitcount_any_w(gi, T->mode_gr) ? 2 : 1;   /* 2: scalefactors too large, try scalefac_scale / subblock_gain */
  if (r == 0) return false;
  if (r == 1) return true;
  return balance_escalate_w(T, wk);
}

__device__ __forceinline__ void copy_gi_w(GranuleInfoDev* dst, const GranuleInfoDev* src) {
  const int n = sizeof(GranuleInfoDev) / 4;
  const int* s = reinterpret_cast<const int*>(src);
  int* d = reinterpret_cast<int*>(dst);
  __syncwarp();                                   /* earlier readers of *dst are done */
  static_assert(sizeof(GranuleInfoDev) / 4 <= 96, "three rounds");
  int v[3];
#pragma unroll
  for (int k = 0; k < 3; k++) { const int i = LANE + 32 * k; if (i < n) v[k] = s[i]; }   /* loads in flight together (HBM rows) */
#pragma unroll
  for (int k = 0; k < 3; k++) { const int i = LANE + 32 * k; if (i < n) d[i] = v[k]; }
  __syncwarp();
}
__device__ __forceinline__ void copy_ix_w(short* dst, const short* src) {
  const int* s = reinterpret_cast<const int*>(src);
  int* d = reinterpret_cast<int*>(dst);
  __syncwarp();
#pragma unroll 1
  for (int i = LANE; i < 288; i += 32) d[i] = s[i];
  __syncwarp();
}

/* bin_search_StepSize (Quantize.js:322-381) on cod_info (wk->b / ixb) */
__device__ __forceinline__ int bin_search_w(const Mp3Tables* T, GcWork* wk, int desired_rate, int* old_value, int* current_step, int stat_base = 0) {
  GranuleInfoDev* gi = &wk->b;
  int nBits;
  int CurrentStep = *current_step;
  bool flagGoneOver = false;
  const int start = *old_value;
  int Direction = 0;
  int gain = start;
  desired_rate -= gi->part2_length;
  __syncwarp();
  for (;;) {
    int step;
    if (LANE == 0) gi->global_gain = gain;
    __syncwarp();
    QSTAT(stat_base);
    nBits = count_bits_w<false>(T, wk, gi, wk->ixw);
    if (CurrentStep == 1 || nBits == desired_rate) break;
    if (nBits > desired_rate) {
      if (Direction == 2) flagGoneOver = true;
      if (flagGoneOver) CurrentStep /= 2;
      Direction = 1;
      step = CurrentStep;
    } else {
      if (Direction == 1) flagGoneOver = true;
      if (flagGoneOver) CurrentStep /= 2;
      Direction = 2;
      step = -CurrentStep;
    }
    gain += step;
    if (gain < 0) { gain = 0; flagGoneOver = true; }
    if (gain > 255) { gain = 255; flagGoneOver = true; }
  }
  while (nBits > desired_rate && gain < 255) {
    gain++;
    if (LANE == 0) gi->global_gain = gain;
    __syncwarp();
    QSTAT(stat_base + 1);
    nBits = count_bits_w<false>(T, wk, gi, wk->ixw);
  }
  *current_step = (start - gain >= 4) ? 4 : 2;
  *old_value = gain;
  if (LANE == 0) gi->part2_3_length = nBits;
  __syncwarp();
  return nBits;
}

/* fingerprint of a GranuleInfoDev (every lane returns the same value): each lane mixes its words with their position,
 * the warp combines them with a sum and an xor (order-free, so no serial chain) */
__device__ __forceinline__ unsigned long long gi_hash(const GranuleInfoDev* gi) {
  const unsigned* w = reinterpret_cast<const unsigned*>(gi);
  unsigned sum = 0, x = 0;
#pragma unroll 1
  for (int i = LANE; i < (int)(sizeof(GranuleInfoDev) / 4); i += 32) {
    unsigned v = (w[i] ^ ((unsigned)i * 0x9E3779B9u)) * 0x85EBCA6Bu;
    v ^= v >> 13; v *= 0xC2B2AE35u; v ^= v >> 16;
    sum += v; x ^= __funnelshift_l(v, v, i & 31);
  }
  sum = __reduce_add_sync(Q_FULL, sum);
  x = __reduce_xor_sync(Q_FULL, x);
  return ((unsigned long long)sum << 32) | x;
}

/* outer_loop (Quantize.js:871-1052) for noise_shaping_amp 1, full_outer_loop 0, substep_shaping 0 */
/* The bin search that opens outer_loop (Quantize.js:884) runs in its own kernel (k_q_search); this is everything after it.
 * gfc.OldValue / CurrentStep are final right after the search (outer_loop never touches them again). */
__device__ __forceinline__ void outer_loop_w(const Mp3Tables* T, GcWork* wk, int targ_bits) {
  const int lane = LANE;
  NoiseRes best, cur;
  int best_part2_3_length = 9999999;
#pragma unroll 1
  for (int i = lane; i < MP3_SFBMAX; i += 32) { wk->pn_step[i] = 0; wk->pn_noise[i] = 0.0f; wk->pn_noise_log[i] = 0.0f; }
  if (lane == 0) { wk->pn_global_gain = 0; wk->pn_sfb_count1 = 0; }
  __syncwarp();
  calc_noise_w(T, wk, &wk->b, wk->ixw, &best);
  best.bits = wk->b.part2_3_length;
  copy_gi_w(&wk->w, &wk->b);
  bool best_here = true;          /* cod_info.l3_enc == the shared-memory buffer (no copy parked in HBM yet) */
  int age = 0;
  const int quant_comp = T->quant_comp;   /* 9 for long and short */
  (void)quant_comp;
  do {
    const int search_limit = 3;
    int maxggain = 255;
    if (!balance_noise_w(T, wk)) break;
    GranuleInfoDev* w = &wk->w;
    if (w->scalefac_scale != 0) maxggain = 254;
    const int huff_bits = targ_bits - w->part2_length;
    if (huff_bits <= 0) break;
    int p23, gg;
    if (best_here) { copy_ix_w(wk->ixg, wk->ixw); best_here = false; }   /* park the best lines before re-quantising */
    int sc_in;                                     /* prev_noise.sfb_count1 as the last count_bits call of this loop saw it */
    for (;;) {                                     /* while (count_bits > huff_bits && global_gain <= maxggain) global_gain++ */
      sc_in = wk->pn_sfb_count1;
      QSTAT(8);
      p23 = count_bits_w<true>(T, wk, w, wk->ixw);
      gg = w->global_gain;
      __syncwarp();                                /* every lane has read the gain before lane 0 bumps it */
      if (!(p23 > huff_bits && gg <= maxggain)) break;
      if (lane == 0) w->global_gain = gg + 1;
      __syncwarp();
    }
    if (lane == 0) w->part2_3_length = p23;
    __syncwarp();
    if (gg > maxggain) break;
    if (best.over_count == 0) {
      /* The reference calls count_bits again at the very gain the loop above stopped at.  Its only input that the
       * previous call can have changed is prev_noise.sfb_count1 (everything else -- gain, scalefactors, xrpow, the cached
       * lines and tables of cod_info_w -- is what that call left behind); if that value did not change the repeat would
       * recompute the identical state and bit count, so it is skipped. */
      bool repeat = wk->pn_sfb_count1 == sc_in;
      for (;;) {
        if (!repeat) { QSTAT(9); p23 = count_bits_w<true>(T, wk, w, wk->ixw); }
        repeat = false;
        gg = w->global_gain;
        __syncwarp();
        if (!(p23 > best_part2_3_length && gg <= maxggain)) break;
        if (lane == 0) w->global_gain = gg + 1;
        __syncwarp();
      }
      if (lane == 0) w->part2_3_length = p23;
      __syncwarp();
      if (gg > maxggain) break;
    }
    QSTAT(10);
    calc_noise_w(T, wk, w, wk->ixw, &cur);
    cur.bits = w->part2_3_length;
    /* quant_compare, case 9 (Quantize.js:493-505,560-567) */
    bool better;
    if (best.over_count > 0) {
      better = cur.over_SSD <= best.over_SSD;
      if (cur.over_SSD == best.over_SSD) better = cur.bits < best.bits;
    } else {
      better = ((cur.max_noise < 0) && ((cur.max_noise * 10 + cur.bits) <= (best.max_noise * 10 + best.bits)));
    }
    if (best.over_count == 0) better = better && cur.bits < best.bits;
    if (better) {
      best_part2_3_length = wk->b.part2_3_length;   /* sic: read before the assign (Quantize.js:996-998) */
      best = cur;
      copy_gi_w(&wk->b, &wk->w);
      best_here = true;
      age = 0;
    } else {
      if (++age > search_limit && best.over_count == 0) break;
    }
    const int cont = (wk->w.global_gain + wk->w.scalefac_scale) < 255;
    __syncwarp();
    if (!cont) break;
  } while (true);
  if (!best_here) copy_ix_w(wk->ixw, wk->ixg);
}

/* athAdjust (QuantizePVT.js:541-561) */
__device__ __noinline__ double ath_adjust_dev(double a, double x, double athFloor) {
  const double o = 90.30873362, p = 94.82444863;
  double u = q_log10(x) * 10.0;
  const double v = a * a;
  double w = 0.0;
  u -= athFloor;
  if (v > 1E-20) w = 1. + q_log10(v) * (10.0 / o);
  if (w < 0) w = 0.;
  u *= w;
  u += athFloor + o - p;
  return q_pow(10., 0.1 * u);
}

/* init_outer_loop + psfb21_analogsilence + init_xrpow + calc_xmin for one gc (Quantize.js:204-306,147-202,105-138;
 * QuantizePVT.js:569-719).  Returns false when the granule is digital silence (all l3_enc = 0). */
__device__ __noinline__ bool gc_prepare_w(const Mp3Tables* T, GcWork* wk, const double* ath_ps, const float* __restrict__ xr_g, int block_type,
                             const PsyRatioDev* __restrict__ ratio, double ath_adjust) {
  const bool need_xmin = true;
  const int lane = LANE;
  GranuleInfoDev* gi = &wk->b;
  const bool is_short = block_type == BT_SHORT;
  if (lane == 0) {
    gi->part2_3_length = 0; gi->big_values = 0; gi->count1 = 0; gi->global_gain = 210; gi->scalefac_compress = 0;
    gi->table_select[0] = gi->table_select[1] = gi->table_select[2] = 0;
    gi->subblock_gain[0] = gi->subblock_gain[1] = gi->subblock_gain[2] = gi->subblock_gain[3] = 0;
    gi->region0_count = 0; gi->region1_count = 0; gi->preflag = 0; gi->scalefac_scale = 0; gi->count1table_select = 0;
    gi->part2_length = 0; gi->block_type = block_type; gi->count1bits = 0;
    gi->sfb_lmax = is_short ? 0 : 21; gi->sfb_smin = is_short ? 0 : 12;
    gi->psy_lmax = is_short ? 0 : 21;
    gi->psymax = is_short ? 36 : 21; gi->sfbmax = is_short ? 36 : 21; gi->sfbdivide = is_short ? 18 : 11;
    gi->max_nonzero_coeff = 575;
#pragma unroll 1
    for (int i = 0; i < MP3_SFBMAX; i++) gi->scalefac[i] = 0;
    gi->xrpow_max = 0;
  }
  /* band geometry: constant per block type; short blocks are reordered band-major on the way in */
  const Mp3Geo* geo = &T->geo[is_short ? 1 : 0];
  if (lane == 0) wk->geo = geo;
  {
    /* the whole row in flight before any of it is used (rows are 2304 B apart: 16-byte vectors); short blocks are scattered
     * to the quantizer's band-major line order */
    float4 v[5];
#pragma unroll
    for (int k = 0; k < 5; k++) { const int q = lane + 32 * k; if (q < 144) v[k] = __ldg(reinterpret_cast<const float4*>(xr_g) + q); }
    if (!is_short) {
#pragma unroll
      for (int k = 0; k < 5; k++) { const int q = lane + 32 * k; if (q < 144) reinterpret_cast<float4*>(wk->xr)[q] = v[k]; }
    } else {
#pragma unroll
      for (int k = 0; k < 5; k++) {
        const int q = lane + 32 * k;
        if (q < 144) {
          const short* ro = geo->reorder + 4 * q;
          wk->xr[__ldg(ro + 0)] = v[k].x; wk->xr[__ldg(ro + 1)] = v[k].y; wk->xr[__ldg(ro + 2)] = v[k].z; wk->xr[__ldg(ro + 3)] = v[k].w;
        }
      }
    }
  }
  __syncwarp();
  /* analog silence in the pseudo bands above sfb21 / sfb12 (Quantize.js:147-202): walking down from the top line, lines
   * below the band's ATH are zeroed until the first one that is not.  Long blocks: the stop line is the highest line at or
   * above its threshold (a max over lanes); everything above it is cleared in parallel.  Short blocks: lane 0, as written. */
  if (!is_short) {
    const int lo = T->psfb21[0];
    const double lf = (double)T->longfact[21];
    int keep = lo - 1;
#pragma unroll 1
    for (int j = lo + lane; j < 576; j += 32) {
      int g = 0;
      while (g < 5 && j >= T->psfb21[g + 1]) g++;
      double ath21 = ath_ps[g];
      if (lf > 1e-12) ath21 *= lf;
      if (!(fabs((double)wk->xr[j]) < ath21)) keep = j;
    }
    keep = wmax(keep);
    __syncwarp();                                   /* every lane's reads above are done before anyone clears lines */
#pragma unroll 1
    for (int j = keep + 1 + lane; j < 576; j += 32) wk->xr[j] = 0.0f;
  } else if (lane == 0) {
#pragma unroll 1
    for (int block = 0; block < 3; block++) {
      bool stop = false;
#pragma unroll 1
      for (int g = 5; g >= 0 && !stop; g--) {
        const int start = T->sfb_s[12] * 3 + (T->sfb_s[13] - T->sfb_s[12]) * block + (T->psfb12[g] - T->psfb12[0]);
        const int end = start + (T->psfb12[g + 1] - T->psfb12[g]);
        double ath12 = ath_ps[g];
        if ((double)T->shortfact[12] > 1e-12) ath12 *= (double)T->shortfact[12];
#pragma unroll 1
        for (int j = end - 1; j >= start; j--) {
          if (fabs((double)wk->xr[j]) < ath12) wk->xr[j] = 0.0f;
          else { stop = true; break; }
        }
      }
    }
  }
  __syncwarp();
  /* ---- init_xrpow: max_nonzero_coeff is still 575 here (set by init_outer_loop) ---- */
  {
    float mx = 0.0f, amax = 0.0f;
#pragma unroll 1
    for (int p = lane; p < 288; p += 32) {
      const float2 x = *reinterpret_cast<const float2*>(&wk->xr[2 * p]);
      const double t0 = fabs((double)x.x), t1 = fabs((double)x.y);
      f32s p0, p1; p0 = sqrt(t0 * sqrt(t0)); p1 = sqrt(t1 * sqrt(t1));
      float2 o; o.x = p0.v; o.y = p1.v;
      *reinterpret_cast<float2*>(&wk->xrpow[2 * p]) = o;
      mx = fmaxf(mx, fmaxf(p0.v, p1.v));
      amax = fmaxf(amax, fmaxf((float)t0, (float)t1));
    }
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) { mx = fmaxf(mx, __shfl_xor_sync(Q_FULL, mx, o)); amax = fmaxf(amax, __shfl_xor_sync(Q_FULL, amax, o)); }
    /* sum > 1e-20 ? (Quantize.js:129): a running sum of non-negative terms is >= its largest term */
    bool energy;
    if ((double)amax > 1E-20) energy = true;
    else {
      if (lane == 0) { double sum = 0; for (int i = 0; i <= 575; ++i) sum += fabs((double)wk->xr[i]); wk->scratch[1] = sum > 1E-20; }
      __syncwarp();
      energy = wk->scratch[1] != 0;
      __syncwarp();
    }
    if (lane == 0) gi->xrpow_max = (double)mx;
    __syncwarp();
    if (!energy) {
#pragma unroll 1
      for (int i = lane; i < 576; i += 32) wk->ixw[i] = 0;
      __syncwarp();
      return false;
    }
  }
  /* ---- calc_xmin ---- */
  const double masking_lower = is_short ? T->masking_lower_short : T->masking_lower_long;
  if (!is_short) {
    if (need_xmin && lane < 21) {
      const int gsfb = lane;
      int j = T->sfb_l[gsfb];
      const int width = wk->geo->width[gsfb];
      double xmin = ath_adjust * (double)T->ath_l[gsfb];
      double en0 = 0.0;
#pragma unroll 1
      for (int l = width >> 1; l > 0; l--) {
        double xa = (double)wk->xr[j] * (double)wk->xr[j]; en0 += xa; j++;
        double xb = (double)wk->xr[j] * (double)wk->xr[j]; en0 += xb; j++;
      }
      const double e = (double)ratio->en_l[gsfb];
      if (e > 0.0) {
        const double x = en0 * (double)ratio->thm_l[gsfb] * masking_lower / e;
        if (xmin < x) xmin = x;
      }
      f32s o; o = xmin * (double)T->longfact[gsfb];
      wk->xmin[gsfb] = o.v;
    }
    /* highest non-zero coefficient (QuantizePVT.js:645-653) */
    int last = -1;
#pragma unroll 1
    for (int i = lane; i < 576; i += 32) if (wk->xr[i] != 0.0f) last = i;
    last = wmax(last);
    int mnz = last + 1;
    if (mnz > 575) mnz = 575;
    if (lane == 0) gi->max_nonzero_coeff = mnz;
  } else {
#pragma unroll 1
    for (int t = lane; need_xmin && t < 36; t += 32) {
      const int sfb = t / 3, b = t - 3 * sfb;
      const int width = wk->geo->width[t];
      int j = 3 * T->sfb_s[sfb] + b * width;
      const double tmpATH = ath_adjust * (double)T->ath_s[sfb];
      double en0 = 0.0;
#pragma unroll 1
      for (int l = width >> 1; l > 0; l--) {
        double xa = (double)wk->xr[j] * (double)wk->xr[j]; en0 += xa; j++;
        double xb = (double)wk->xr[j] * (double)wk->xr[j]; en0 += xb; j++;
      }
      double xmin = tmpATH;
      const double e = (double)ratio->en_s[sfb][b];
      if (e > 0.0) {
        const double x = en0 * (double)ratio->thm_s[sfb][b] * masking_lower / e;
        if (xmin < x) xmin = x;
      }
      f32s o; o = xmin * (double)T->shortfact[sfb];
      wk->xmin[t] = o.v;
    }
    __syncwarp();
    if (need_xmin && lane < 12) {   /* temporal smoothing across the three windows (useTemporal, QuantizePVT.js:707-714) */
      f32s* p = reinterpret_cast<f32s*>(&wk->xmin[3 * lane]);
      if ((double)p[0] > (double)p[1]) p[1] += ((double)p[0] - (double)p[1]) * T->decay;
      if ((double)p[1] > (double)p[2]) p[2] += ((double)p[1] - (double)p[2]) * T->decay;
    }
    if (lane == 0) gi->max_nonzero_coeff = 575;
  }
  __syncwarp();
  return true;
}

/* best_scalefac_store without the scfsi part (Takehiro.js:809-875), then scfsi_calc for gr1 (lane 0 logic) */
/* g0: final side info of gr0 of the same channel (HBM), read only when gr == 1; scfsi[4]: this channel's flags */
__device__ __noinline__ void best_scalefac_store_w(GcWork* wk, int* scfsi, const GranuleInfoDev* __restrict__ g0, int gr, int mode_gr) {
  const int lane = LANE;
  GranuleInfoDev* gi = &wk->b;
  /* bands whose quantised lines are all zero */
#pragma unroll 1
  for (int s0 = 0; s0 < gi->sfbmax; s0 += 32) {
    const int sfb = s0 + lane;
    if (sfb < gi->sfbmax) {
      const int j = wk->geo->start[sfb];
      bool any = false;
#pragma unroll 1
      for (int l = 0; l < wk->geo->width[sfb]; l += 2) if (*reinterpret_cast<const unsigned*>(&wk->ixw[j + l]) != 0) { any = true; break; }
      wk->mode[sfb] = any ? 1 : 0;
    }
  }
  __syncwarp();
  const int sfbmax = gi->sfbmax;
  int recalc_w = 0;                                  /* warp-uniform copy of `recalc` up to the scfsi step */
  {
    bool z = false;
#pragma unroll 1
    for (int sfb = lane; sfb < sfbmax; sfb += 32) if (!wk->mode[sfb]) { gi->scalefac[sfb] = -2; z = true; }
    if (__any_sync(Q_FULL, z)) recalc_w = -2;
  }
  __syncwarp();
  if (0 == gi->scalefac_scale && 0 == gi->preflag) {
    int sor = 0;
#pragma unroll 1
    for (int sfb = lane; sfb < sfbmax; sfb += 32) { const int v = gi->scalefac[sfb]; if (v > 0) sor |= v; }
    sor = (int)__reduce_or_sync(Q_FULL, (unsigned)sor);
    if (0 == (sor & 1) && sor != 0) {
#pragma unroll 1
      for (int sfb = lane; sfb < sfbmax; sfb += 32) { const int v = gi->scalefac[sfb]; if (v > 0) gi->scalefac[sfb] = v >> 1; }
      __syncwarp();
      if (lane == 0) gi->scalefac_scale = 1;
      recalc_w = 1;
    }
  }
  __syncwarp();
  if (0 == gi->preflag && gi->block_type != BT_SHORT && mode_gr == 2) {
    const bool in = lane >= 11 && lane < 21;
    const int v = in ? gi->scalefac[lane] : 0, pt = pretab_of(lane);
    const bool ok = !in || !(v < pt && v != -2);
    if (__all_sync(Q_FULL, ok)) {
      if (in && v > 0) gi->scalefac[lane] = v - pt;
      __syncwarp();
      if (lane == 0) gi->preflag = 1;
      recalc_w = 1;
    }
  }
  __syncwarp();
  if (lane == 0) {
    int recalc = recalc_w;
#pragma unroll 1
    for (int i = 0; i < 4; i++) scfsi[i] = 0;
    if (gr == 1 && g0->block_type != BT_SHORT && gi->block_type != BT_SHORT) {
      /* scfsi_calc (Takehiro.js:877-943) */
      const int* g0sf = g0->scalefac;
      const int band[5] = {0, 6, 11, 16, 21};
      int sfb;
#pragma unroll 1
      for (int i = 0; i < 4; i++) {
#pragma unroll 1
        for (sfb = band[i]; sfb < band[i + 1]; sfb++)
          if (g0sf[sfb] != gi->scalefac[sfb] && gi->scalefac[sfb] >= 0) break;
        if (sfb == band[i + 1]) {
#pragma unroll 1
          for (sfb = band[i]; sfb < band[i + 1]; sfb++) gi->scalefac[sfb] = -1;
          scfsi[i] = 1;
        }
      }
      int s1 = 0, c1 = 0;
#pragma unroll 1
      for (sfb = 0; sfb < 11; sfb++) {
        if (gi->scalefac[sfb] == -1) continue;
        c1++;
        if (s1 < gi->scalefac[sfb]) s1 = gi->scalefac[sfb];
      }
      int s2 = 0, c2 = 0;
#pragma unroll 1
      for (; sfb < 21; sfb++) {
        if (gi->scalefac[sfb] == -1) continue;
        c2++;
        if (s2 < gi->scalefac[sfb]) s2 = gi->scalefac[sfb];
      }
#pragma unroll 1
      for (int i = 0; i < 16; i++) {
        if (s1 < c_slen1_n[i] && s2 < c_slen2_n[i]) {
          const int c = c_slen1_tab[i] * c1 + c_slen2_tab[i] * c2;
          if (gi->part2_length > c) { gi->part2_length = c; gi->scalefac_compress = i; }
        }
      }
      recalc = 0;
    }
    wk->scratch[0] = recalc;
  }
  __syncwarp();
#pragma unroll 1
  for (int sfb = lane; sfb < sfbmax; sfb += 32) if (gi->scalefac[sfb] == -2) gi->scalefac[sfb] = 0;
  __syncwarp();
  const int recalc = wk->scratch[0];
  __syncwarp();
  if (recalc != 0) scale_bitcount_any_w(gi, mode_gr);
}

/* ---- best_huffman_divide (Takehiro.js:666-800) on cod_info (wk->b); wk->w is free to use as cod_info2 -----------------
 * recalc_divide_init tries every region0/region1 split (up to 16 x 8 choose_table calls) and recalc_divide_sub every
 * region2 start.  All those regions are unions of whole scalefactor bands (plus the partial band below big_values), so the
 * work is done once per band: largest value, number of escape values, and the packed code-length sums under every table
 * class the band can appear in (a band's class can only be raised by its neighbours).  A region is then a max and a few
 * adds over its bands.  The scratch overlays xrpow, which is dead once outer_loop has returned. */
struct DivScratch {
  unsigned ab[23][7];               /* band b, class c: field a | field b << 16 (valid for c >= the band's own class) */
  unsigned short cc[23][7];         /* field c */
  unsigned short bmax[23], nesc[23];
  int r0bits[16]; unsigned char r0t[16];
  int cbits[128]; unsigned char ct1[128];   /* (r0, r1) combinations; reused per region2 start by recalc_divide_sub */
};
static_assert(sizeof(DivScratch) <= 576 * sizeof(float), "DivScratch must fit into the xrpow array");

/* per-band statistics of the pairs below big_values; returns the number of bands (a partial last band counts) */
__device__ __noinline__ int band_stats_w(const Mp3Tables* T, const short* ix, int bigv, DivScratch* ds) {
  const int lane = LANE;
  const unsigned* w32 = reinterpret_cast<const unsigned*>(ix);
  int B = 0;
  while (B < 22 && T->sfb_l[B + 1] <= bigv) B++;                 /* bands 0..B-1 lie entirely below big_values */
  const int nb = (B < 22 && T->sfb_l[B] < bigv) ? B + 1 : B;      /* band B = [sfb_l[B], big_values) if not empty */
  __syncwarp();
#pragma unroll 1
  for (int b = lane; b < nb; b += 32) {
    const int lo = T->sfb_l[b] >> 1, hi = (b < B ? T->sfb_l[b + 1] : bigv) >> 1;
    unsigned m = 0, ne = 0;
#pragma unroll 1
    for (int p = lo; p < hi; p++) { const unsigned w = w32[p]; m = __vmaxu2(m, w); ne += ((w & 0xffffu) > 14u) + ((w >> 16) > 14u); }
    ds->bmax[b] = (unsigned short)max(m & 0xffffu, m >> 16);
    ds->nesc[b] = (unsigned short)ne;
  }
  __syncwarp();
#pragma unroll 1
  for (int t = lane; t < nb * 7; t += 32) {                       /* one (band, class) task per lane and round */
    const int b = t / 7, c = t - 7 * b;
    const int mx = ds->bmax[b];
    const int lowc = mx <= 1 ? 0 : (mx <= 3 ? mx - 1 : (mx <= 5 ? 3 : (mx <= 7 ? 4 : (mx <= 15 ? 5 : 6))));
    if (c < lowc) continue;
    const unsigned int* tab = g_cat_tab[c];
    const int lo = T->sfb_l[b] >> 1, hi = (b < B ? T->sfb_l[b + 1] : bigv) >> 1;
    unsigned sa = 0, sb = 0, sc = 0;
#pragma unroll 1
    for (int p = lo; p < hi; p++) {
      const unsigned w = w32[p];
      const unsigned v = __ldg(&tab[min(w & 0xffffu, 15u) * 16 + min(w >> 16, 15u)]);
      sa += v & 0x7ffu; sb += (v >> 11) & 0x7ffu; sc += v >> 22;
    }
    DOMAIN_MISS(DOM_BITSUM_FIELD, sa > 0xffffu || sb > 0xffffu || sc > 0xffffu);
    ds->ab[b][c] = sa | (sb << 16);
    ds->cc[b][c] = (unsigned short)sc;
  }
  __syncwarp();
  return nb;
}

/* choose_table over the bands b0..b1 from the statistics: table, and its bits added to *bits */
__device__ __forceinline__ int region_from_bands(const DivScratch* ds, int b0, int b1, int* bits) {
  int mx = 0;
#pragma unroll 1
  for (int b = b0; b <= b1; b++) mx = max(mx, (int)ds->bmax[b]);
  if (mx == 0) return 0;
  const RegionClass rc = region_class(mx);
  int sa = 0, sb = 0, sc = 0, ne = 0;
#pragma unroll 1
  for (int b = b0; b <= b1; b++) {
    const unsigned u = ds->ab[b][rc.cat];
    sa += (int)(u & 0xffffu); sb += (int)(u >> 16); sc += ds->cc[b][rc.cat]; ne += ds->nesc[b];
  }
  if (rc.cat == 6) { sa += ne * (int)(rc.lin & 0x7ffu); sb += ne * (int)((rc.lin >> 11) & 0x7ffu); sc = sb; }
  return region_pick(mx, rc, sa, sb, sc, bits);
}

/* recalc_divide_init (Takehiro.js:666-700): best (region0, region1) split for every region1 end */
__device__ __noinline__ void divide_init_w(const Mp3Tables* T, DivScratch* ds, int bigv, int* r01_bits, int* r01_div, int* r0_tbl, int* r1_tbl) {
  const int lane = LANE;
  if (lane < 16) {
    int bits0 = -1, t0 = 0;
    if (T->sfb_l[lane + 1] < bigv) { bits0 = 0; t0 = region_from_bands(ds, 0, lane, &bits0); }
    ds->r0bits[lane] = bits0; ds->r0t[lane] = (unsigned char)t0;
  }
  __syncwarp();
#pragma unroll 1
  for (int k = lane; k < 128; k += 32) {
    const int r0 = k >> 3, r1 = k & 7;
    int bits = -1, t1 = 0;
    if (ds->r0bits[r0] >= 0 && r0 + r1 + 2 <= 22 && T->sfb_l[r0 + r1 + 2] < bigv) {
      bits = ds->r0bits[r0];
      t1 = region_from_bands(ds, r0 + 1, r0 + r1 + 1, &bits);
    }
    ds->cbits[k] = bits; ds->ct1[k] = (unsigned char)t1;
  }
  __syncwarp();
  if (lane < 23) {                                   /* the reference visits r0 ascending and keeps the first minimum */
    const int sidx = lane;
    int best = Q_LARGE_BITS;
#pragma unroll 1
    for (int r0 = 0; r0 < 16; r0++) {
      const int r1 = sidx - r0;
      if (r1 < 0 || r1 > 7) continue;
      const int bits = ds->cbits[r0 * 8 + r1];
      if (bits < 0) continue;
      if (best > bits) { best = bits; r01_div[sidx] = r0; r0_tbl[sidx] = ds->r0t[r0]; r1_tbl[sidx] = ds->ct1[r0 * 8 + r1]; }
    }
    r01_bits[sidx] = best;
  }
  __syncwarp();
}

/* recalc_divide_sub (Takehiro.js:702-725); `ds` holds the statistics for cod_info2->big_values */
__device__ __noinline__ void recalc_divide_sub_w(const Mp3Tables* T, GcWork* wk, DivScratch* ds, int nb, const GranuleInfoDev* cod_info2,
                                                 const int* r01_bits, const int* r01_div, const int* r0_tbl, const int* r1_tbl) {
  const int lane = LANE;
  GranuleInfoDev* gi = &wk->b;
  const int bigv = cod_info2->big_values;
  /* region2 = bands r2 .. nb-1 for every candidate start */
  if (lane + 2 <= 22) {
    const int r2 = lane + 2;
    int bits2 = 0, t2 = 0;
    if (T->sfb_l[r2] < bigv) t2 = region_from_bands(ds, r2, nb - 1, &bits2);
    ds->cbits[r2] = bits2; ds->ct1[r2] = (unsigned char)t2;
  }
  __syncwarp();
  int cur = gi->part2_3_length, best_r2 = -1;
  const int c1bits = cod_info2->count1bits;
#pragma unroll 1
  for (int r2 = 2; r2 < 22 + 1; r2++) {               /* the sequential acceptance rule, on precomputed numbers */
    if (T->sfb_l[r2] >= bigv) break;
    int bits = r01_bits[r2 - 2] + c1bits;
    if (cur <= bits) break;
    bits += ds->cbits[r2];
    if (cur <= bits) continue;
    cur = bits; best_r2 = r2;
  }
  __syncwarp();
  if (best_r2 >= 0) {
    if (cod_info2 != gi) copy_gi_w(gi, cod_info2);
    if (lane == 0) {
      gi->part2_3_length = cur;
      gi->region0_count = r01_div[best_r2 - 2];
      gi->region1_count = best_r2 - 2 - r01_div[best_r2 - 2];
      gi->table_select[0] = r0_tbl[best_r2 - 2];
      gi->table_select[1] = r1_tbl[best_r2 - 2];
      gi->table_select[2] = ds->ct1[best_r2];
    }
    __syncwarp();
  }
}

__device__ __noinline__ void best_huffman_divide_w(const Mp3Tables* T, GcWork* wk) {
  const int lane = LANE;
  GranuleInfoDev* gi = &wk->b;
  GranuleInfoDev* c2 = &wk->w;
  const short* ix = wk->ixw;
  /* 23 entries each; the noise cache and the distortion array are dead after outer_loop */
  int* r01_bits = reinterpret_cast<int*>(wk->pn_noise_log);
  int* r01_div = reinterpret_cast<int*>(wk->distort);
  int* r0_tbl = wk->pn_step;
  int* r1_tbl = reinterpret_cast<int*>(wk->pn_noise);
  DivScratch* ds = reinterpret_cast<DivScratch*>(wk->xrpow);
  if (gi->block_type == BT_SHORT && T->mode_gr == 1) return;   /* "SHORT BLOCK stuff fails for MPEG2" (Takehiro.js:735-737) */
  copy_gi_w(c2, gi);
  if (gi->block_type == BT_NORM) {
    const int bigv = gi->big_values;
    const int nb = band_stats_w(T, ix, bigv, ds);
    divide_init_w(T, ds, bigv, r01_bits, r01_div, r0_tbl, r1_tbl);
    recalc_divide_sub_w(T, wk, ds, nb, c2, r01_bits, r01_div, r0_tbl, r1_tbl);
  }
  int i = c2->big_values;
  if (i == 0 || (ix[i - 2] | ix[i - 1]) > 1) return;
  i = gi->count1 + 2;
  if (i > 576) return;
  copy_gi_w(c2, gi);
  int a1 = 0, a2 = 0;
  {
    /* quadruples from count1+2 down to the old big_values; integer sums, any order */
    const int top = i, bv = c2->big_values;
    int v1 = 0, v2 = 0, n = 0;
#pragma unroll 1
    for (int q = lane; top - 4 * q > bv; q += 32) {
      const int e = top - 4 * q;
      const int p = ((ix[e - 4] * 2 + ix[e - 3]) * 2 + ix[e - 2]) * 2 + ix[e - 1];
      v1 += __ldg(&g_t32l[p]); v2 += __ldg(&g_t33l[p]); n++;
    }
    a1 = wsum(v1); a2 = wsum(v2);
    i = top - 4 * wsum(n);
  }
  __syncwarp();
  if (lane == 0) {
    c2->count1 = gi->count1 + 2;
    c2->big_values = i;
    c2->count1table_select = 0;
    int a = a1;
    if (a1 > a2) { a = a2; c2->count1table_select = 1; }
    c2->count1bits = a;
  }
  __syncwarp();
  if (a1 > a2) a1 = a2;
  if (c2->block_type == BT_NORM) {
    const int nb2 = band_stats_w(T, ix, i, ds);        /* big_values moved down: the partial last band changed */
    recalc_divide_sub_w(T, wk, ds, nb2, c2, r01_bits, r01_div, r0_tbl, r1_tbl);
  } else {
    int p23 = a1;
    int b1 = T->sfb_l[7 + 1];
    if (b1 > i) b1 = i;
    int t0 = c2->table_select[0], t1 = c2->table_select[1];
    if (b1 > 0) t0 = region_table_w(ix, 0, b1, &p23);
    if (i > b1) t1 = region_table_w(ix, b1, i, &p23);
    __syncwarp();
    if (lane == 0) { c2->part2_3_length = p23; c2->table_select[0] = t0; c2->table_select[1] = t1; }
    __syncwarp();
    if (gi->part2_3_length > c2->part2_3_length) copy_gi_w(gi, c2);
  }
}

/* ---- bit packing (BitStream.js:110-138,428-689) --------------------------------------------------------- */
__device__ Q_HELPER void put_bits(unsigned int* buf, int pos, unsigned int val, int n) {
  if (n <= 0) return;
  val &= (n >= 32) ? 0xffffffffu : ((1u << n) - 1u);
  const int w = pos >> 5, off = pos & 31;
  const int room = 32 - off;
  if (n <= room) atomicOr(&buf[w], val << (room - n));
  else {
    atomicOr(&buf[w], val >> (n - room));
    atomicOr(&buf[w + 1], val << (32 - (n - room)));
  }
}

/* main data of one gc, starting at bit `pos` of the frame buffer; returns nothing (lengths are already known) */
/* sign of line i of the spectrum the quantizer saw (xr < 0), from the 576-bit mask k_q_prepare keeps per granule-channel */
#define QNEG(i) (((neg[(i) >> 5] >> ((i) & 31)) & 1u) != 0u)
__device__ __noinline__ void pack_gc_w(const Mp3Tables* T, unsigned int* buf, const GranuleInfoDev* gi, const short* ixq,
                                       const unsigned* neg, int pos) {
  const int lane = LANE;
  /* scalefactors (writeMainData, BitStream.js:609-625): serial, <= 36 values */
  if (lane == 0 && T->mode_gr == 1) {
    /* MPEG-2 / 2.5 (BitStream.js:641-687): four partitions, slen bits each, negative (unused) scalefactors sent as 0 */
    int p = pos, i = 0;
#pragma unroll 1
    for (int part = 0; part < 4; part++) {
      const int cnt = gi->part_row == 1 ? 9 : (part == 0 ? 6 : 5), sl = gi->slen[part];
#pragma unroll 1
      for (int k = 0; k < cnt; k++, i++) { put_bits(buf, p, (unsigned)max(gi->scalefac[i], 0), sl); p += sl; }
    }
  } else if (lane == 0) {
    const int slen1 = c_slen1_tab[gi->scalefac_compress], slen2 = c_slen2_tab[gi->scalefac_compress];
    int p = pos;
#pragma unroll 1
    for (int sfb = 0; sfb < gi->sfbmax; sfb++) {
      if (gi->scalefac[sfb] == -1) continue;
      const int sl = sfb < gi->sfbdivide ? slen1 : slen2;
      put_bits(buf, p, (unsigned)gi->scalefac[sfb], sl);
      p += sl;
    }
  }
  pos += gi->part2_length;
  const int bigv = gi->big_values;
  int r1s, r2s;
  if (gi->block_type == BT_SHORT) {
    r1s = 3 * T->sfb_s[3];
    if (r1s > bigv) r1s = bigv;
    r2s = bigv;
  } else {
    r1s = T->sfb_l[gi->region0_count + 1];
    r2s = T->sfb_l[gi->region0_count + 1 + gi->region1_count + 1];
    if (r1s > bigv) r1s = bigv;
    if (r2s > bigv) r2s = bigv;
  }
  /* big_values pairs: lane handles a contiguous run of pairs so that one prefix sum gives every bit position */
  const int npairs = bigv >> 1;
  const int per = (npairs + 31) >> 5;
  const int p0 = lane * per, p1 = min(npairs, p0 + per);
  int mybits = 0;
#pragma unroll 1
  for (int pass = 0; pass < 2; pass++) {
    int at = 0;
    if (pass == 1) {
      int incl = mybits;
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(Q_FULL, incl, o); if (lane >= o) incl += v; }
      at = pos + incl - mybits;
    }
#pragma unroll 1
    for (int pr = p0; pr < p1; pr++) {
      const int i = 2 * pr;
      int tb = i < r1s ? gi->table_select[0] : (i < r2s ? gi->table_select[1] : gi->table_select[2]);
      if (tb == 14) tb = 16;                      /* encodeSideInfo2 rewrites 14 -> 16 before the main data is coded */
      if (tb == 0) continue;
      const int hx = c_huff_xlen[tb];
      int linbits = hx, xlen = hx;
      int cbits = 0, xbits = 0;
      unsigned ext = 0;
      int x1 = ixq[i], x2 = ixq[i + 1];
      if (x1 != 0) { if (QNEG(i)) ext++; cbits--; }
      if (tb > 15) {
        if (x1 > 14) { ext |= (unsigned)(x1 - 15) << 1; xbits = linbits; x1 = 15; }
        if (x2 > 14) { ext <<= linbits; ext |= (unsigned)(x2 - 15); xbits += linbits; x2 = 15; }
        xlen = 16;
      }
      if (x2 != 0) { ext <<= 1; if (QNEG(i + 1)) ext++; cbits--; }
      const int idx = x1 * xlen + x2;
      xbits -= cbits;
      cbits += __ldg(&g_huff_len[c_huff_off[tb] + idx]);
      if (pass == 0) mybits += cbits + xbits;
      else {
        put_bits(buf, at, __ldg(&g_huff_code[c_huff_off[tb] + idx]), cbits);
        put_bits(buf, at + cbits, ext, xbits);
        at += cbits + xbits;
      }
    }
  }
  const int big_bits = wsum(mybits);
  pos += big_bits;
  /* count1 quadruples */
  const int nquads = (gi->count1 - bigv) >> 2;
  const int perq = (nquads + 31) >> 5;
  const int q0 = lane * perq, q1 = min(nquads, q0 + perq);
  const int tb = gi->count1table_select + 32;
  mybits = 0;
#pragma unroll 1
  for (int pass = 0; pass < 2; pass++) {
    int at = 0;
    if (pass == 1) {
      int incl = mybits;
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(Q_FULL, incl, o); if (lane >= o) incl += v; }
      at = pos + incl - mybits;
    }
#pragma unroll 1
    for (int q = q0; q < q1; q++) {
      const int i = bigv + 4 * q;
      int huffbits = 0, p = 0;
      if (ixq[i] != 0) { p += 8; if (QNEG(i)) huffbits++; }
      if (ixq[i + 1] != 0) { p += 4; huffbits *= 2; if (QNEG(i + 1)) huffbits++; }
      if (ixq[i + 2] != 0) { p += 2; huffbits *= 2; if (QNEG(i + 2)) huffbits++; }
      if (ixq[i + 3] != 0) { p++; huffbits *= 2; if (QNEG(i + 3)) huffbits++; }
      const int len = __ldg(&g_huff_len[c_huff_off[tb] + p]);
      if (pass == 0) mybits += len;
      else { put_bits(buf, at, (unsigned)huffbits + __ldg(&g_huff_code[c_huff_off[tb] + p]), len); at += len; }
    }
  }
  __syncwarp();
}

/* writeheader (BitStream.js:218-229): n bits of val at bit pos, byte by byte, each byte OR-ed with ((val >> j) << shift)
 * truncated to 8 bits -- val is not masked to n bits, so a value that does not fit its field (part2_3_length + part2_length
 * above 4095 in a 12-bit field, which an LSF granule of loud input can reach) sets bits of the fields before it in the same
 * byte, as lamejs's bytes show */
__device__ __forceinline__ void put_header_bits(unsigned int* buf, int pos, int val, int n) {
  while (n > 0) {
    const int k = min(n, 8 - (pos & 7));
    n -= k;
    const unsigned byte = ((unsigned)(val >> n) << (8 - (pos & 7) - k)) & 0xffu;
    const int b = pos >> 3;
    atomicOr(&buf[b >> 2], byte << (24 - 8 * (b & 3)));
    pos += k;
  }
}

/* header + side info (encodeSideInfo2, BitStream.js:259-426, MPEG-1) by one thread */
/* fin: the frame's four (two) finished GranuleInfoDev in HBM, [gr * nch + ch]; scfsi: [ch][4] */
__device__ __noinline__ void pack_sideinfo(const Mp3Tables* T, unsigned int* buf, const GranuleInfoDev* __restrict__ fin,
                                           const int* scfsi, int padding) {
  int p = 0;
#define WH(v, n) do { put_header_bits(buf, p, (int)(v), (n)); p += (n); } while (0)
  const int nch = T->nch;
  WH(T->mpeg25 ? 0xffe : 0xfff, 12); WH(T->version, 1); WH(4 - 3, 2); WH(1, 1);
  WH(T->bitrate_index, 4); WH(T->samplerate_index, 2); WH(padding, 1); WH(0, 1);
  WH(T->mono ? 3 : 0, 2); WH(0, 2); WH(0, 1); WH(1, 1); WH(0, 2);
  if (T->version == 1) {
    WH(0, 9);
    WH(0, nch == 2 ? 3 : 5);
#pragma unroll 1
    for (int ch = 0; ch < nch; ch++) for (int b = 0; b < 4; b++) WH(scfsi[ch * 4 + b], 1);
  } else {
    WH(0, 8);                       /* main_data_begin */
    WH(0, nch);                     /* private bits */
  }
#pragma unroll 1
  for (int gr = 0; gr < T->mode_gr; gr++) for (int ch = 0; ch < nch; ch++) {
    const GranuleInfoDev* gi = &fin[gr * nch + ch];
    WH(gi->part2_3_length + gi->part2_length, 12);
    WH(gi->big_values / 2, 9);
    WH(gi->global_gain, 8);
    WH(gi->scalefac_compress, T->version == 1 ? 4 : 9);
    int ts0 = gi->table_select[0], ts1 = gi->table_select[1], ts2 = gi->table_select[2];
    if (ts0 == 14) ts0 = 16;
    if (ts1 == 14) ts1 = 16;
    if (gi->block_type != BT_NORM) {
      WH(1, 1); WH(gi->block_type, 2); WH(0, 1);
      WH(ts0, 5); WH(ts1, 5);
      WH(gi->subblock_gain[0], 3); WH(gi->subblock_gain[1], 3); WH(gi->subblock_gain[2], 3);
    } else {
      WH(0, 1);
      if (ts2 == 14) ts2 = 16;
      WH(ts0, 5); WH(ts1, 5); WH(ts2, 5);
      WH(gi->region0_count, 4); WH(gi->region1_count, 3);
    }
    if (T->version == 1) WH(gi->preflag, 1);
    WH(gi->scalefac_scale, 1); WH(gi->count1table_select, 1);
  }
#undef WH
}

/* on_pe with the reservoir disabled (QuantizePVT.js:421-484 + Reservoir.js:190-229): gr0 gets mean_bits, gr1 additionally
 * what gr0 left over; per channel trunc(tbits / nch), capped at 4095, rescaled if the pair exceeds 7680; PE never matters
 * because extra_bits == 0.  Returns targ_bits of channel `ch` (every lane computes the same value). */
__device__ __forceinline__ int granule_budget(int nch, int mean_bits, int gr, int used0, int used1, int ch) {
  int tbits = mean_bits;
  if (gr == 1) {
    const int resv = -(used0 + (nch == 2 ? used1 : 0)) + mean_bits;   /* ResvSize + mean_bits */
    if (resv * 10 > 0) tbits += resv;
  }
  double t = (double)tbits / nch;
  if (t > 4095) t = 4095;
  int targ = (int)t;                      /* the same value for every channel */
  const int bits = targ * nch;
  if (bits > 7680) { targ = targ * 7680; targ = (int)((double)targ / bits); }
  (void)ch;
  return targ;
}

/* ---- the quantizer pipeline ---------------------------------------------------------------------------------------
 * One frame's four granule-channels depend on each other only through a few scalars (gr1's bit budget needs the bits both
 * channels spent in gr0; bin_search_StepSize starts at the gain the previous granule of the channel ended with), so the
 * rate loop is cut into phases, each its own kernel over ALL frames of the batch:
 *     k_q_prepare            init_outer_loop + analog silence + init_xrpow + calc_xmin       task = granule-channel
 *     k_q_search  (gr0)      bin_search_StepSize                                             task = (frame, channel)
 *     k_q_outer   (gr0)      noise-shaping loop + iteration_finish_one                       task = (frame, channel)
 *     k_q_search  (gr1), k_q_outer (gr1)
 *     k_q_pack               format_bitstream                                                task = frame
 * A task is one warp; warps pull tasks from an atomic counter (persistent blocks), so uneven loop counts balance at warp
 * granularity and no warp ever waits for another.  Code run once per task stays out of the rate loop's kernel (the single
 * fused kernel of round 1 had a 135 KB body and was instruction-fetch bound; code bytes per kernel: DESIGN.md §4) and all
 * warps run the same few loops.  The hand-over (prepared xr / xrpow rows, the quantised lines, side info) goes through HBM/L2: ~20 KB per
 * granule-channel per pass against ~35 k warp instructions of work. */
#ifndef Q_WARPS
#define Q_WARPS 4
#endif
#ifndef Q_BLOCKS_PER_SM
#define Q_BLOCKS_PER_SM 7     /* k_q_outer with its rate loop inlined: 72 registers, no stack.  C2 on an H100 80GB HBM3 (700 W), k_q_outer
                                 * 6 / 7 blocks -> 2.012 / 1.939 ms per step (the call-based loop: 80 registers and an 80-byte frame at 6) */
#endif
#define Q_THREADS (32 * Q_WARPS)

__device__ __forceinline__ int next_task(int* counter) {
  int t = 0;
  if (LANE == 0) t = atomicAdd(counter, 1);
  return __shfl_sync(Q_FULL, t, 0);
}
template <int STRIDE = (int)sizeof(WarpShared)>
__device__ __forceinline__ WarpShared* warp_shared() {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  return reinterpret_cast<WarpShared*>(smem_raw + (threadIdx.x >> 5) * STRIDE);
}
/* init_outer_loop's scalar part (Quantize.js:204-260) for the search / rate-loop kernels, from what k_q_prepare kept */
__device__ __forceinline__ void gi_init_w(GranuleInfoDev* gi, const GcPrep* __restrict__ pr) {
  __syncwarp();
  int* w = reinterpret_cast<int*>(gi);
#pragma unroll 1
  for (int i = LANE; i < (int)(sizeof(GranuleInfoDev) / 4); i += 32) w[i] = 0;
  __syncwarp();
  if (LANE == 0) {
    const int bt = pr->block_type;
    const bool is_short = bt == BT_SHORT;
    gi->global_gain = 210; gi->block_type = bt;
    gi->sfb_lmax = is_short ? 0 : 21; gi->sfb_smin = is_short ? 0 : 12; gi->psy_lmax = is_short ? 0 : 21;
    gi->psymax = is_short ? 36 : 21; gi->sfbmax = is_short ? 36 : 21; gi->sfbdivide = is_short ? 18 : 11;
    gi->max_nonzero_coeff = pr->mnz; gi->xrpow_max = pr->xrpow_max;
  }
  __syncwarp();
}
__device__ __forceinline__ void copy_row16_w(void* dst, const void* src, int nbytes) {   /* 16-byte vectors, coalesced */
  __syncwarp();
  const int n = nbytes >> 4;                       /* 144 (a 576-float row) or 72 (a 576-short row) */
  int4 v[5];
#pragma unroll
  for (int k = 0; k < 5; k++) { const int i = LANE + 32 * k; if (i < n) v[k] = reinterpret_cast<const int4*>(src)[i]; }   /* all loads in flight */
#pragma unroll
  for (int k = 0; k < 5; k++) { const int i = LANE + 32 * k; if (i < n) reinterpret_cast<int4*>(dst)[i] = v[k]; }
  __syncwarp();
}
struct FrameGeom { int z, f, padding, frame_bytes, mean_bits; long long kabs; };
__device__ __forceinline__ FrameGeom frame_geom(const Mp3Tables* T, const StreamDesc* streams, const QuantFrameState* q) {
  FrameGeom g;
  g.z = q->stream; g.f = q->rel_frame;
  g.kabs = (long long)streams[g.z].frame0 + g.f;
  g.padding = (int)(pad_count(g.kabs, T->frac_SpF, T->samplerate) - pad_count(g.kabs - 1, T->frac_SpF, T->samplerate));
  g.frame_bytes = T->frame_bytes_nopad + g.padding;
  g.mean_bits = (8 * g.frame_bytes - T->sideinfo_len * 8) / T->mode_gr;   /* Reservoir.js:83 (exact: a multiple of 4 / of 8) */
  return g;
}

/* ---- phase 1: everything of a granule-channel that does not depend on the bit budget ---- */
__global__ void __launch_bounds__(Q_THREADS, Q_BLOCKS_PER_SM)
k_q_prepare(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, const float* __restrict__ xr,
            const PsyRatioDev* __restrict__ ratio, const signed char* __restrict__ bt_final, const double* __restrict__ ath_q,
            const QuantFrameState* __restrict__ qs, float* __restrict__ xrq, float* __restrict__ xrpow_g, unsigned* __restrict__ neg_g,
            GcPrep* __restrict__ prep,
            int nframes, int* __restrict__ counter) {
  WarpShared* ws = warp_shared();
  GcWork* wk = &ws->wk;
  const int lane = LANE, nch = T->nch;
  const int G = T->mode_gr;
  const int ntasks = nframes * G * nch;
#pragma unroll 1
  for (int t = next_task(counter); t < ntasks; t = next_task(counter)) {
    const int frow = t / (G * nch), rem = t - frow * G * nch, gr = rem / nch, ch = rem - gr * nch;
    const QuantFrameState* q = qs + frow;
    const int z = q->stream, f = q->rel_frame;
    const StreamDesc& sd = streams[z];
    const double ath_adjust = ath_q[frow];
    const size_t urow = (size_t)sd.unit_base + G * f + gr, gidx = urow * nch + ch;
    const int bt = bt_final[urow * 2 + ch];
    /* masking of psy unit (G f + gr - 1): halo-shifted row = unit_base + z + (G f + gr - 1) + 1 */
    const PsyRatioDev* rt = ratio + ((size_t)sd.unit_base + z + G * f + gr) * nch + ch;
    __syncwarp();
    if (lane < 6) ws->ath[lane] = ath_adjust_dev(ath_adjust, (double)(bt == BT_SHORT ? T->ath_psfb12[lane] : T->ath_psfb21[lane]), T->ath_floor);
    __syncwarp();
    const bool have = gc_prepare_w(T, wk, ws->ath, xr + gidx * 576, bt, rt, ath_adjust);
    copy_row16_w(xrq + gidx * 576, wk->xr, 2304);
    {   /* the packer needs only the signs: 18 words instead of the 2304-byte row */
      unsigned mine = 0;
#pragma unroll 1
      for (int k = 0; k < 18; k++) { const unsigned m = __ballot_sync(Q_FULL, wk->xr[lane + 32 * k] < 0.0f); if (lane == k) mine = m; }
      if (lane < 18) neg_g[gidx * 18 + lane] = mine;
    }
    copy_row16_w(xrpow_g + gidx * 576, wk->xrpow, 2304);
    GcPrep* pr = prep + gidx;
#pragma unroll 1
    for (int i = lane; i < MP3_SFBMAX; i += 32) pr->xmin[i] = wk->xmin[i];
    if (lane == 0) { pr->have = have ? 1 : 0; pr->mnz = wk->b.max_nonzero_coeff; pr->block_type = bt; pr->xrpow_max = wk->b.xrpow_max; }
  }
}

/* ---- phase 2/4: bin_search_StepSize of granule `gr` for every (frame, channel) of the work list ----
 * revalidate = 0: first pass over all frames (in-state of frames other than a stream's first is a guess).
 * revalidate = 1: frames listed by k_qstate_verify, whose true in-state is now known.  The in-state enters a frame only
 * through the two searches: gr0 starts at (OldValue, CurrentStep); gr1 starts at gr0's gain with the step derived from where
 * gr0 started.  If gr0 lands on the recorded gain with the same cod_info fingerprint, its bytes and the bits it spent stand;
 * gr1's search is then re-run only if its start step changed, and stands if it lands on the recorded gain too.  Whatever
 * does not stand is flagged in q->redo for the rate-loop and pack kernels of this pass. */
__global__ void __launch_bounds__(Q_THREADS, Q_SLIM_BLOCKS)
k_q_search(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, QuantFrameState* __restrict__ qs,
           GranuleInfoDev* __restrict__ ginfo, short* __restrict__ l3enc, const float* __restrict__ xrpow_g,
           const GcPrep* __restrict__ prep, int gr, const int* __restrict__ list, const int* __restrict__ count_ptr, int count_direct,
           int revalidate, int* __restrict__ counter, int* __restrict__ list2, int* __restrict__ count2,
           int* __restrict__ list3, int* __restrict__ count3) {
  WarpShared* ws = warp_shared<Q_STRIDE_NOXR>();
  GcWork* wk = &ws->wk;
  const int lane = LANE, nch = T->nch;
  const int ntasks = (count_ptr ? *count_ptr : count_direct) * nch;
#pragma unroll 1
  for (int t = next_task(counter); t < ntasks; t = next_task(counter)) {
    const int wi = t / nch, ch = t - wi * nch;
    const int frow = list ? list[wi] : wi;
    QuantFrameState* q = qs + frow;
    /* revalidate: 0 first pass; 1 re-validation (gr1: channels whose start step changed, both channels when gr0 was redone);
     * 3 = gr1 of the frames whose gr0 stands (the frames with a redone gr0 are on the repair list, handled on its stream) */
    const int flags = revalidate ? q->redo : 0;
    if (revalidate == 3 && (flags & Q_R0_ANY)) continue;
    if (revalidate && gr == 1 && !(flags & (Q_R0_ANY | Q_R1S(ch)))) continue;
    const FrameGeom fg = frame_geom(T, streams, q);
    const StreamDesc& sd = streams[fg.z];
    const size_t urow = (size_t)sd.unit_base + T->mode_gr * fg.f + gr, gidx = urow * nch + ch;
    const int targ = granule_budget(nch, fg.mean_bits, gr, q->used0[0], q->used0[1], ch);
    int ov = gr == 0 ? q->in_old[ch] : q->bs_gain0[ch];
    int cs = gr == 0 ? q->in_step[ch] : q->bs_step0[ch];
    const GcPrep* pr = prep + gidx;
    const bool have = pr->have != 0;
    gi_init_w(&wk->b, pr);
    if (lane == 0) wk->geo = &T->geo[pr->block_type == BT_SHORT ? 1 : 0];
    unsigned long long h = 0;
    if (have) {
      copy_row16_w(wk->xrpow, xrpow_g + gidx * 576, 2304);
      QSTAT(revalidate ? 12 + gr : 11);
      bin_search_w(T, wk, targ, &ov, &cs, revalidate ? 2 + 2 * gr : 0);
      h = gi_hash(&wk->b);
    } else {
      __syncwarp();
#pragma unroll 1
      for (int i = lane; i < 288; i += 32) reinterpret_cast<unsigned*>(wk->ixw)[i] = 0;
      __syncwarp();
    }
    bool store;
    if (!revalidate) {
      store = true;
      /* a frame encoded from a guessed in-state also guesses the step gr1's search starts with: 2, what a stationary
       * signal produces (the formula would give 4 whenever the guessed start lies 4 above the landing gain); the value
       * used is recorded, and re-validation re-runs gr1's search only when the true step differs from it */
      if (gr == 0 && fg.f != 0 && T->mode_gr == 2) cs = Q_SPEC_GR1_STEP;
      if (lane == 0) {
        q->bs_hash[gr][ch] = h;
        if (gr == 0) { q->bs_gain0[ch] = ov; q->bs_step0[ch] = cs; }
        if (gr == T->mode_gr - 1) { q->out_old[ch] = ov; q->out_step[ch] = cs; }   /* the frame's last granule leaves the out-state */
      }
    } else if (gr == 0) {
      store = ov != q->bs_gain0[ch] || h != q->bs_hash[0][ch];
      const bool step_changed = cs != q->bs_step0[ch];
      __syncwarp();
      if (lane == 0) {
        int old = -1;
        if (T->mode_gr == 1) { q->out_old[ch] = ov; q->out_step[ch] = cs; }   /* LSF: gr0 is the frame's last granule */
        if (store) {
          q->bs_gain0[ch] = ov; q->bs_step0[ch] = cs; q->bs_hash[0][ch] = h; old = atomicOr(&q->redo, Q_R0(ch));
          if ((old & Q_R0_ANY) == 0) list3[atomicAdd(count3, 1)] = frow;     /* repair list: gr0 must be redone (a handful) */
        } else if (step_changed && T->mode_gr == 2) { q->bs_step0[ch] = cs; old = atomicOr(&q->redo, Q_R1S(ch)); }
        /* frames with anything left to do go on the short list the remaining kernels of this pass walk */
        if (old == 0) list2[atomicAdd(count2, 1)] = frow;
      }
    } else {
      store = (flags & Q_R0_ANY) || ov != q->out_old[ch] || h != q->bs_hash[1][ch];
      __syncwarp();
      if (lane == 0) {
        q->out_step[ch] = cs;
        if (store) { q->out_old[ch] = ov; q->bs_hash[1][ch] = h; atomicOr(&q->redo, Q_R1(ch)); }
      }
    }
    if (store) {
      copy_row16_w(l3enc + gidx * 576, wk->ixw, 1152);
      copy_gi_w(&ginfo[gidx], &wk->b);
    }
  }
}

/* ---- phase 3/5: noise-shaping loop (outer_loop after its search) + iteration_finish_one of granule `gr` ---- */
__global__ void __launch_bounds__(Q_THREADS, Q_BLOCKS_PER_SM)
k_q_outer(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, QuantFrameState* __restrict__ qs,
          GranuleInfoDev* __restrict__ ginfo, short* __restrict__ l3enc, const float* __restrict__ xrq,
          const float* __restrict__ xrpow_g, const GcPrep* __restrict__ prep, int gr, const int* __restrict__ list,
          const int* __restrict__ count_ptr, int count_direct, int revalidate, int* __restrict__ counter) {
  WarpShared* ws = warp_shared();
  GcWork* wk = &ws->wk;
  const int lane = LANE, nch = T->nch;
  const int ntasks = (count_ptr ? *count_ptr : count_direct) * nch;
#pragma unroll 1
  for (int t = next_task(counter); t < ntasks; t = next_task(counter)) {
    const int wi = t / nch, ch = t - wi * nch;
#ifdef Q_REVERSE
    const int frow = list ? list[wi] : (ntasks / nch - 1 - wi);
#else
    const int frow = list ? list[wi] : wi;
#endif
    QuantFrameState* q = qs + frow;
    /* revalidate: 0 every listed frame; 1 only what the re-validating searches flagged; 2 every channel of the listed
     * frames; -1 all frames except those on the repair list (gr0 redone: their gr1 runs on the repair stream) */
    if (revalidate == 1 && !(q->redo & (gr == 0 ? Q_R0(ch) : Q_R1(ch)))) continue;
    if (revalidate == -1 && (q->redo & Q_R0_ANY)) continue;
    if (revalidate > 0) QSTAT(14);
    const FrameGeom fg = frame_geom(T, streams, q);
    const StreamDesc& sd = streams[fg.z];
    const size_t urow = (size_t)sd.unit_base + T->mode_gr * fg.f + gr, gidx = urow * nch + ch;
    const int targ = granule_budget(nch, fg.mean_bits, gr, q->used0[0], q->used0[1], ch);
    const GcPrep* pr = prep + gidx;
    const bool have = pr->have != 0;
    short* const ixrow = l3enc + gidx * 576;
    __syncwarp();
    if (lane == 0) { wk->geo = &T->geo[pr->block_type == BT_SHORT ? 1 : 0]; wk->ixg = ixrow; }
    copy_gi_w(&wk->b, &ginfo[gidx]);
    copy_row16_w(wk->ixw, ixrow, 1152);
#ifdef Q_TASKSTAT
    const long long ts_t0 = clock64();
    const int ts_gain = wk->b.global_gain, ts_bits = wk->b.part2_3_length;
#endif
    if (have) {
      copy_row16_w(wk->xr, xrq + gidx * 576, 2304);
      copy_row16_w(wk->xrpow, xrpow_g + gidx * 576, 2304);
#pragma unroll 1
      for (int i = lane; i < MP3_SFBMAX; i += 32) wk->xmin[i] = pr->xmin[i];
      __syncwarp();
      outer_loop_w(T, wk, targ);
    }
#ifdef Q_TASKSTAT
    if (lane == 0 && revalidate <= 0 && gidx < (1u << 16)) {
      int* r = g_taskstat[gidx];
      r[0] = (int)((clock64() - ts_t0) >> 6); r[1] = gr; r[2] = wk->b.max_nonzero_coeff; r[3] = wk->b.block_type;
      r[4] = ts_gain; r[5] = ts_bits; r[6] = targ; r[7] = wk->b.global_gain;
    }
#endif
    copy_gi_w(&ginfo[gidx], &wk->b);
    copy_row16_w(ixrow, wk->ixw, 1152);
  }
}

/* ---- iteration_finish_one (Quantize.js:1059-1078) of granule `gr`: best_scalefac_store (+ scfsi in gr1) and
 * best_huffman_divide.  Needs only the quantised lines and the side info; its 25 KB of code stay out of the rate loop's
 * instruction-cache footprint. ---- */
__global__ void __launch_bounds__(Q_THREADS, Q_SLIM_BLOCKS)
k_q_finish(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, QuantFrameState* __restrict__ qs,
           GranuleInfoDev* __restrict__ ginfo, short* __restrict__ l3enc, int gr, const int* __restrict__ list,
           const int* __restrict__ count_ptr, int count_direct, int revalidate, int* __restrict__ counter) {
  WarpShared* ws = warp_shared<Q_STRIDE_NOXR>();
  GcWork* wk = &ws->wk;
  const int lane = LANE, nch = T->nch;
  const int ntasks = (count_ptr ? *count_ptr : count_direct) * nch;
#pragma unroll 1
  for (int t = next_task(counter); t < ntasks; t = next_task(counter)) {
    const int wi = t / nch, ch = t - wi * nch;
    const int frow = list ? list[wi] : wi;
    QuantFrameState* q = qs + frow;
    if (revalidate == 1 && !(q->redo & (gr == 0 ? Q_R0(ch) : Q_R1(ch)))) continue;
    if (revalidate == -1 && (q->redo & Q_R0_ANY)) continue;
    const StreamDesc& sd = streams[q->stream];
    const size_t urow = (size_t)sd.unit_base + T->mode_gr * q->rel_frame + gr, gidx = urow * nch + ch;
    short* const ixrow = l3enc + gidx * 576;
    copy_gi_w(&wk->b, &ginfo[gidx]);
    copy_row16_w(wk->ixw, ixrow, 1152);
    if (lane == 0) wk->geo = &T->geo[wk->b.block_type == BT_SHORT ? 1 : 0];
    __syncwarp();
    best_scalefac_store_w(wk, ws->scfsi, gr == 1 ? &ginfo[gidx - nch] : nullptr, gr, T->mode_gr);
    best_huffman_divide_w(T, wk);
    copy_gi_w(&ginfo[gidx], &wk->b);
    if (gr == 0) { if (lane == 0) q->used0[ch] = wk->b.part2_3_length + wk->b.part2_length; }
    else if (lane < 4) q->scfsi[ch][lane] = ws->scfsi[lane];
  }
}

/* ---- phase 6: format_bitstream (BitStream.js:836-901): side info, main data, ancillary stuffing, one warp per frame ---- */
struct __align__(16) PackShared {
  unsigned int bits[368];         /* frame bit buffer (<= 1441 bytes), filled with shared-memory atomic ORs */
  short ix[576];
  unsigned neg[20];               /* sign mask of the spectrum (18 words used) */
  GranuleInfoDev gi;
  int scfsi[8];
};
__global__ void __launch_bounds__(Q_THREADS)
k_q_pack(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, QuantFrameState* __restrict__ qs,
         const GranuleInfoDev* __restrict__ ginfo, const short* __restrict__ l3enc, const unsigned* __restrict__ neg_g,
         const int* __restrict__ list, const int* __restrict__ count_ptr, int count_direct, int revalidate,
         int* __restrict__ counter, uint8_t* __restrict__ out, int* __restrict__ over_budget) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PackShared* ps = reinterpret_cast<PackShared*>(smem_raw) + (threadIdx.x >> 5);
  const int lane = LANE, nch = T->nch;
  const int ntasks = count_ptr ? *count_ptr : count_direct;
#pragma unroll 1
  for (int t = next_task(counter); t < ntasks; t = next_task(counter)) {
    const int frow = list ? list[t] : t;
    QuantFrameState* q = qs + frow;
    if (revalidate && !(q->redo & (Q_R0_ANY | Q_R1_ANY))) continue;
    if (revalidate) QSTAT(5);
    const FrameGeom fg = frame_geom(T, streams, q);
    const StreamDesc& sd = streams[fg.z];
    const size_t g0 = ((size_t)sd.unit_base + T->mode_gr * fg.f) * nch;   /* first of the frame's mode_gr * nch granule-channels */
    /* A frame whose granules do not fit its slot is not packed (nothing is written past ps->bits): lamejs throws there
     * (format_bitstream's consistency check, BitStream.js:856-885).  *over_budget counts the frames whose latest pack was
     * refused (q->valid == 2), so a frame a re-validation pass repacks within budget takes its count back. */
    int used = 0;
#pragma unroll 1
    for (int k = 0; k < T->mode_gr * nch; k++) used += ginfo[g0 + k].part2_3_length + ginfo[g0 + k].part2_length;
    const bool over = used > 8 * (fg.frame_bytes - T->sideinfo_len);
    if (lane == 0 && over != (q->valid == 2)) atomicAdd(over_budget, over ? 1 : -1);
    if (over) { if (lane == 0) q->valid = 2; continue; }
    __syncwarp();
#pragma unroll 1
    for (int i = lane; i < 368; i += 32) ps->bits[i] = 0;
    if (lane < 8) ps->scfsi[lane] = q->scfsi[lane >> 2][lane & 3];
    __syncwarp();
    int pos = 8 * T->sideinfo_len;
#pragma unroll 1
    for (int k = 0; k < T->mode_gr * nch; k++) {                     /* gr0ch0, gr0ch1, gr1ch0, gr1ch1 back to back */
      copy_gi_w(&ps->gi, &ginfo[g0 + k]);
      copy_row16_w(ps->ix, l3enc + (g0 + k) * 576, 1152);
      if (lane < 18) ps->neg[lane] = neg_g[(g0 + k) * 18 + lane];
      __syncwarp();
      pack_gc_w(T, ps->bits, &ps->gi, ps->ix, ps->neg, pos);
      pos += ps->gi.part2_3_length + ps->gi.part2_length;
      __syncwarp();
    }
    if (lane == 0) {
      pack_sideinfo(T, ps->bits, ginfo + g0, ps->scfsi, fg.padding);
      /* drain_into_ancillary (BitStream.js:175-213): "LAME" + the version string pushed through `>>` as numbers */
      int remaining = 8 * fg.frame_bytes - pos;
      const unsigned char tag[10] = {0x4c, 0x41, 0x4d, 0x45, 3, 0, 9, 8, 0, 4};
      int k = 0;
      for (; k < 4 && remaining >= 8; k++) { put_bits(ps->bits, pos, tag[k], 8); pos += 8; remaining -= 8; }
      if (remaining >= 32) for (; k < 10 && remaining >= 8; k++) { put_bits(ps->bits, pos, tag[k], 8); pos += 8; remaining -= 8; }
    }
    __syncwarp();
    /* store the frame (big-endian bit order -> bytes) at its closed-form offset */
    const long long off = sd.out_base + (long long)fg.f * T->frame_bytes_nopad +
                          (pad_count(fg.kabs - 1, T->frac_SpF, T->samplerate) - pad_count((long long)sd.frame0 - 1, T->frac_SpF, T->samplerate));
    uint8_t* dst = out + off;
#pragma unroll 1
    for (int i = lane; i < fg.frame_bytes; i += 32) dst[i] = (uint8_t)(ps->bits[i >> 2] >> (24 - 8 * (i & 3)));
    if (lane == 0) q->valid = 1;
  }
}

/* qstate init: one thread per frame row */
__global__ void k_qstate_init(const StreamDesc* __restrict__ streams, int nstreams, QuantFrameState* __restrict__ qs) {
  const int z = blockIdx.y;
  const StreamDesc sd = streams[z];
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= sd.nframes) return;
  QuantFrameState* q = qs + sd.frame_base + f;
  q->stream = z; q->rel_frame = f; q->valid = 0; q->redo = 0;
#pragma unroll 1
  for (int c = 0; c < 2; c++) {
    /* first frame: the stream's true state; others: speculation (re-validated afterwards).  The speculative search
     * starts with a step of Q_SPEC_STEP -- a real state only ever holds 2 or 4 -- so that it brackets the target in a
     * few big strides and then halves down to 1, landing where the search from the true state lands. */
    q->in_old[c] = f == 0 ? sd.old_value[c] : Q_SPEC_START;
    q->in_step[c] = f == 0 ? sd.current_step[c] : Q_SPEC_STEP;
    q->out_old[c] = q->out_step[c] = 0;
    q->used0[c] = 0; q->bs_gain0[c] = q->bs_step0[c] = 0;
    for (int b = 0; b < 4; b++) q->scfsi[c][b] = 0;
  }
}

/* compare each frame's assumed in-state with its predecessor's out-state; append mismatches to the work list */
/* predict_step (LSF, first verification only): the predecessor's out-step was computed from ITS guessed start; the step it
 * will have once it is re-searched from its true start (its own predecessor's gain) is (start - gain >= 4) ? 4 : 2 if its gain
 * stands -- hand that to the successor right away instead of discovering it one pass later.  A wrong prediction is caught by
 * the next verification like any other wrong guess. */
__global__ void k_qstate_verify(const StreamDesc* __restrict__ streams, QuantFrameState* __restrict__ qs, long long nframes,
                                int* __restrict__ list, int* __restrict__ counter, int predict_step) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nframes) return;
  QuantFrameState* q = qs + r;
  if (q->rel_frame == 0) return;
  const QuantFrameState* p = q - 1;
  int pstep[2] = {p->out_step[0], p->out_step[1]};
  if (predict_step && p->rel_frame != 0) {
    const QuantFrameState* pp = p - 1;
#pragma unroll 1
    for (int c = 0; c < 2; c++) pstep[c] = (pp->out_old[c] - p->out_old[c] >= 4) ? 4 : 2;
  }
  bool same = true;
#pragma unroll 1
  for (int c = 0; c < 2; c++) if (q->in_old[c] != p->out_old[c] || q->in_step[c] != pstep[c]) same = false;
  if (!same) {
#pragma unroll 1
    for (int c = 0; c < 2; c++) { q->in_old[c] = p->out_old[c]; q->in_step[c] = pstep[c]; }
    q->redo = 0;
    list[atomicAdd(counter, 1)] = (int)r;
  }
}

/* after the fixed point: hand the last frame's out-state back to the stream descriptor (streaming handles) */
__global__ void k_qstate_commit(StreamDesc* __restrict__ streams, int nstreams, const QuantFrameState* __restrict__ qs) {
  const int z = blockIdx.x * blockDim.x + threadIdx.x;
  if (z >= nstreams) return;
  StreamDesc& sd = streams[z];
  if (sd.nframes <= 0) return;
  const QuantFrameState* q = qs + sd.frame_base + sd.nframes - 1;
#pragma unroll 1
  for (int c = 0; c < 2; c++) { sd.old_value[c] = q->out_old[c]; sd.current_step[c] = q->out_step[c]; }
}

/* The fixed-point loop as a CUDA graph (QuantLoop): runs after each k_qstate_verify of the graph's WHILE body and decides
 * whether the body goes on.  st[2] counts the passes of the launch group (2 after the first pass, +1 for each re-validation
 * that found work), st[0] keeps the largest count of the call.  A count beyond max_passes (which cannot be reached: each
 * pass fixes at least the first dirty frame) stops the loop with st[1] = 1 and an empty work list, so the rest of the body
 * has nothing to do. */
__global__ void k_qstate_loop_cond(cudaGraphConditionalHandle loop, int* __restrict__ count, int* __restrict__ st, int max_passes) {
  const int n = *count;
  int passes = st[2];
  bool more = n != 0;
  if (more) passes++;
  if (passes > max_passes) { st[1] = 1; *count = 0; more = false; }
  st[2] = passes;
  if (passes > st[0]) st[0] = passes;
  cudaGraphSetConditional(loop, more ? 1u : 0u);
}

/* device buffers of the quantizer stage (owned by the Workspace) */
struct QuantBuffers {
  const float* xr; const PsyRatioDev* ratio; const signed char* bt; const double* ath_q;
  QuantFrameState* qs; GranuleInfoDev* ginfo; short* l3enc; float* xrq; float* xrpow; unsigned* neg; GcPrep* prep;
  int* over_budget;               /* frames over their bit budget (k_q_pack), [1] */
  int* list; int* counter;        /* list: 2 x (frames + 1) entries (verify list, short list); counter[0..1]: their lengths;
                                     counter[2..Q_NCOUNTERS): task counters, one per launch */
};
#define Q_NCOUNTERS 256
#define Q_REPAIR_BLOCKS 16
enum { QE_START, QE_PREP, QE_S0, QE_O0, QE_F0, QE_S1, QE_MID, QE_O1, QE_F1, QE_PK, QE_COUNT };   /* timing event slots */

/* The fixed-point loop on the device, so that no launch waits for the host: a graph of a memset (st[2] = 2) and a
 * conditional WHILE node whose body is one re-validation pass -- the counter memsets, k_qstate_verify, k_qstate_loop_cond,
 * then the searches, rate loops and finishes of the listed frames and k_q_pack, every launch taking its count from the
 * device and sized for all F frames.  quant_run launches `exec` on the main stream; when it is null it first captures and
 * instantiates the graph for this launch's shape on `capture` and hands it back in `exec`.  The graph holds the buffers'
 * addresses: the caller keeps one per shape and workspace. */
struct QuantLoop {
  cudaStream_t capture = nullptr;  /* a stream of the caller's, only captured on */
  int* st = nullptr;               /* device [3]: the call's largest pass count, fault flag, passes of this launch group */
  cudaGraphExec_t exec = nullptr;
};

static int quant_run(const Mp3Tables* dT, const Mp3Tables& hT, StreamDesc* d_streams, int S, int nstreams_with_frames, int max_frames, long long F,
                     const QuantBuffers& B, cudaStream_t st_main, cudaStream_t st_repair, cudaEvent_t ev_fork, cudaEvent_t ev_join,
                     cudaEvent_t ev_pass1, cudaEvent_t* evq, int* evq_pred, std::atomic<long long>* launches, QuantLoop& loop) {
  cudaStream_t st = st_main;       /* the launch helpers below use `st`; the repair chain temporarily points it at st_repair */
  static std::mutex attr_mu;
  static bool attr_done[64] = {};
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t smem = sizeof(WarpShared) * Q_WARPS, smem_slim = (size_t)Q_STRIDE_NOXR * Q_WARPS, smem_pack = sizeof(PackShared) * Q_WARPS;
  {
    std::lock_guard<std::mutex> lk(attr_mu);
    if (dev < 64 && !attr_done[dev]) {            /* the attribute is per device */
      if (cudaFuncSetAttribute(k_q_prepare, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -100;
      if (cudaFuncSetAttribute(k_q_search, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_slim) != cudaSuccess) return -100;
      if (cudaFuncSetAttribute(k_q_outer, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -100;
      if (cudaFuncSetAttribute(k_q_finish, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_slim) != cudaSuccess) return -100;
      if (cudaFuncSetAttribute(k_q_pack, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_pack) != cudaSuccess) return -100;
      attr_done[dev] = true;
    }
  }
  if (F <= 0) return 0;
  const int nch = hT.nch;
  int next_counter = Q_NCOUNTERS;                 /* forces the first memset */
  auto fresh_counter = [&]() -> int* {            /* a zeroed task counter for the next launch */
    if (next_counter >= Q_NCOUNTERS) { cudaMemsetAsync(B.counter + 3, 0, sizeof(int) * (Q_NCOUNTERS - 3), st); next_counter = 3; }
    return B.counter + next_counter++;
  };
  auto grid_for = [&](long long tasks, int per_sm) -> int {   /* persistent blocks, never more than the tasks need */
    long long g = (tasks + Q_WARPS - 1) / Q_WARPS, cap = (long long)sms * per_sm;
    if (g > cap) g = cap;
    return (int)(g < 1 ? 1 : g);
  };
  {
    dim3 g((max_frames + 127) / 128, S);
    k_qstate_init<<<g, 128, 0, st>>>(d_streams, S, B.qs);
    (*launches)++;
  }
  /* per-kernel timings: mark(slot) records evq[slot] and remembers which event preceded it (the launch order differs
   * between MPEG-1 and LSF streams); the caller computes span(slot) = evq[slot] - evq[pred[slot]] after the final sync */
  for (int i = 0; i < QE_COUNT; i++) evq_pred[i] = -1;
  int last_slot = -1;
  auto mark = [&](int slot) { cudaEventRecord(evq[slot], st); evq_pred[slot] = last_slot; last_slot = slot; };
  int* const prep_counter = fresh_counter();     /* (may enqueue the counter memset: keep it out of the timed span) */
  mark(QE_START);
  k_q_prepare<<<grid_for(F * hT.mode_gr * nch, Q_BLOCKS_PER_SM), Q_THREADS, smem, st>>>(dT, d_streams, B.xr, B.ratio, B.bt, B.ath_q, B.qs, B.xrq, B.xrpow, B.neg,
                                                                              B.prep, (int)F, prep_counter);
  mark(QE_PREP);
  (*launches)++;
  /* counter[0]: length of the verify list; counter[1]: length of the short list (frames a re-validation pass must touch
   * beyond gr0's search); the task counters start at 2.  A launch takes its work either from all frames (list == nullptr,
   * count on the host) or from a list whose length lives on the device (grids are sized for the worst case; persistent
   * warps leave at once when there is nothing to pull). */
  int* const list1 = B.list;                     /* frames listed by k_qstate_verify */
  int* const list2 = B.list + (F + 1);           /* short list built by the re-validating gr0 search: any flag */
  int* const list3 = B.list + 2 * (F + 1);       /* repair list: frames whose gr0 must be redone */
  auto search = [&](int gr, const int* list, const int* cptr, long long count, int reval) {
    k_q_search<<<grid_for(count * nch, Q_SLIM_BLOCKS), Q_THREADS, smem_slim, st>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, B.xrpow, B.prep, gr, list, cptr, (int)count,
                                                                             reval, fresh_counter(), list2, B.counter + 1, list3, B.counter + 2);
    (*launches)++;
  };
  int reserve_blocks = 0;          /* blocks left free for the repair stream while it runs beside the main stream */
  auto finish = [&](int gr, const int* list, const int* cptr, long long count, int reval) {
    k_q_finish<<<max(1, grid_for(count * nch, Q_SLIM_BLOCKS) - reserve_blocks), Q_THREADS, smem_slim, st>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, gr, list, cptr, (int)count, reval, fresh_counter());
    (*launches)++;
  };
  auto outer = [&](int gr, const int* list, const int* cptr, long long count, int reval) {
    k_q_outer<<<max(1, grid_for(count * nch, Q_BLOCKS_PER_SM) - reserve_blocks), Q_THREADS, smem, st>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, B.xrq, B.xrpow, B.prep, gr, list, cptr, (int)count,
                                                                            reval, fresh_counter());
    (*launches)++;
  };
  /* rate loop, then the finish phase of one granule.  (Both in one launch, the finish tasks filling the rate loop's tail behind
   * per-row completion flags, and the finish kernel as a programmatic dependent launch were measured: slower, the tail's few
   * very long tasks lose the SMs they have to themselves -- DESIGN.md 4.) */
  auto outer_finish = [&](int gr, long long count, int reval, int slot_o, int slot_f) {
    outer(gr, nullptr, nullptr, count, reval); mark(slot_o);
    finish(gr, nullptr, nullptr, count, reval); mark(slot_f);
  };
  auto pack = [&](const int* list, const int* cptr, long long count, int reval) {
    k_q_pack<<<grid_for(count, 9), Q_THREADS, smem_pack, st>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, B.neg, list, cptr, (int)count, reval, fresh_counter(), nullptr, B.over_budget);
    (*launches)++;
  };
  auto verify = [&](int predict_step = 0) {
    cudaMemsetAsync(B.counter, 0, 3 * sizeof(int), st);
    k_qstate_verify<<<(int)((F + 255) / 256), 256, 0, st>>>(d_streams, B.qs, F, list1, B.counter, predict_step);
    (*launches)++;
  };
  const int G = hT.mode_gr;
  /* every stream contributes at most its first frame of this launch (a live encoder advancing one frame per call): all
   * in-states are the true ones, nothing is speculated, nothing to verify -- no extra launches, no host round trip */
  const bool speculated = F > nstreams_with_frames;
  /* ---- first pass, with the first re-validation folded in ----
   * The out-state of every frame is known as soon as its LAST granule's search has run (it does not depend on the rate
   * loop of that granule), so the in-state assumptions are verified right there and the few frames whose searches do not
   * stand are repaired before the big rate-loop / finish / pack launches of the last granule touch them: the repair's
   * latency chain (a handful of single-warp tasks) is short and those launches then see final data.
   *   MPEG-1: S0 O0 F0 S1 | verify, S0' (listed), O0' F0' S1' (short list) | O1 F1 PACK
   *   LSF:    S0          | verify, S0' (listed)                            | O0 F0 PACK */
  search(0, nullptr, nullptr, F, 0); mark(QE_S0);
  if (G == 2) {
    outer_finish(0, F, 0, QE_O0, QE_F0);
    search(1, nullptr, nullptr, F, 0); mark(QE_S1);
  }
  bool forked = false;
  if (Q_SPEC_FOLD && speculated) {
    verify(G == 1 ? 1 : 0);
    search(0, list1, B.counter, F, 1);
    if (G == 2) {
      /* gr1's search of the frames whose gr0 stands but whose start step changed (a third of the frames on C2; cheap with
       * the whole machine): afterwards every frame but the repair list is ready for gr1's rate loop */
      search(1, list2, B.counter + 1, F, 3);
      /* The repair list (frames whose gr0 search did not stand: a handful) is redone on a second stream -- gr0 rate loop,
       * finish, gr1 search, then their whole gr1: single-warp tasks, pure latency -- while the main stream
       * runs the gr1 rate loop of all other frames. */
      int* const c0 = fresh_counter(); int* const c1 = fresh_counter(); int* const c2 = fresh_counter();
      int* const c3 = fresh_counter(); int* const c4 = fresh_counter();
      cudaEventRecord(ev_fork, st_main);
      cudaStreamWaitEvent(st_repair, ev_fork, 0);
      /* the main stream's persistent grid would occupy every block slot for a millisecond: it leaves Q_REPAIR_BLOCKS slots
       * free (under 2 % of its warps) and the repair kernels never ask for more */
      const int gq = Q_REPAIR_BLOCKS, gs = Q_REPAIR_BLOCKS;
      const int* cp = B.counter + 2;
      k_q_outer<<<gq, Q_THREADS, smem, st_repair>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, B.xrq, B.xrpow, B.prep, 0, list3, cp, (int)F, 1, c0);
      k_q_finish<<<gs, Q_THREADS, smem_slim, st_repair>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, 0, list3, cp, (int)F, 1, c1);
      k_q_search<<<gs, Q_THREADS, smem_slim, st_repair>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, B.xrpow, B.prep, 1, list3, cp, (int)F, 1, c2, list2, B.counter + 1,
                                                          list3, B.counter + 2);
      k_q_outer<<<gq, Q_THREADS, smem, st_repair>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, B.xrq, B.xrpow, B.prep, 1, list3, cp, (int)F, 2, c3);
      k_q_finish<<<gs, Q_THREADS, smem_slim, st_repair>>>(dT, d_streams, B.qs, B.ginfo, B.l3enc, 1, list3, cp, (int)F, 2, c4);
      cudaEventRecord(ev_join, st_repair);
      (*launches) += 5;
      forked = true;
    }
  }
  mark(QE_MID);
  if (G == 2) {
    reserve_blocks = forked ? Q_REPAIR_BLOCKS : 0;
    outer_finish(1, F, forked ? -1 : 0, QE_O1, QE_F1);
    reserve_blocks = 0;
    if (forked) cudaStreamWaitEvent(st_main, ev_join, 0);
  } else {
    outer_finish(0, F, 0, QE_O0, QE_F0);
  }
  pack(nullptr, nullptr, F, 0); mark(QE_PK);
  if (cudaEventRecord(ev_pass1, st) != cudaSuccess) return -100;
  /* ---- fixed point: a repaired frame may hand its successor a different in-state than the one it was verified with ----
   * The loop's graph (QuantLoop), captured here for this launch's shape when the caller has none.  Its body is one
   * re-validation pass over the frames verify() listed, as many as counter[0] says on the device (grids sized for all F). */
  if (speculated) {
    if (!loop.exec) {
      cudaGraph_t g = nullptr;
      cudaGraphConditionalHandle cond;
      cudaGraphNode_t reset, node;
      cudaMemsetParams mp = {};
      mp.dst = loop.st + 2; mp.value = 2; mp.elementSize = sizeof(int); mp.width = 1; mp.height = 1;
      cudaGraphNodeParams cp = {};
      cp.type = cudaGraphNodeTypeConditional;
      if (cudaGraphCreate(&g, 0) != cudaSuccess) return -100;
      bool ok = cudaGraphConditionalHandleCreate(&cond, g, 1, cudaGraphCondAssignDefault) == cudaSuccess &&
                cudaGraphAddMemsetNode(&reset, g, nullptr, 0, &mp) == cudaSuccess;
      cp.conditional.handle = cond; cp.conditional.type = cudaGraphCondTypeWhile; cp.conditional.size = 1;
      ok = ok && cudaGraphAddNode(&node, g, &reset, 1, &cp) == cudaSuccess;
      cudaGraph_t body = ok ? cp.conditional.phGraph_out[0] : nullptr;
      if (ok && cudaStreamBeginCaptureToGraph(loop.capture, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
        std::atomic<long long> captured{0};        /* launches are counted when the graph runs, not when it is captured */
        std::atomic<long long>* const counted = launches;
        launches = &captured;
        st = loop.capture;
        next_counter = Q_NCOUNTERS;                /* the body zeroes its own task counters */
        verify();
        k_qstate_loop_cond<<<1, 1, 0, st>>>(cond, B.counter, loop.st, max_frames + 3);
        search(0, list1, B.counter, F, 1);
        outer(0, list2, B.counter + 1, F, 1);
        finish(0, list2, B.counter + 1, F, 1);
        if (G == 2) {
          search(1, list2, B.counter + 1, F, 1);
          outer(1, list2, B.counter + 1, F, 1);
          finish(1, list2, B.counter + 1, F, 1);
        }
        pack(list2, B.counter + 1, F, 1);
        st = st_main;
        launches = counted;
        cudaGraph_t captured_body = nullptr;
        ok = cudaStreamEndCapture(loop.capture, &captured_body) == cudaSuccess && captured_body == body &&
             cudaGraphInstantiate(&loop.exec, g, 0) == cudaSuccess;
      } else {
        ok = false;
      }
      cudaGraphDestroy(g);
      if (!ok) { loop.exec = nullptr; return -100; }
    }
    if (cudaGraphLaunch(loop.exec, st) != cudaSuccess) return -100;
    (*launches)++;
  }
  k_qstate_commit<<<(S + 63) / 64, 64, 0, st>>>(d_streams, S, B.qs);
  (*launches)++;
  return 0;
}

#endif
