/* k_psy.cuh -- K2 / K3pre / K3a / K3b: psycho-acoustic model (lamejs L3psycho_anal_ns) as four kernels.
 *
 * Reference: src/js/PsyModel.js L3psycho_anal_ns :1000-1383 with compute_ffts :251-324, mask_add :403-473,
 * calc_interchannel_masking :525-543, convert_partition2scalefac_s/_l :644-734, compute_masking_s :736-782,
 * block_type_set :784-826, calc_energy :906, calc_mask_index_l :930; src/js/FFT.js fht :31-115,
 * fft_short :140-183, fft_long :185-224; src/js/Encoder.js adjust_ATH :166-243.
 *
 * lamejs runs one psy call per granule ("unit" c, analysing stream samples [576c-224, 576c+800)) and carries
 * state from call to call.  Here the work is split by what it depends on:
 *   k_psy_analysis   pure function of PCM, every unit: fs/4 HPF + 9 sub-block peaks, 1024-pt FHT, line energies,
 *                    long partition energies / tonality index
 *                    (and the ordered 512-term loudness sum, psycho_loudness_approx: terms in parallel, additions on one
 *                    thread per unit); PSY_UNITS consecutive units of one channel per block
 *   k_attack_prepass pure function of two consecutive units: attack candidates (before the lastAttacks FSM)
 *   k_stream_scan    the only sequential part: per stream, the attack / block-type FSM and the ATH-adjust IIR
 *   k_psy_short_list after the scan: the units whose short-block half is read (psy_short_read, DESIGN.md 2)
 *   k_psy_short      pure function of PCM, listed units only: 3x256-pt FHT, short partition energies, short spreading sums
 *   k_psy_masking    long-block spreading with mask_add (needs ATH.adjust), short thresholds (need the previous
 *                    block type; units whose short half is read only), partition -> scalefactor-band conversion,
 *                    inter-channel masking
 * With the reservoir disabled pcfact == 0 (PsyModel.js:1036-1038), so every NS_INTERP pre-echo branch returns
 * its second argument and nb_1/nb_2 are never read; PE (pecalc_*) feeds only dead values (SURVEY.md 7.6).
 */
#ifndef MP3B200_K_PSY_CUH
#define MP3B200_K_PSY_CUH
#include "mp3_device.cuh"
#include "mp3_tables.h"

#ifndef PSY_THREADS
#define PSY_THREADS 128     /* k_psy_short: 4 warps per (unit, channel) task */
#endif
#define MASK_THREADS 128

/* long half of a psy unit, written for every unit */
struct PsyUnit {
  float eb_l[MP3_CBANDS];
  float peaks[9];                   /* en_subshort[3..11] */
  float loudness;                   /* psycho_loudness_approx */
  unsigned char mask_idx[MP3_CBANDS];
  unsigned char attack[4];          /* pre-FSM ns_attacks[0..3] */
  unsigned char pad_;
};
/* short half, a separate array: written by k_psy_short for the units on the short list only; the other rows are stale */
struct PsyShort {
  double ecb_s[3][MP3_CBANDS];      /* short-block spreading sums (double; float32 of it is lamejs nb_s1) */
  float eb_s[3][MP3_CBANDS];
};
/* en_s / thm_s are written only for the units whose short half is read (psy_short_read); elsewhere they are stale */
struct PsyRatioDev { float en_l[22], thm_l[22], en_s[13][3], thm_s[13][3]; };

__constant__ unsigned char c_fft_rv[128];
/* indexed per lane by data: global + read-only cache instead of __constant__ (divergent constant reads serialise) */
__device__ double c_tab[9];
__device__ double c_table1[25];
__device__ double c_table2[10];
__device__ double c_table3[14];
__constant__ double c_fircoef[10];

static int psy_upload_constants() {
  static const double tab[9] = {1.0, 0.79433, 0.63096, 0.63096, 0.63096, 0.63096, 0.63096, 0.25119, 0.11749};
  static const double r1[25] = {3.3246, 3.23837, 3.15437, 3.00412, 2.86103, 2.65407, 2.46209, 2.284, 2.11879, 1.96552, 1.82335,
    1.69146, 1.56911, 1.46658, 1.37074, 1.31036, 1.25264, 1.20648, 1.16203, 1.12765, 1.09428, 1.0659, 1.03826, 1.01895, 1};
  static const double r2[10] = {1.33352, 1.35879, 1.38454, 1.39497, 1.40548, 1.3537, 1.30382, 1.22321, 1.14758, 1};
  static const double r3[14] = {2.35364, 2.29259, 2.23313, 2.12675, 2.02545, 1.87894, 1.74303, 1.61695, 1.49999, 1.39148,
    1.29083, 1.19746, 1.11084, 1.03826};
  static const double fir_half[10] = {-8.65163e-18, -0.00851586, -6.74764e-18, 0.0209036, -3.36639e-17, -0.0438162,
    -1.54175e-17, 0.0931738, -5.52212e-17, -0.313819};
  for (int j = 0; j < 128; j++) {    /* k_psy_analysis reads fft_rv[j] as 2 rev7(j) */
    int r = 0;
    for (int bit = 0; bit < 7; bit++) r |= (j >> bit & 1) << (6 - bit);
    if (MP3_FFT_RV[j] != 2 * r) return -100;
  }
  double t1[25], t2[10], t3[14], fir[10];
  for (int i = 0; i < 25; i++) t1[i] = r1[i] * r1[i];       /* PsyModel.js:378-398 spells them as x*x */
  for (int i = 0; i < 10; i++) t2[i] = r2[i] * r2[i];
  for (int i = 0; i < 14; i++) t3[i] = r3[i] * r3[i];
  for (int i = 0; i < 10; i++) fir[i] = fir_half[i] * 2;     /* PsyModel.js:994-998 */
  if (cudaMemcpyToSymbol(c_fft_rv, MP3_FFT_RV, 128) != cudaSuccess) return -100;
  if (cudaMemcpyToSymbol(c_tab, tab, sizeof tab) != cudaSuccess) return -100;
  if (cudaMemcpyToSymbol(c_table1, t1, sizeof t1) != cudaSuccess) return -100;
  if (cudaMemcpyToSymbol(c_table2, t2, sizeof t2) != cudaSuccess) return -100;
  if (cudaMemcpyToSymbol(c_table3, t3, sizeof t3) != cudaSuccess) return -100;
  if (cudaMemcpyToSymbol(c_fircoef, fir, sizeof fir) != cudaSuccess) return -100;
  return 0;
}

/* Float32 cell of the FHT work arrays.  Reading widens float32 -> double; the hardware conversion runs on the XU pipe, which
 * the round-2 profile shows 52 % busy (the limiter of k_psy_analysis), while the integer pipe idles.  PSY_ALU_WIDEN widens with
 * integer operations instead -- exact for zero and normal numbers; FHT data are products and sums of window x Int16 samples,
 * never subnormal, infinite or NaN (>= 1e-16 in magnitude or exactly 0).  Writing rounds with the hardware conversion. */
struct f32w {
  float v;
  __device__ __forceinline__ operator double() const {
#ifdef PSY_ALU_WIDEN
    const unsigned u = __float_as_uint(v);
    const unsigned hi = (u & 0x7fffffffu) ? ((u & 0x80000000u) | (((u >> 3) & 0x0fffffffu) + 0x38000000u)) : u;
    return __hiloint2double((int)hi, (int)(u << 29));
#else
    return (double)v;
  }
  __device__ __forceinline__ f32w& operator=(double d) { v = (float)d; return *this; }
};
#endif

/* ---- one butterfly task of an FHT stage (FFT.js:31-115), fz float32 in shared memory ------------------- */
/* one pad word per 16 floats: the stage-0/1 butterflies stride 16 / 64 floats across lanes (first profile: 116 M bank conflicts) */
#define FHT_PAD(i) ((i) + ((i) >> 4))
/* Stage `stage` (k1 = 4, 16, 64, 256) of an n-point transform consists of n / (8 k1) groups of kx = k1 / 2 tasks: task i = 0
 * does the group's two twiddle-free butterflies (at the group base and at base + kx), task i = 1..kx-1 the butterfly pair
 * (base + i, base + k1 - i).  Tasks per stage: n / 8 -- 128 for the 1024-point, 32 for a 256-point transform -- and group /
 * index follow from the task number by shifts (stage is a compile-time constant after unrolling). */
__device__ __forceinline__ void fht_task(f32w* fz, int stage, int task, const double* __restrict__ tw, const int* tw_off) {
  const int k1 = 4 << (2 * stage);          /* 4,16,64,256 */
  const int kx = k1 >> 1, k2 = k1 << 1, k3 = k2 + k1, k4 = k2 << 1;
  const int g = task >> (2 * stage + 1), i = task & (kx - 1);
  if (i == 0) {
    {
      const int fi = g * k4;
      double f0, f1, f2, f3;
      f1 = fz[FHT_PAD(fi + 0)] - fz[FHT_PAD(fi + k1)];
      f0 = fz[FHT_PAD(fi + 0)] + fz[FHT_PAD(fi + k1)];
      f3 = fz[FHT_PAD(fi + k2)] - fz[FHT_PAD(fi + k3)];
      f2 = fz[FHT_PAD(fi + k2)] + fz[FHT_PAD(fi + k3)];
      fz[FHT_PAD(fi + k2)] = f0 - f2;
      fz[FHT_PAD(fi + 0)] = f0 + f2;
      fz[FHT_PAD(fi + k3)] = f1 - f3;
      fz[FHT_PAD(fi + k1)] = f1 + f3;
    }
    {
      const int gi = g * k4 + kx;
      double f0, f1, f2, f3;
      f1 = fz[FHT_PAD(gi + 0)] - fz[FHT_PAD(gi + k1)];
      f0 = fz[FHT_PAD(gi + 0)] + fz[FHT_PAD(gi + k1)];
      f3 = (SQRT2_D * fz[FHT_PAD(gi + k3)]);
      f2 = (SQRT2_D * fz[FHT_PAD(gi + k2)]);
      fz[FHT_PAD(gi + k2)] = f0 - f2;
      fz[FHT_PAD(gi + 0)] = f0 + f2;
      fz[FHT_PAD(gi + k3)] = f1 - f3;
      fz[FHT_PAD(gi + k1)] = f1 + f3;
    }
    return;
  }
  const double* e = tw + 4 * (tw_off[stage] + i);
  const double c1 = e[0], s1 = e[1], c2 = e[2], s2 = e[3];
  const int fi = g * k4 + i, gi = g * k4 + k1 - i;
  double a, b, g0, f0, f1, g1, f2, g2, f3, g3;
  b = s2 * fz[FHT_PAD(fi + k1)] - c2 * fz[FHT_PAD(gi + k1)];
  a = c2 * fz[FHT_PAD(fi + k1)] + s2 * fz[FHT_PAD(gi + k1)];
  f1 = fz[FHT_PAD(fi + 0)] - a;
  f0 = fz[FHT_PAD(fi + 0)] + a;
  g1 = fz[FHT_PAD(gi + 0)] - b;
  g0 = fz[FHT_PAD(gi + 0)] + b;
  b = s2 * fz[FHT_PAD(fi + k3)] - c2 * fz[FHT_PAD(gi + k3)];
  a = c2 * fz[FHT_PAD(fi + k3)] + s2 * fz[FHT_PAD(gi + k3)];
  f3 = fz[FHT_PAD(fi + k2)] - a;
  f2 = fz[FHT_PAD(fi + k2)] + a;
  g3 = fz[FHT_PAD(gi + k2)] - b;
  g2 = fz[FHT_PAD(gi + k2)] + b;
  b = s1 * f2 - c1 * g3;
  a = c1 * f2 + s1 * g3;
  fz[FHT_PAD(fi + k2)] = f0 - a;
  fz[FHT_PAD(fi + 0)] = f0 + a;
  fz[FHT_PAD(gi + k3)] = g1 - b;
  fz[FHT_PAD(gi + k1)] = g1 + b;
  b = c1 * g2 - s1 * f3;
  a = s1 * g2 + c1 * f3;
  fz[FHT_PAD(gi + k2)] = g0 - a;
  fz[FHT_PAD(gi + 0)] = g0 + a;
  fz[FHT_PAD(fi + k3)] = f1 - b;
  fz[FHT_PAD(fi + k1)] = f1 + b;
}

/* psy row of (stream z, relative unit u >= -1): unit_base + z + u + 1 */
__device__ __forceinline__ size_t psy_row(const StreamDesc& sd, int z, int u) { return (size_t)sd.unit_base + z + u + 1; }

/* the PCM span [x0, x0 + N) widened to double (zero outside the stream), all of a thread's loads in flight at once
 * (they were one dependent HBM round trip per iteration) */
template <bool F32_PCM, int NT, int N = 1024>
__device__ __forceinline__ void psy_load_span(const Mp3Tables* __restrict__ T, const StreamDesc& sd, int ch, long long x0, double* xs) {
  using Sample = pcm_sample_t<F32_PCM>;
  const int tid = threadIdx.x;
  const int scale_applied = T->scale_applied;
  const double scale = T->scale;
  const Sample* __restrict__ pbuf = static_cast<const Sample*>(sd.pcm[ch]);
  const long long pbase = sd.pcm_base, pend = sd.pcm_end;
  constexpr int NB = (N + NT - 1) / NT;
  Sample v[NB];
#pragma unroll
  for (int k = 0; k < NB; k++) {
    const int j = tid + k * NT;
    const long long i = x0 + j;
    v[k] = (j < N && i >= 0 && i < pend) ? __ldg(&pbuf[i - pbase]) : (Sample)0;
  }
#pragma unroll
  for (int k = 0; k < NB; k++) {
    const int j = tid + k * NT;
    if (j < N) xs[j] = pcm_value(v[k], scale_applied, scale);
  }
}

/* Block shape of k_psy_analysis: PSY_UNITS consecutive units of one channel per block.  Consecutive units overlap by 448
 * of their 1024 samples, so the block loads and widens the union span (576 (U - 1) + 1024 samples) once; the FHTs and the
 * partition phases of its units share one set of barriers.  PSY_UNIT_THREADS (P) >= 64 threads per unit: unit k's
 * partitions run on threads P k .. P k + npart_l - 1, its loudness chain on thread P k + P - 1 (one warp per unit holds it,
 * idle in the partition phases when npart_l < P). */
#ifndef PSY_UNITS
#define PSY_UNITS 2
#endif
#ifndef PSY_UNIT_THREADS
#define PSY_UNIT_THREADS 64
#endif
#define PSY_A_THREADS (PSY_UNITS * PSY_UNIT_THREADS)
#ifndef PSY_MIN_BLOCKS
#define PSY_MIN_BLOCKS 8      /* 2 units x 64 threads: 58 / 64 registers (<false> / <true>), no spills, 26 112 B shared memory
                                 -> 8 blocks (32 warps) per SM.  C2 on an H100 80GB HBM3 (700 W), `psy` phase 0.458 ms; with
                                 1 unit x 128 threads, 12 blocks, 0.456 ms (DESIGN.md 6) */
#endif
static_assert(PSY_UNIT_THREADS >= 64 && PSY_UNIT_THREADS % 32 == 0, "one thread per long partition of each unit");

#ifdef PSY_PHASESTAT
/* tuning build: clock64() at the phase boundaries of every PSY_STAT_EVERY-th block of channel 0 of stream 0 (tools/psy_phasestat.py) */
#define PSY_STAT_EVERY 16
#define PSY_STAT_ROWS 4096
#define PSY_STAT_COLS 13
__device__ long long g_psystat[PSY_STAT_ROWS][PSY_STAT_COLS];
#define PSY_CLOCK(col, who) do { if (stat_row >= 0 && (who)) g_psystat[stat_row][col] = clock64(); } while (0)
#else
#define PSY_CLOCK(col, who) do { } while (0)
#endif

/* a unit belongs to the upload slice `chunk` of `nchunks` (the host uploads every stream's PCM in time slices and launches
 * this kernel once per slice as it lands) when that slice holds the last sample of its 1024-sample window */
__device__ __forceinline__ bool psy_unit_in_slice(const StreamDesc& sd, long long c, int chunk, int nchunks) {
  if (nchunks <= 1) return true;
  const long long n = sd.pcm_end - sd.pcm_base;
  long long last = 576 * c - 224 + 1023 - sd.pcm_base;
  if (last > n - 1) last = n - 1;
  int mine = 0;
  while (mine < nchunks - 1 && last >= n * (mine + 1) / nchunks) mine++;
  return mine == chunk;
}

/* grid (ceil((max_units + 1) / PSY_UNITS), nch, nstreams).  F32_PCM: sd.pcm[ch] points at Float32 samples already at the
 * encoding rate and scaled (the resampler's output, k_resample) instead of Int16 input.  Every unit of the block is
 * computed; only the units that exist and belong to this slice are written. */
template <bool F32_PCM>
__global__ void __launch_bounds__(PSY_A_THREADS, PSY_MIN_BLOCKS)
k_psy_analysis(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, PsyUnit* __restrict__ out,
               int chunk, int nchunks, int u_base) {
  constexpr int U = PSY_UNITS, NT = PSY_A_THREADS;
  const int z = blockIdx.z;
  const StreamDesc& sd = streams[z];
  const int u0 = (int)blockIdx.x * U + u_base;        /* relative unit of the block's first unit, -1 = halo */
  const int ch = blockIdx.y;
  const int nch = T->nch;
  const int nunits = T->mode_gr * sd.nframes;
  const long long c0 = (long long)T->mode_gr * sd.frame0 + u0;   /* absolute psy call index (one call per granule) */
  const int tid = threadIdx.x;
  PsyUnit* const o0 = out + psy_row(sd, z, u0) * nch + ch;        /* unit k's row: o0 + k * nch */
#ifdef PSY_PHASESTAT
  const int stat_row = (z == 0 && ch == 0 && blockIdx.x % PSY_STAT_EVERY == 0 && blockIdx.x / PSY_STAT_EVERY < PSY_STAT_ROWS)
                       ? (int)blockIdx.x / PSY_STAT_EVERY : -1;
#endif
  PSY_CLOCK(0, tid == 0);

  unsigned act = 0;                                   /* bit k: unit k is written by this block */
#pragma unroll
  for (int k = 0; k < U; k++) {
    const int u = u0 + k;
    if (u >= nunits || !psy_unit_in_slice(sd, c0 + k, chunk, nchunks)) continue;
    if (c0 + k < 0) {   /* before the first call: psymodel_init values (PsyModel.js:2573-2595) */
      PsyUnit* o = o0 + k * nch;
      if (tid < MP3_CBANDS) { o->eb_l[tid] = 0.0f; o->mask_idx[tid] = 0; }
      if (tid < 9) o->peaks[tid] = 10.0f;
      if (tid == 0) o->loudness = 0.0f;
      if (tid < 4) o->attack[tid] = 0;
      continue;
    }
    act |= 1u << k;
  }
  if (act == 0) return;

  /* Region A holds the PCM span widened once (the HPF reads each sample 21 times) and the high-pass output; the span is
   * dead after the first radix-4 pass, the high-pass output after the peaks (FHT stage 0).  From the line energies on it
   * holds, per unit: the energies fe[513], the partition max / avg, and the 512 loudness terms energy[i] * eql_w[i]
   * (double products, computed by the threads that produce the energies). */
  constexpr int SPAN = 576 * (U - 1) + 1024;
  constexpr int HP_OFF = SPAN * 8;
  constexpr int POST = 2064 + 2 * 4 * MP3_CBANDS + 512 * 8;        /* fe, s_max, s_avg, loudness terms */
  constexpr int A_BYTES = HP_OFF + U * 576 * 4 > U * POST ? HP_OFF + U * 576 * 4 : U * POST;
  static_assert(POST % 16 == 0 && (2064 + 2 * 4 * MP3_CBANDS) % 8 == 0, "per-unit layout of region A");
  __shared__ __align__(16) unsigned char s_a[A_BYTES];
  double* const xs = reinterpret_cast<double*>(s_a);
  f32s* const hp = reinterpret_cast<f32s*>(s_a + HP_OFF);                          /* unit k: hp + 576 k */
  __shared__ f32w wl[U][1024 + 64];

  psy_load_span<F32_PCM, NT, SPAN>(T, sd, ch, 576 * c0 - 224, xs);
  __syncthreads();
  PSY_CLOCK(1, tid == 0);

  /* fs/4 high-pass (PsyModel.js:1051-1069): firbuf index = bufPos + 397 + i + j; unit k's output i is q = 576 k + i.
   * Each thread computes the outputs q = 2p and 2p + 1 from the 24 samples xs[396 + 2p ..], read as 16-byte pairs: the
   * reads were 22 8-byte loads per output, and shared-memory wavefronts are what this kernel runs out of first. */
  for (int p = tid; p < U * 288; p += NT) {
    double v[24];
    const double2* src = reinterpret_cast<const double2*>(xs + 396 + 2 * p);
#pragma unroll
    for (int t = 0; t < 12; t++) { const double2 d = src[t]; v[2 * t] = d.x; v[2 * t + 1] = d.y; }
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const double* fb = v + 1 + r;
      double sum1 = fb[10], sum2 = 0.0;
#pragma unroll
      for (int j = 0; j < 9; j += 2) {
        sum1 += c_fircoef[j] * (fb[j] + fb[21 - j]);
        sum2 += c_fircoef[j + 1] * (fb[j + 1] + fb[21 - j - 1]);
      }
      hp[2 * p + r] = sum1 + sum2;
    }
  }
  /* windowing + first radix-4 pass of fft_long (FFT.js:185-224): iteration jj writes y[4jj..4jj+3], y[512+4jj..] and reads
   * the samples from i = fft_rv[jj] = 2 rev7(jj) on (psy_upload_constants checks the table).  Thread p runs iteration
   * jj = rev7(p), so that a warp reads consecutive samples and window values (in table order a warp's 32 reads of xs lie
   * multiples of 64 bytes apart, in two pairs of banks) and writes y conflict-free (x = 4 jj spreads over the padded banks). */
  for (int q = tid; q < U * 128; q += NT) {
    const int k = q >> 7, p = q & 127, jj = (int)(__brev((unsigned)p) >> 25);
    const int i = 2 * p, x = 4 * jj;
    const float* w = T->fft_window;
    const double* xu = xs + 576 * k;
    f32w* const y = wl[k];
    double f0, f1, f2, f3, wv;
    f0 = (double)w[i] * (double)xu[i];
    wv = (double)w[i + 0x200] * (double)xu[i + 0x200];
    f1 = f0 - wv; f0 = f0 + wv;
    f2 = (double)w[i + 0x100] * (double)xu[i + 0x100];
    wv = (double)w[i + 0x300] * (double)xu[i + 0x300];
    f3 = f2 - wv; f2 = f2 + wv;
    y[FHT_PAD(x + 0)] = f0 + f2; y[FHT_PAD(x + 2)] = f0 - f2; y[FHT_PAD(x + 1)] = f1 + f3; y[FHT_PAD(x + 3)] = f1 - f3;
    f0 = (double)w[i + 0x001] * (double)xu[i + 0x001];
    wv = (double)w[i + 0x201] * (double)xu[i + 0x201];
    f1 = f0 - wv; f0 = f0 + wv;
    f2 = (double)w[i + 0x101] * (double)xu[i + 0x101];
    wv = (double)w[i + 0x301] * (double)xu[i + 0x301];
    f3 = f2 - wv; f2 = f2 + wv;
    y[FHT_PAD(x + 512 + 0)] = f0 + f2; y[FHT_PAD(x + 512 + 2)] = f0 - f2; y[FHT_PAD(x + 512 + 1)] = f1 + f3; y[FHT_PAD(x + 512 + 3)] = f1 - f3;
  }
  __syncthreads();
  PSY_CLOCK(2, tid == 0);

  /* 9 sub-block peaks of the high-passed signal per unit (PsyModel.js:1125-1132): max(1, |hp|) over 64 samples each, one
   * warp per sub-block (unit k's sub-block s is sb = 9 k + s, its samples hp[64 sb ..]); the values are non-negative
   * float32, whose order is the order of their bit patterns, so a warp max of the bits is the exact max */
  for (int sb = tid >> 5; sb < 9 * U; sb += NT / 32) {
    const int lane = tid & 31;
    const unsigned m = __reduce_max_sync(0xffffffffu, max(__float_as_uint(fabsf(hp[64 * sb + lane].v)),
                                                          __float_as_uint(fabsf(hp[64 * sb + 32 + lane].v))));
    const int k = sb / 9;
    if (lane == 0 && (act >> k & 1)) o0[k * nch].peaks[sb - 9 * k] = __uint_as_float(max(m, __float_as_uint(1.0f)));
  }
  /* FHT stages: 128 tasks per unit and stage (task numbers map to butterflies by shifts) */
#pragma unroll
  for (int stage = 0; stage < 4; stage++) {
    for (int t = tid; t < U * 128; t += NT) fht_task(wl[t >> 7], stage, t & 127, T->tw, T->tw_off);
    __syncthreads();
    PSY_CLOCK(3 + stage, tid == 0);
  }

  /* line energies (PsyModel.js:278-298) and the loudness terms */
  for (int q = tid; q < U * 512; q += NT) {
    const int k = q >> 9, j = q & 511;
    unsigned char* const pk = s_a + k * POST;
    f32s* const fe = reinterpret_cast<f32s*>(pk);
    double* const prod = reinterpret_cast<double*>(pk + 2064 + 2 * 4 * MP3_CBANDS);
    const double re = wl[k][FHT_PAD(512 - j)], im = wl[k][FHT_PAD(512 + j)];
    f32s e; e = (re * re + im * im) * 0.5;
    fe[512 - j] = (double)e;
    if (j > 0) prod[512 - j] = (double)e * (double)T->eql_w[512 - j];   /* the loudness sum runs over 0..511 */
  }
  if (tid < U) {
    unsigned char* const pk = s_a + tid * POST;
    f32s* const fe = reinterpret_cast<f32s*>(pk);
    double* const prod = reinterpret_cast<double*>(pk + 2064 + 2 * 4 * MP3_CBANDS);
    f32s t0; t0 = (double)wl[tid][0]; t0 *= (double)t0; fe[0] = (double)t0; prod[0] = (double)t0 * (double)T->eql_w[0];
  }
  __syncthreads();
  PSY_CLOCK(7, tid == 0);

  /* partition phases: unit k = tid / PSY_UNIT_THREADS, partition b = tid % PSY_UNIT_THREADS */
  const int k = tid / PSY_UNIT_THREADS, b = tid % PSY_UNIT_THREADS;
  const int npl = T->npart_l;
  unsigned char* const pk = s_a + k * POST;
  f32s* const fe = reinterpret_cast<f32s*>(pk);
  f32s* const s_max = reinterpret_cast<f32s*>(pk + 2064);
  f32s* const s_avg = s_max + MP3_CBANDS;
  const double* const prod = reinterpret_cast<const double*>(pk + 2064 + 2 * 4 * MP3_CBANDS);
  const bool mine = act >> k & 1;
  PsyUnit* const o = o0 + k * nch;
  if (b < npl) {     /* calc_energy (PsyModel.js:906-928) */
    double ebb = 0, m = 0;
    const int l0 = T->line0_l[b], l1 = T->line0_l[b + 1];
    for (int j = l0; j < l1; j++) { const double el = fe[j]; ebb += el; if (m < el) m = el; }
    if (mine) o->eb_l[b] = (float)ebb;
    s_max[b] = m;
    s_avg[b] = ebb * (double)T->rnumlines_l[b];
  }
  /* psycho_loudness_approx (PsyModel.js:241-249): ONE ordered 512-term double sum per unit, half in each partition phase,
   * on a thread of its own per unit (in different warps), so that the units' chains run side by side */
  const bool chain = b == PSY_UNIT_THREADS - 1 && mine;
  double loud = 0.0;
  if (chain) {
#pragma unroll 8
    for (int i = 0; i < 256; ++i) loud += prod[i];
  }
  PSY_CLOCK(11, chain && k == 0);
  PSY_CLOCK(8, tid == 0);
  __syncthreads();
  PSY_CLOCK(9, tid == 0);

  if (b < npl) {     /* calc_mask_index_l (PsyModel.js:930-992) */
    const int lo = b > 0 ? b - 1 : b, hi = b < npl - 1 ? b + 1 : b;
    double a = 0; double m = 0; int lines = 0;
    for (int q = lo; q <= hi; q++) {
      if (q == lo) { a = (double)s_avg[q]; m = (double)s_max[q]; }
      else { a = a + (double)s_avg[q]; if (m < (double)s_max[q]) m = (double)s_max[q]; }
      lines += T->numlines_l[q];
    }
    int kk = 0;
    if (a > 0.0) {
      const double cnt = (double)(hi - lo + 1);
      a = 20.0 * (m * cnt - a) / (a * (lines - 1));
      kk = js_trunc<DOM_TRUNC_MASK_IDX>(a);
      if (kk > 8) kk = 8;
    }
    if (mine) o->mask_idx[b] = (unsigned char)kk;
  }
  PSY_CLOCK(10, tid == 0);
  if (chain) {
#pragma unroll 8
    for (int i = 256; i < 512; ++i) loud += prod[i];
    loud *= (1. / (14752. * 14752.) / 512);
    o->loudness = (float)loud;
  }
  PSY_CLOCK(12, chain && k == 0);
}

/* ---- the short-block half (PsyModel.js:1000-1383 for shortblock, compute_masking_s :740-761) --------------------------
 * Read only for granules encoded as short blocks and their neighbours (psy_short_read): computed after the block-type scan
 * for a compacted list of (unit, channel) pairs. */

/* R(u): the ratio row of unit u (relative, of stream sd) needs en_s / thm_s.  The quantizer of granule u + 1 reads it
 * (calc_xmin's short branch) when either channel of that granule is a short block (per unit: inter-channel masking mixes
 * both channels' thm_s); a stream's last unit is always complete, as its row is carried to the next call (halo_out) and
 * into state blobs.  The halo row (u = -1) is never computed by the masking.  all: every unit (the stage taps). */
__device__ __forceinline__ bool psy_short_read(const Mp3Tables* __restrict__ T, const StreamDesc& sd,
                                               const signed char* __restrict__ bt_final, int u, int all) {
  const int n = T->mode_gr * sd.nframes;
  if (u < 0 || u >= n) return false;
  if (all || u == n - 1) return true;
  const size_t row = (size_t)(sd.unit_base + u + 1) * 2;
  return bt_final[row] == BT_SHORT || (T->nch == 2 && bt_final[row + 1] == BT_SHORT);
}

/* grid ((max_units + 1 + 127) / 128, nstreams) x 128.  Appends (stream, unit, channel) for every unit u >= -1 with
 * S(u) = R(u) || R(u + 1) (the thresholds of unit u + 1 read ecb_s of unit u: nb_s1 / nb_s2) to list; count[0] is its
 * length and count[1] k_psy_short's task counter, both zero on entry. */
__global__ void __launch_bounds__(128)
k_psy_short_list(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, const signed char* __restrict__ bt_final,
                 int all, int2* __restrict__ list, int* __restrict__ count) {
  const int z = blockIdx.y;
  const StreamDesc& sd = streams[z];
  const int u = (int)(blockIdx.x * blockDim.x + threadIdx.x) - 1;
  if (u >= T->mode_gr * sd.nframes) return;
  if (!psy_short_read(T, sd, bt_final, u, all) && !psy_short_read(T, sd, bt_final, u + 1, all)) return;
  const int nch = T->nch;
  const int at = atomicAdd(count, nch);
  for (int ch = 0; ch < nch; ch++) list[at + ch] = make_int2(z, ((u + 1) << 1) | ch);
}

/* persistent blocks of PSY_THREADS pulling (stream, unit, channel) tasks from the list k_psy_short_list built */
#ifndef PSY_SHORT_BLOCKS
#define PSY_SHORT_BLOCKS 8    /* resident blocks per SM */
#endif
template <bool F32_PCM>
__global__ void __launch_bounds__(PSY_THREADS)
k_psy_short(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, PsyShort* __restrict__ out,
            const int2* __restrict__ list, int* __restrict__ count) {
  const int ntasks = count[0];
  if (ntasks == 0) return;
  const int tid = threadIdx.x;
  const int nch = T->nch, nps = T->npart_s;
  __shared__ double xs[1024];
  __shared__ f32w wsh[3][256 + 16];
  __shared__ f32s fes[3][129];
  __shared__ f32s s_ebs[3][MP3_CBANDS];
  __shared__ int s_task;
  for (;;) {
    if (tid == 0) s_task = atomicAdd(count + 1, 1);
    __syncthreads();
    const int t = s_task;
    if (t >= ntasks) return;
    const int2 e = list[t];
    const int z = e.x, u = (e.y >> 1) - 1, ch = e.y & 1;
    const StreamDesc& sd = streams[z];
    const long long c = (long long)T->mode_gr * sd.frame0 + u;
    PsyShort* o = out + psy_row(sd, z, u) * nch + ch;
    if (c < 0) {   /* before the first call: psymodel_init values (PsyModel.js:2573-2595) */
      for (int i = tid; i < 3 * MP3_CBANDS; i += PSY_THREADS) { (&o->ecb_s[0][0])[i] = 1.0; (&o->eb_s[0][0])[i] = 0.0f; }
      __syncthreads();
      continue;
    }
    psy_load_span<F32_PCM, PSY_THREADS>(T, sd, ch, 576 * c - 224, xs);
    __syncthreads();
    /* fft_short (FFT.js:140-183): block b, iteration j writes x_real[b][4j..], [128+4j..] */
    for (int q = tid; q < 96; q += PSY_THREADS) {
      const int b = q >> 5, j = q & 31;
      const int i = c_fft_rv[j << 2], x = 4 * j, k = 192 * (b + 1);
      const float* w = T->fft_window_s;
      const double* bx = xs + i + k;
      double f0, f1, f2, f3, wv;
      f0 = (double)w[i] * (double)bx[0];
      wv = (double)w[0x7f - i] * (double)bx[0x80];
      f1 = f0 - wv; f0 = f0 + wv;
      f2 = (double)w[i + 0x40] * (double)bx[0x40];
      wv = (double)w[0x3f - i] * (double)bx[0xc0];
      f3 = f2 - wv; f2 = f2 + wv;
      wsh[b][FHT_PAD(x + 0)] = f0 + f2; wsh[b][FHT_PAD(x + 2)] = f0 - f2; wsh[b][FHT_PAD(x + 1)] = f1 + f3; wsh[b][FHT_PAD(x + 3)] = f1 - f3;
      f0 = (double)w[i + 0x01] * (double)bx[0x01];
      wv = (double)w[0x7e - i] * (double)bx[0x81];
      f1 = f0 - wv; f0 = f0 + wv;
      f2 = (double)w[i + 0x41] * (double)bx[0x41];
      wv = (double)w[0x3e - i] * (double)bx[0xc1];
      f3 = f2 - wv; f2 = f2 + wv;
      wsh[b][FHT_PAD(x + 128 + 0)] = f0 + f2; wsh[b][FHT_PAD(x + 128 + 2)] = f0 - f2; wsh[b][FHT_PAD(x + 128 + 1)] = f1 + f3; wsh[b][FHT_PAD(x + 128 + 3)] = f1 - f3;
    }
    __syncthreads();
    /* FHT stages 0..2: 32 tasks per stage for each of the three transforms */
#pragma unroll
    for (int stage = 0; stage < 3; stage++) {
      for (int q = tid; q < 96; q += PSY_THREADS) fht_task(wsh[q >> 5], stage, q & 31, T->tw, T->tw_off);
      __syncthreads();
    }
    /* line energies (PsyModel.js:300-316) */
    for (int q = tid; q < 3 * 128; q += PSY_THREADS) {
      const int b = q >> 7, j = q & 127;
      const double re = wsh[b][FHT_PAD(128 - j)], im = wsh[b][FHT_PAD(128 + j)];
      fes[b][128 - j] = (re * re + im * im) * 0.5;
    }
    if (tid < 3) { f32s t0; t0 = (double)wsh[tid][0]; t0 *= (double)t0; fes[tid][0] = (double)t0; }
    __syncthreads();
    for (int q = tid; q < 3 * MP3_CBANDS; q += PSY_THREADS) {   /* short partition energies (compute_masking_s :740-750) */
      const int sb = q >> 6, b = q & 63;
      if (b < nps) {
        double ebb = 0;
        const int l0 = T->line0_s[b], l1 = T->line0_s[b + 1];
        for (int j = l0; j < l1; j++) ebb += (double)fes[sb][j];
        s_ebs[sb][b] = ebb;
        o->eb_s[sb][b] = (float)ebb;
      }
    }
    __syncthreads();
    for (int q = tid; q < 3 * MP3_CBANDS; q += PSY_THREADS) {   /* short spreading sums (compute_masking_s :753-761) */
      const int sb = q >> 6, b = q & 63;
      if (b < nps) {
        int kk = T->s3lo_s[b];
        int j = T->s3off_s[b];
        double ecb = (double)T->s3_ss[j++] * (double)s_ebs[sb][kk];
        ++kk;
        while (kk <= T->s3hi_s[b]) { ecb += (double)T->s3_ss[j] * (double)s_ebs[sb][kk]; ++j; ++kk; }
        o->ecb_s[sb][b] = ecb;
      }
    }
    __syncthreads();   /* s_task, xs and the work arrays are reused by the next task */
  }
}

struct ScanIn { unsigned attack4; float loudness; };

__global__ void k_attack_prepass(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, PsyUnit* __restrict__ psy,
                                 ScanIn* __restrict__ sin) {
  const int z = blockIdx.z;
  const StreamDesc& sd = streams[z];
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= T->mode_gr * sd.nframes) return;
  const int nch = T->nch;
  const double thr = T->attack_threshold;
  for (int ch = 0; ch < nch; ch++) {
    PsyUnit* cur = psy + psy_row(sd, z, u) * nch + ch;
    const PsyUnit* prev = psy + psy_row(sd, z, u - 1) * nch + ch;
    f32s en_subshort[12], attack_intensity[12];
    double en_short[4] = {0, 0, 0, 0};
    int a[4] = {0, 0, 0, 0};
    for (int i = 0; i < 3; i++) {
      en_subshort[i] = (double)prev->peaks[i + 6];
      attack_intensity[i] = (double)en_subshort[i] / (double)prev->peaks[i + 4];
      en_short[0] += (double)en_subshort[i];
    }
    for (int i = 0; i < 9; i++) {
      double p = (double)cur->peaks[i];
      en_subshort[i + 3] = p;
      if (i % 3 == 0) en_short[1 + i / 3] += p;      /* fractional JS index: only i%3==0 lands (SURVEY 8a) */
      if (p > (double)en_subshort[i + 3 - 2]) p = p / (double)en_subshort[i + 3 - 2];
      else if ((double)en_subshort[i + 3 - 2] > p * 10.0) p = (double)en_subshort[i + 3 - 2] / (p * 10.0);
      else p = 0.0;
      attack_intensity[i + 3] = p;
    }
    for (int i = 0; i < 12; i += 3)
      if ((double)attack_intensity[i] > thr) a[i / 3] = 1;
    for (int i = 1; i < 4; i++) {
      double ratio;
      if (en_short[i - 1] > en_short[i]) ratio = en_short[i - 1] / en_short[i];
      else ratio = en_short[i] / en_short[i - 1];
      if (ratio < 1.7) { a[i] = 0; if (i == 1) a[0] = 0; }
    }
    for (int i = 0; i < 4; i++) cur->attack[i] = (unsigned char)a[i];
    ScanIn si;
    si.attack4 = (unsigned)a[0] | ((unsigned)a[1] << 8) | ((unsigned)a[2] << 16) | ((unsigned)a[3] << 24);
    si.loudness = cur->loudness;
    sin[psy_row(sd, z, u) * nch + ch] = si;
    if (u == 0) { si.attack4 = 0; si.loudness = prev->loudness; sin[psy_row(sd, z, -1) * nch + ch] = si; }
  }
}

/* ---- sequential scans, parallelised by speculation ---------------------------------------------------------
 * Two recurrences run through a stream: the attack / block-type FSM (PsyModel.js:1183-1204, 784-826; state =
 * lastAttacks and blocktype_old of both channels) and the ATH auto-adjust IIR (Encoder.js:166-243; state = adjust,
 * adjustLimit).  Both forget their past quickly (two attack-free granules reset the FSM to (0, NORM); two loud frames
 * reset the ATH state to (1, 1)), so each 16-frame chunk is run from a guessed in-state by its own thread, the
 * guesses are checked against the predecessor's out-state, and only wrong chunks are redone until nothing changes.
 * The result equals the sequential scan exactly; the worst case degenerates to it.  One block per stream. */
#define SCAN_FRAMES 16
#define SCAN_THREADS 1024
/* The in-state every chunk but a stream's first starts from: lastAttacks and blocktype_old of both channels, and the ATH
 * (adjust, adjustLimit) pair.  Only the number of redo rounds depends on it (tests/test_gpu_speculation.py builds the
 * library with wrong guesses and checks the bytes). */
#ifndef SCAN_GUESS_LA
#define SCAN_GUESS_LA 0
#endif
#ifndef SCAN_GUESS_BT
#define SCAN_GUESS_BT BT_NORM
#endif
#ifndef SCAN_GUESS_ATH
#define SCAN_GUESS_ATH 1.0
#endif
struct ScanChunk { int fsm_in, fsm_out, dirty_fsm, dirty_ath; double ath_in[2], ath_out[2]; };

__device__ __forceinline__ int fsm_pack(int la0, int la1, int o0, int o1) { return la0 | (la1 << 2) | (o0 << 4) | (o1 << 6); }

__device__ void scan_fsm_chunk(const Mp3Tables* T, const StreamDesc& sd, int z, const ScanIn* sin, signed char* bt_final,
                               signed char* bt_prev, int f0, int f1, ScanChunk* ck) {
  const int nch = T->nch, coupled = T->coupled_short_blocks;
  int la[2] = {ck->fsm_in & 3, (ck->fsm_in >> 2) & 3};
  int old[2] = {(ck->fsm_in >> 4) & 3, (ck->fsm_in >> 6) & 3};
  const int G = T->mode_gr;
  /* (preloading the chunk's inputs into registers was measured slower: spills with 1024 threads, too few threads with 256) */
  for (int u = G * f0; u < G * f1; u++) {
    int uselong[2] = {1, 1};
    for (int ch = 0; ch < nch; ch++) {
      const unsigned av = sin[psy_row(sd, z, u) * nch + ch].attack4;
      int a0 = av & 0xff, a1 = (av >> 8) & 0xff, a2 = (av >> 16) & 0xff, a3 = (av >> 24) & 0xff;
      if (a0 != 0 && la[ch] != 0) a0 = 0;
      if (la[ch] == 3 || (a0 + a1 + a2 + a3) != 0) {
        uselong[ch] = 0;
        if (a1 != 0 && a0 != 0) a1 = 0;
        if (a2 != 0 && a1 != 0) a2 = 0;
        if (a3 != 0 && a2 != 0) a3 = 0;
      }
      la[ch] = a2;
    }
    if (coupled && !(uselong[0] != 0 && uselong[1] != 0)) uselong[0] = uselong[1] = 0;
    const size_t row = (size_t)(sd.unit_base + u) * 2;
    for (int ch = 0; ch < nch; ch++) {
      bt_prev[row + ch] = (signed char)old[ch];          /* what compute_masking_s of this call saw */
      int bt = BT_NORM;
      if (uselong[ch] != 0) {
        if (old[ch] == BT_SHORT) bt = BT_STOP;
      } else {
        bt = BT_SHORT;
        if (old[ch] == BT_NORM) old[ch] = BT_START;
        if (old[ch] == BT_STOP) old[ch] = BT_SHORT;
      }
      bt_final[row + ch] = (signed char)old[ch];
      old[ch] = bt;
    }
  }
  ck->fsm_out = fsm_pack(la[0], la[1], old[0], old[1]);
}

__device__ void scan_ath_chunk(const Mp3Tables* T, const StreamDesc& sd, int z, const ScanIn* sin, double* ath_psy,
                               double* ath_q, int f0, int f1, ScanChunk* ck) {
  const int nch = T->nch;
  double adjust = ck->ath_in[0], limit = ck->ath_in[1];
  const double sens = T->aa_sensitivity_p;
  const int G = T->mode_gr;
  for (int f = f0; f < f1; f++) {
    ath_psy[sd.frame_base + f] = adjust;
    /* loudness_sq[gr][ch] is the loudness of the unit BEFORE call G f + gr (one-call delay, PsyModel.js:321-322) */
    const ScanIn* r0 = sin + psy_row(sd, z, G * f - 1) * nch;
    double max_pow = (double)r0[0].loudness;
    if (nch == 2) max_pow += (double)r0[1].loudness;
    else max_pow += max_pow;
    if (G == 2) {                                     /* Encoder.js:187: the second granule only exists in MPEG-1 */
      const ScanIn* r1 = sin + psy_row(sd, z, G * f) * nch;
      double gr2_max = (double)r1[0].loudness;
      if (nch == 2) gr2_max += (double)r1[1].loudness;
      else gr2_max += gr2_max;
      max_pow = js_dmax(max_pow, gr2_max);
    }
    max_pow *= 0.5;
    max_pow *= sens;
    if (max_pow > 0.03125) {
      if (adjust >= 1.0) adjust = 1.0;
      else if (adjust < limit) adjust = limit;
      limit = 1.0;
    } else {
      const double adj_lim_new = 31.98 * max_pow + 0.000625;
      if (adjust >= adj_lim_new) {
        adjust *= adj_lim_new * 0.075 + 0.925;
        if (adjust < adj_lim_new) adjust = adj_lim_new;
      } else {
        if (limit >= adj_lim_new) adjust = adj_lim_new;
        else if (adjust < limit) adjust = limit;
      }
      limit = adj_lim_new;
    }
    ath_q[sd.frame_base + f] = adjust;
  }
  ck->ath_out[0] = adjust; ck->ath_out[1] = limit;
}

/* grid: nstreams blocks x SCAN_THREADS.  chunks: scratch rows [sd.scan_base, sd.scan_base + nchunks) */
__global__ void __launch_bounds__(SCAN_THREADS)
k_stream_scan(const Mp3Tables* __restrict__ T, StreamDesc* __restrict__ streams, int nstreams,
              const ScanIn* __restrict__ sin, signed char* __restrict__ bt_final,
              signed char* __restrict__ bt_prev, double* __restrict__ ath_psy, double* __restrict__ ath_q,
              ScanChunk* __restrict__ scratch) {
  /* The scan is one block per stream -- with a single long stream the machine idles while it runs.  The subband analysis
   * (k_subband_analysis, needs PCM only) is launched behind it as a programmatic dependent: as soon as every scan block is
   * resident it may start and take the rest of the machine.  (On a side stream it either fought the psy analysis for SMs or
   * kept this 1024-thread block, which needs a whole SM's registers, waiting until it had drained: both measured.) */
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int z = blockIdx.x;
  if (z >= nstreams) return;
  const StreamDesc& sd = streams[z];
  const int nchunks = (sd.nframes + SCAN_FRAMES - 1) / SCAN_FRAMES;
  ScanChunk* ck = scratch + sd.scan_base;
  const int tid = threadIdx.x;
  for (int c = tid; c < nchunks; c += SCAN_THREADS) {
    ck[c].fsm_in = c == 0 ? fsm_pack(sd.last_attacks[0], sd.last_attacks[1], sd.blocktype_old[0], sd.blocktype_old[1])
                          : fsm_pack(SCAN_GUESS_LA, SCAN_GUESS_LA, SCAN_GUESS_BT, SCAN_GUESS_BT);
    ck[c].ath_in[0] = c == 0 ? sd.ath_adjust : SCAN_GUESS_ATH;
    ck[c].ath_in[1] = c == 0 ? sd.ath_adjust_limit : SCAN_GUESS_ATH;
    ck[c].dirty_fsm = ck[c].dirty_ath = 1;
  }
  for (;;) {
    for (int c = tid; c < nchunks; c += SCAN_THREADS) {
      const int f0 = c * SCAN_FRAMES, f1 = min(sd.nframes, f0 + SCAN_FRAMES);
      if (ck[c].dirty_fsm) scan_fsm_chunk(T, sd, z, sin, bt_final, bt_prev, f0, f1, &ck[c]);
      if (ck[c].dirty_ath) scan_ath_chunk(T, sd, z, sin, ath_psy, ath_q, f0, f1, &ck[c]);
    }
    __syncthreads();
    int any = 0;
    for (int c = tid; c < nchunks; c += SCAN_THREADS) {
      ck[c].dirty_fsm = ck[c].dirty_ath = 0;
      if (c == 0) continue;
      if (ck[c].fsm_in != ck[c - 1].fsm_out) { ck[c].fsm_in = ck[c - 1].fsm_out; ck[c].dirty_fsm = 1; any = 1; }
      if (ck[c].ath_in[0] != ck[c - 1].ath_out[0] || ck[c].ath_in[1] != ck[c - 1].ath_out[1]) {
        ck[c].ath_in[0] = ck[c - 1].ath_out[0]; ck[c].ath_in[1] = ck[c - 1].ath_out[1]; ck[c].dirty_ath = 1; any = 1;
      }
    }
    if (!__syncthreads_or(any)) break;
  }
  if (tid == 0 && nchunks > 0) {
    const ScanChunk& l = ck[nchunks - 1];
    streams[z].last_attacks[0] = l.fsm_out & 3; streams[z].last_attacks[1] = (l.fsm_out >> 2) & 3;
    streams[z].blocktype_old[0] = (l.fsm_out >> 4) & 3; streams[z].blocktype_old[1] = (l.fsm_out >> 6) & 3;
    streams[z].ath_adjust = l.ath_out[0]; streams[z].ath_adjust_limit = l.ath_out[1];
  }
}

__device__ __noinline__ double psy_log10(double x) { return m3_log10(x); }
/* 0 | (log10(ratio) * 16) for 1 <= ratio < 10^1.5, from the threshold table when the host validated it (mp3_config.h) */
__device__ __forceinline__ int log10_times16_trunc(const Mp3Tables* T, double ratio) {
  if (!T->l16_ok) return js_trunc<DOM_TRUNC_LOG16>(psy_log10(ratio) * 16.0);
  DOMAIN_MISS(DOM_LOG16_TABLE, !(ratio >= 1.0 && ratio < 31.622776601683793));
  int i = 0;
#pragma unroll
  for (int k = 1; k <= 24; k++) i += ratio >= T->l16_thr[k] ? 1 : 0;
  return i;
}

/* mask_add (PsyModel.js:403-473), long blocks only (shortblock == 0) */
__device__ __forceinline__ double mask_add_dev(double m1, double m2, int kk, int b, const Mp3Tables* T, double ath_adjust) {
  double ratio;
  if (m2 > m1) {
    if (m2 < (m1 * T->ma_max_i2)) ratio = m2 / m1;
    else return (m1 + m2);
  } else {
    if (m1 >= (m2 * T->ma_max_i2)) return (m1 + m2);
    ratio = m1 / m2;
  }
  m1 += m2;
  if ((b + 3) <= 3 + 3) {                    /* sic: signed compare in lamejs */
    if (ratio >= T->ma_max_i1) return m1;
    const int i = log10_times16_trunc(T, ratio);
    return m1 * c_table2[i];
  }
  const int i = log10_times16_trunc(T, ratio);
  m2 = (double)T->ath_cb_l[kk] * ath_adjust;
  if (m1 < T->ma_max_m * m2) {
    if (m1 > m2) {
      double f = 1.0, r;
      if (i <= 13) f = c_table3[i];
      r = psy_log10(m1 / m2) * (10.0 / 15.0);
      return m1 * ((c_table1[i] - f) * r + f);
    }
    if (i > 13) return m1;
    return m1 * c_table3[i];
  }
  return m1 * c_table1[i];
}

/* grid (max_units + 1, 1, nstreams); threads: 64 per channel.  The short half (thresholds, conversion, pre-echo factor,
 * inter-channel masking) only where psy_short_read holds. */
__global__ void __launch_bounds__(MASK_THREADS)
k_psy_masking(const Mp3Tables* __restrict__ T, const StreamDesc* __restrict__ streams, const PsyUnit* __restrict__ psy,
              const PsyShort* __restrict__ psy_s, const signed char* __restrict__ bt_prev, const signed char* __restrict__ bt_final,
              int all_short, const double* __restrict__ ath_psy, PsyRatioDev* __restrict__ ratio) {
  const int z = blockIdx.z;
  const StreamDesc& sd = streams[z];
  const int u = (int)blockIdx.x - 1;
  if (u >= T->mode_gr * sd.nframes) return;
  const int nch = T->nch;
  const long long c = (long long)T->mode_gr * sd.frame0 + u;
  const int tid = threadIdx.x, ch = tid >> 6, b = tid & 63;
  PsyRatioDev* out = ratio + psy_row(sd, z, u) * nch;
  if (u < 0) {
    if (c < 0) {   /* en/thm start values 1e20 (PsyModel.js:2579-2587) */
      const float big = (float)1e20;
      for (int i = tid; i < nch * 122; i += MASK_THREADS) (&out[0].en_l[0])[i] = big;
    }
    else if (sd.halo_in) {   /* streaming handle: masking of the unit before frame0, carried on the device */
      for (int i = tid; i < nch * 122; i += MASK_THREADS) (&out[0].en_l[0])[i] = sd.halo_in[i];
    }
    return;
  }
  __shared__ f32s s_thr[2][MP3_CBANDS + 2], s_eb[2][MP3_CBANDS + 2];
  __shared__ f32s s_thr_s[2][3][MP3_CBANDS + 2];
  __shared__ PsyRatioDev s_out[2];
  const int npl = T->npart_l, nps = T->npart_s;
  /* (staging these rows in shared memory was measured slower: the extra barrier costs more than the L1 hits) */
  const PsyUnit* pu = (ch < nch) ? psy + psy_row(sd, z, u) * nch + ch : nullptr;
  const PsyShort* ps = (ch < nch) ? psy_s + psy_row(sd, z, u) * nch + ch : nullptr;
  const PsyShort* pp = (ch < nch) ? psy_s + psy_row(sd, z, u - 1) * nch + ch : nullptr;
  const bool short_read = psy_short_read(T, sd, bt_final, u, all_short);
  const double ath_adjust = ath_psy[sd.frame_base + u / T->mode_gr];

  if (ch < nch) {
    /* long-block spreading + mask_add (PsyModel.js:1274-1324); thr[b] = ecb because pcfact == 0 */
    if (b < npl) {
      int kk = T->s3lo_l[b];
      int k = T->s3off_l[b];
      double eb2 = (double)pu->eb_l[kk] * c_tab[pu->mask_idx[kk]];
      double ecb = (double)T->s3_ll[k++] * eb2;
      while (++kk <= T->s3hi_l[b]) {
        eb2 = (double)pu->eb_l[kk] * c_tab[pu->mask_idx[kk]];
        ecb = mask_add_dev(ecb, (double)T->s3_ll[k++] * eb2, kk, kk - b, T, ath_adjust);
      }
      ecb *= 0.158489319246111;
      s_thr[ch][b] = ecb;
      s_eb[ch][b] = (double)pu->eb_l[b];
    } else { s_thr[ch][b] = 0.0; s_eb[ch][b] = 0.0; }
    /* short-block thresholds (compute_masking_s :753-777); nb_s1/nb_s2 = float32 ecb of the two previous sub-blocks */
    const int prev_short = bt_prev[(size_t)(sd.unit_base + u) * 2 + ch] == BT_SHORT;
    for (int sb = 0; short_read && sb < 3; sb++) {
      if (b < nps) {
        const double ecb = ps->ecb_s[sb][b];
        const float nb1 = sb >= 1 ? (float)ps->ecb_s[sb - 1][b] : (float)pp->ecb_s[2][b];
        const float nb2 = sb == 2 ? (float)ps->ecb_s[0][b] : (sb == 1 ? (float)pp->ecb_s[2][b] : (float)pp->ecb_s[1][b]);
        f32s t;
        t = js_dmin(ecb, 2 * (double)nb1);
        if (prev_short) { const double x = 16 * (double)nb2, y = (double)t; t = js_dmin(x, y); }
        s_thr_s[ch][sb][b] = (double)t;
      } else s_thr_s[ch][sb][b] = 0.0;
    }
  }
  __syncthreads();

  /* partition -> scalefactor band (convert_partition2scalefac_l/_s): every band is its own ordered accumulation over the
   * slice of partitions the reference's cursor walk gives it (Mp3Conv), one thread per band (and sub-block) */
  if (ch < nch && b < 22) {
    const int sbi = b;
    f32s* en = reinterpret_cast<f32s*>(s_out[ch].en_l);
    f32s* thm = reinterpret_cast<f32s*>(s_out[ch].thm_l);
    const int init = T->conv_l.init[sbi];
    if (init == -2) { en[sbi] = 0.0; thm[sbi] = 0.0; }
    else {
      double enn = 0.0, thmm = 0.0;
      if (init >= 0) {
        const double w_next = 1.0 - (double)T->bo_l_weight[sbi - 1];
        enn = w_next * (double)s_eb[ch][init];
        thmm = w_next * (double)s_thr[ch][init];
      }
      const int p1 = T->conv_l.end[sbi];
      for (int p = T->conv_l.start[sbi]; p < p1; p++) { enn += (double)s_eb[ch][p]; thmm += (double)s_thr[ch][p]; }
      en[sbi] = enn; thm[sbi] = thmm;
      const int bd = T->conv_l.bound[sbi];
      if (bd >= 0) {
        const double w_curr = (double)T->bo_l_weight[sbi];
        en[sbi] += w_curr * (double)s_eb[ch][bd];
        thm[sbi] += w_curr * (double)s_thr[ch][bd];
      }
    }
  } else if (short_read && ch < nch && b >= 22 && b < 22 + 39) {
    const int q = b - 22, sbi = q / 3, sblock = q - 3 * sbi;
    f32s(*en)[3] = reinterpret_cast<f32s(*)[3]>(s_out[ch].en_s);
    f32s(*thm)[3] = reinterpret_cast<f32s(*)[3]>(s_out[ch].thm_s);
    const int init = T->conv_s.init[sbi];
    if (init == -2) { en[sbi][sblock] = 0.0; thm[sbi][sblock] = 0.0; }
    else {
      double enn = 0.0, thmm = 0.0;
      if (init >= 0) {
        const double w_next = 1.0 - (double)T->bo_s_weight[sbi - 1];
        enn = w_next * (double)ps->eb_s[sblock][init];
        thmm = w_next * (double)s_thr_s[ch][sblock][init];
      }
      const int p1 = T->conv_s.end[sbi];
      for (int p = T->conv_s.start[sbi]; p < p1; p++) { enn += (double)ps->eb_s[sblock][p]; thmm += (double)s_thr_s[ch][sblock][p]; }
      en[sbi][sblock] = enn; thm[sbi][sblock] = thmm;
      const int bd = T->conv_s.bound[sbi];
      if (bd >= 0) {
        const double w_curr = (double)T->bo_s_weight[sbi];
        en[sbi][sblock] += w_curr * (double)ps->eb_s[sblock][bd];
        thm[sbi][sblock] += w_curr * (double)s_thr_s[ch][sblock][bd];
      }
    }
    /* pre-echo factor and pulse detection (PsyModel.js:1231-1266; NS_INTERP(.,thmm,0) == thmm) */
    const double e3 = (double)pu->peaks[sblock * 3 + 0], e4 = (double)pu->peaks[sblock * 3 + 1], e5 = (double)pu->peaks[sblock * 3 + 2];
    double t = (double)thm[sbi][sblock];
    t *= 0.8;
    const double enn2 = e3 + e4 + e5;
    if (e5 * 6 < enn2) { t *= 0.5; if (e4 * 6 < enn2) t *= 0.5; }
    thm[sbi][sblock] = t;
  }
  __syncthreads();
  /* inter-channel masking (PsyModel.js:525-543), stereo with interChRatio > 0 */
  if (nch == 2 && T->interch_ratio > 0.0 && tid < (short_read ? 22 + 39 : 22)) {
    const double r = T->interch_ratio;
    f32s* t0 = reinterpret_cast<f32s*>(tid < 22 ? &s_out[0].thm_l[tid] : &s_out[0].thm_s[0][0] + (tid - 22));
    f32s* t1 = reinterpret_cast<f32s*>(tid < 22 ? &s_out[1].thm_l[tid] : &s_out[1].thm_s[0][0] + (tid - 22));
    const double l = (double)*t0, rr = (double)*t1;
    *t0 += rr * r;
    *t1 += l * r;
  }
  __syncthreads();
  for (int i = tid; i < nch * 122; i += MASK_THREADS)
    if (short_read || i % 122 < 44) (&out[0].en_l[0])[i] = (&s_out[0].en_l[0])[i];
  if (sd.halo_out && u == T->mode_gr * sd.nframes - 1)
    for (int i = tid; i < nch * 122; i += MASK_THREADS) sd.halo_out[i] = (&s_out[0].en_l[0])[i];
}

#endif
