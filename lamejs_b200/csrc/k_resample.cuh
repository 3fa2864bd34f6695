/* k_resample.cuh -- the resampler lamejs runs in front of the encoder when the output rate divides the input rate.
 *
 * Included after every other kernel header: its __constant__ table then sits behind theirs, and their constant-bank
 * addresses (and code) stay as they were.
 */
#ifndef MP3B200_K_RESAMPLE_CUH
#define MP3B200_K_RESAMPLE_CUH
#include "mp3_device.cuh"

/* ---- resampler: lamejs fill_buffer_resample (Lame.js:1719-1843) for an integer rate ratio r = in / out ----
 * With out | in the filter bank has one row in use (bpc = 1, offset 0) and the input position of output m is r m exactly,
 * whatever the call sizes, so output m of a stream is
 *   y[m] = Float32( sum_{i=0..32} (double)h[i] * xs[r m - 16 + i] ),  summed in double in tap order from 0.0,
 * xs = Float32(Int16 * scale) (lamejs scales its Float32Array before resampling), 0 before the stream and past its end
 * (inbuf_old starts zeroed; flush feeds zeros).  y then stands where the input would: the rest of the pipeline reads it
 * like PCM at the output rate (k_psy_analysis<true>, k_subband_analysis<true>). */
#define RS_THREADS 256
#define RS_MAX_RATIO 6                          /* 48 kHz -> 8 kHz */
__constant__ float c_rs_h[RS_MAX_RATIO + 1][MP3_RS_TAPS];   /* row r: the filter of ratio r (the taps depend on r only) */

struct ResampleDesc {
  const void* x[2];         /* input of each channel (In), at stream sample x_base */
  long long x_base, x_end;  /* input samples [x_base, x_end) are there; samples >= x_end (and < 0) read as 0 */
  float* y[2];              /* outputs y_base .. y_base + ny - 1 of each channel */
  long long y_base, ny;
};

/* grid (ceil(max ny / RS_THREADS), nch, nstreams); thread = one output.  In: int16_t (the caller's Int16 samples) or float
 * (Float32 rows, already Float32(x * scale) when staged by k_stage_f32: the launch passes scale_applied = 0 then). */
template <class In>
__global__ void __launch_bounds__(RS_THREADS)
k_resample(const ResampleDesc* __restrict__ descs, int ratio, int scale_applied, double scale) {
  __shared__ double xs[RS_MAX_RATIO * RS_THREADS + MP3_RS_TAPS];
  const ResampleDesc& d = descs[blockIdx.z];
  const int ch = blockIdx.y, tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * RS_THREADS;     /* first output of the block, relative to y_base */
  if (m0 >= d.ny) return;
  /* the block's input span: r * RS_THREADS + 32 samples from r (y_base + m0) - 16, widened once */
  const long long k0 = (long long)ratio * (d.y_base + m0) - MP3_RS_HALF;
  const int span = ratio * RS_THREADS + MP3_RS_TAPS - 1;
  const In* __restrict__ x = static_cast<const In*>(d.x[ch]);
  for (int j = tid; j < span; j += RS_THREADS) {
    const long long k = k0 + j;
    double s;
    if constexpr (sizeof(In) == 2) {
      const int v = (k >= 0 && k < d.x_end) ? (int)__ldg(&x[k - d.x_base]) : 0;
      s = (double)v;
    } else {
      s = (k >= 0 && k < d.x_end) ? (double)__ldg(&x[k - d.x_base]) : 0.0;
    }
    if (scale_applied) s = (double)(float)(s * scale);
    xs[j] = s;
  }
  __syncthreads();
  const long long m = m0 + tid;
  if (m >= d.ny) return;
  const double* w = xs + ratio * tid;
  const float* h = c_rs_h[ratio];
  double acc = 0.;
#pragma unroll
  for (int i = 0; i < MP3_RS_TAPS; i++) acc += w[i] * (double)h[i];
  d.y[ch][m] = (float)acc;
}

/* ---- Float32 input: lamejs's store and scale (Lame.js:1500-1510, 1554-1560) ----
 * encodeBuffer stores each caller value into a Float32Array, x = Float32(v) (the caller's float rows hold that already), and
 * scales it in place, x = Float32((double)x * scale), when the preset's scale is not 1.  k_stage_f32 writes those rows,
 * where the <true> instantiations of the psy analysis and the filterbank, k_resample<float> and the ReplayGain analysis read
 * them.  A non-finite value (before or after the scale), or one beyond MP3_F32_MAX_SAMPLE after it, sets refused[0] and is
 * staged as 0, so that nothing downstream sees it: such a call is refused, and its output is not used.
 * MP3_F32_MAX_SAMPLE (2^40, 2^25 x full scale) lies just above the rung 3.3e7 x full scale of
 * tests/golden/lamejs_loud_golden.json, the loudest at which the library equals lamejs stage by stage and byte for byte with
 * every domain counter (mp3_device.cuh) at zero.  At 1e9 x full scale a Float32 store overflows; from 1e15 lamejs's own
 * masking energies overflow Float32, from 1e30 its MDCT lines, and it encodes (when it does not throw) from infinities and
 * NaNs (DESIGN.md 12).  A test build may set another limit with
 * -DMP3_F32_MAX_SAMPLE=...; non-finite samples stay refused. */
#ifndef MP3_F32_MAX_SAMPLE
#define MP3_F32_MAX_SAMPLE 1099511627776.0f
#endif
#define STAGE_THREADS 256
#define STAGE_PER_THREAD 4
struct StageDesc {
  const float* x[2];        /* the caller's rows */
  float* y[2];              /* staged rows */
  long long n;              /* samples per channel */
};

/* grid (ceil(max n / (STAGE_THREADS * STAGE_PER_THREAD)), nch, nstreams) */
__global__ void __launch_bounds__(STAGE_THREADS)
k_stage_f32(const StageDesc* __restrict__ descs, int scale_applied, double scale, int* __restrict__ refused) {
  const StageDesc& d = descs[blockIdx.z];
  const int ch = blockIdx.y;
  const float* __restrict__ x = d.x[ch];
  float* __restrict__ y = d.y[ch];
  const long long i0 = (long long)blockIdx.x * (STAGE_THREADS * STAGE_PER_THREAD) + threadIdx.x;
  bool bad = false;
#pragma unroll
  for (int k = 0; k < STAGE_PER_THREAD; k++) {
    const long long i = i0 + (long long)k * STAGE_THREADS;
    if (i >= d.n) break;
    float v = __ldg(&x[i]);
    if (scale_applied) v = (float)((double)v * scale);
    if (!(fabsf(v) <= MP3_F32_MAX_SAMPLE)) { bad = true; v = 0.0f; }
    y[i] = v;
  }
  if (bad) atomicOr(refused, 1);
}

/* ---- stereo WAV data: interleaved little-endian Int16 frames (L R L R ...) to the planar rows whole streams read ----
 * worker.js:31-38 splits the data chunk the same way: left[i] = view[2 i], right[i] = view[2 i + 1].  The samples are
 * copied as they are (the Int16 path applies lamejs's scale itself).  Mono data regions already are rows and are not staged.
 * Slice j of nchunks stages the frames [n j / nchunks, n (j + 1) / nchunks) of every file, the rule the sliced upload and
 * k_psy_analysis share, so slice j reads only bytes that slice j's copy has landed. */
#define WAV_STAGE_THREADS 256
struct WavStageDesc {
  const uint8_t* x;         /* the file's data region, 16-byte aligned: frame i at x + 4 i */
  int16_t* y[2];            /* left row (8-byte aligned), right row */
  long long n;              /* frames (samples per channel) */
};

/* grid (ceil(max groups of 4 frames in a slice / WAV_STAGE_THREADS), files); thread = 4 frames at 4 g .. 4 g + 3 */
__global__ void __launch_bounds__(WAV_STAGE_THREADS)
k_stage_wav(const WavStageDesc* __restrict__ descs, int j, int nchunks) {
  const WavStageDesc& d = descs[blockIdx.y];
  const long long lo = d.n * j / nchunks, hi = d.n * (j + 1) / nchunks;
  const long long g = (lo >> 2) + (long long)blockIdx.x * WAV_STAGE_THREADS + threadIdx.x, i0 = 4 * g;
  if (i0 >= hi) return;
  int16_t* __restrict__ yl = d.y[0] + i0;
  int16_t* __restrict__ yr = d.y[1] + i0;
  if (i0 >= lo && i0 + 4 <= hi) {         /* the whole group is in the slice: one 16-byte load, two 8-byte rows */
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(d.x) + g);
    const uint2 l = make_uint2(__byte_perm(v.x, v.y, 0x5410), __byte_perm(v.z, v.w, 0x5410));
    const uint2 r = make_uint2(__byte_perm(v.x, v.y, 0x7632), __byte_perm(v.z, v.w, 0x7632));
    *reinterpret_cast<uint2*>(yl) = l;
    if ((reinterpret_cast<uintptr_t>(yr) & 7) == 0) {
      *reinterpret_cast<uint2*>(yr) = r;
    } else {
      yr[0] = (int16_t)(r.x & 0xffff); yr[1] = (int16_t)(r.x >> 16); yr[2] = (int16_t)(r.y & 0xffff); yr[3] = (int16_t)(r.y >> 16);
    }
    return;
  }
  for (int k = 0; k < 4; k++) {           /* a group cut by the slice's ends: its frames one by one */
    const long long i = i0 + k;
    if (i < lo || i >= hi) continue;
    const unsigned w = __ldg(reinterpret_cast<const unsigned*>(d.x) + i);
    yl[k] = (int16_t)(w & 0xffff);
    yr[k] = (int16_t)(w >> 16);
  }
}

#endif
