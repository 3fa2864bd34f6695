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
 * MP3_F32_MAX_SAMPLE (2^35, 2^20 x full scale) is the loudest input the library has been compared with lamejs at, stage by
 * stage and byte for byte (tests/golden/lamejs_loud_golden.json).  Louder rungs the fixtures hold, up to 3.3e7 x full scale,
 * still encode in lamejs on some signals but not yet byte-identically here; from 1e15 x full scale lamejs's own masking
 * energies overflow Float32, from 1e30 its MDCT lines, and it encodes (when it does not throw) from infinities and NaNs
 * (DESIGN.md 12). */
#define MP3_F32_MAX_SAMPLE 34359738368.0f
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

#endif
