/* mp3_device.cuh -- shared device-side definitions of the H100 MP3 encoder kernels.
 *
 * Arithmetic contract (DESIGN.md "numerics"): lamejs computes in IEEE double and rounds to float32 exactly
 * where it stores into a Float32Array.  `f32s` reproduces that: reading converts to double, writing rounds
 * (RNE).  All kernels are compiled with -fmad=false so no multiply-add is contracted.
 */
#ifndef MP3B200_DEVICE_CUH
#define MP3B200_DEVICE_CUH
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "mp3_config.h"
#include "mp3_math.cuh"

struct f32s {
  float v;
  __host__ __device__ __forceinline__ operator double() const { return (double)v; }
  __host__ __device__ __forceinline__ f32s& operator=(double d) { v = (float)d; return *this; }
  __host__ __device__ __forceinline__ f32s& operator+=(double d) { v = (float)((double)v + d); return *this; }
  __host__ __device__ __forceinline__ f32s& operator-=(double d) { v = (float)((double)v - d); return *this; }
  __host__ __device__ __forceinline__ f32s& operator*=(double d) { v = (float)((double)v * d); return *this; }
};

/* JS `0 | x` for finite |x| < 2^31 (all call sites on the hot path are range-checked by the reference:
 * count_bits rejects xrpow_max*istep > IXMAX_VAL before quantizing). NaN -> 0 like ToInt32: that is what the
 * hardware conversion (cvt.rzi.s32.f64) returns for NaN. */
__device__ __forceinline__ int js_trunc(double d) { return __double2int_rz(d); }
__device__ __forceinline__ double js_dmax(double a, double b) {   /* Math.max, no NaN/-0 inputs on our paths */
  return a > b ? a : b;
}
__device__ __forceinline__ double js_dmin(double a, double b) { return a < b ? a : b; }

enum { BT_NORM = 0, BT_START = 1, BT_SHORT = 2, BT_STOP = 3 };

/* One stream (= one lamejs Mp3Encoder instance) inside a batch. */
struct StreamDesc {
  const void* pcm[2];      /* device pointers to sample index `pcm_base` of each channel (pcm_sample_t of the launch) */
  long long pcm_base;      /* stream sample index of pcm[ch][0] (history kept by streaming handles) */
  long long pcm_end;       /* samples with index >= pcm_end (and < 0) read as 0: lead-in and flush padding */
  int frame0;              /* first frame of this launch (absolute index within the stream) */
  int nframes;             /* frames encoded by this launch */
  int unit_base;           /* row of frame0's granule 0 in the per-granule arrays */
  int frame_base;          /* row of frame0 in the per-frame arrays */
  long long out_base;      /* byte offset of frame0 in the output buffer */
  int scan_base;           /* first row of this stream in the scan-chunk scratch */
  int pad_;
  /* streaming handles: masking (en/thm, nch x 122 floats) of the psy unit before frame0, carried on the device between
   * calls; halo_out receives the masking of this launch's last unit.  Both null for whole-stream batches. */
  const float* halo_in;
  float* halo_out;
  /* sequential state at the start of frame0 (lamejs gfc.* carried across frames) */
  double ath_adjust, ath_adjust_limit;
  int blocktype_old[2], last_attacks[2];
  int old_value[2], current_step[2];
};

/* The rows a launch's descriptors point at: the caller's Int16 samples, scale still to apply, or Float32 rows already
 * scaled (k_stage_f32 / k_resample).  pcm_value gives the sample as lamejs holds it in mfbuf, Float32( Int16 * scale )
 * (Lame.js:1506-1560), widened to double; unscaled Int16 widens in one conversion. */
template <bool F32> using pcm_sample_t = std::conditional_t<F32, float, int16_t>;
__device__ __forceinline__ double pcm_value(int16_t v, int scale_applied, double scale) {
  double d = (double)(int)v;
  if (scale_applied) d = (double)(float)(d * scale);
  return d;
}
__device__ __forceinline__ double pcm_value(float v, int, double) { return (double)v; }

/* padding bits: number of padded frames among frames 0..k  (Encoder.js:442-446 in closed form) */
__device__ __host__ __forceinline__ long long pad_count(long long k, int frac, int sr) {
  return k < 0 ? 0 : (k * frac + sr - 1) / sr;
}

#endif
