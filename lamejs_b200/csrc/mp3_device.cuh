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

/* ---- domain check (test builds with -DMP3_DOMAIN_CHECK) ----
 * The helpers below and the quantizer's packed fields are exact only on a stated domain.  The check build counts, per site,
 * every argument outside it in g_domain_hits (read and cleared by mp3b200_debug_domain_hits); it never traps.  Without the
 * define DOMAIN_MISS is empty and the kernels are unchanged. */
enum DomainSite {
  DOM_TRUNC_MASK_IDX,     /* js_trunc: calc_mask_index_l's ratio (k_psy_analysis) */
  DOM_TRUNC_LOG16,        /* js_trunc: 0 | log10(ratio) * 16 without the table (mask_add) */
  DOM_TRUNC_QUANT,        /* js_trunc: quantize_xrpow's lines and adj43 index (count_bits) */
  DOM_TRUNC_NOISE,        /* js_trunc: calc_noise's 0 | (noise * 10 + .5) */
  DOM_DMAX,               /* js_dmax: NaN or -0 argument */
  DOM_DMIN,               /* js_dmin: NaN or -0 argument */
  DOM_PACK_SEARCH,        /* quantised line above 32767 (l3enc is i16; a pair is x | y << 16): bin_search's quantizer */
  DOM_PACK_OUTER,         /* the same in the band-walking quantizer */
  DOM_REGION_MX,          /* region_pick / choose_table: region maximum above IXMAX_VAL */
  DOM_BITSUM_FIELD,       /* region_table_w: a lane's 11-bit code-length field, or band_stats_w's 16-bit field, overflows */
  DOM_LOG16_TABLE,        /* log10_times16_trunc's table path: ratio outside [1, 10^1.5) */
  DOM_F32_OVERFLOW,       /* f32s store: a finite double that rounds to an infinite float */
  DOM_NSITES
};
#ifdef MP3_DOMAIN_CHECK
__device__ unsigned long long g_domain_hits[DOM_NSITES];
#define DOMAIN_MISS(site, cond) do { if (cond) atomicAdd(&g_domain_hits[site], 1ull); } while (0)
#else
#define DOMAIN_MISS(site, cond) do { } while (0)
#endif

struct f32s {
  float v;
  __host__ __device__ __forceinline__ operator double() const { return (double)v; }
  __host__ __device__ __forceinline__ f32s& operator=(double d) {
    v = (float)d;
#if defined(MP3_DOMAIN_CHECK) && defined(__CUDA_ARCH__)
    DOMAIN_MISS(DOM_F32_OVERFLOW, isfinite(d) && !isfinite(v));
#endif
    return *this;
  }
  __host__ __device__ __forceinline__ f32s& operator+=(double d) { return *this = (double)v + d; }
  __host__ __device__ __forceinline__ f32s& operator-=(double d) { return *this = (double)v - d; }
  __host__ __device__ __forceinline__ f32s& operator*=(double d) { return *this = (double)v * d; }
};

/* JS `0 | x` for finite |x| < 2^31 (all call sites on the hot path are range-checked by the reference:
 * count_bits rejects xrpow_max*istep > IXMAX_VAL before quantizing). NaN -> 0 like ToInt32: that is what the
 * hardware conversion (cvt.rzi.s32.f64) returns for NaN.  Beyond 2^31 the conversion saturates where ToInt32 wraps. */
template <int SITE>
__device__ __forceinline__ int js_trunc(double d) {
  DOMAIN_MISS(SITE, fabs(d) >= 2147483648.0);
  return __double2int_rz(d);
}
__device__ __forceinline__ bool js_nan_or_negzero(double a) { return a != a || (a == 0.0 && signbit(a)); }
__device__ __forceinline__ double js_dmax(double a, double b) {   /* Math.max, no NaN/-0 inputs on our paths */
  DOMAIN_MISS(DOM_DMAX, js_nan_or_negzero(a) || js_nan_or_negzero(b));
  return a > b ? a : b;
}
__device__ __forceinline__ double js_dmin(double a, double b) {
  DOMAIN_MISS(DOM_DMIN, js_nan_or_negzero(a) || js_nan_or_negzero(b));
  return a < b ? a : b;
}

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
  long long out_base;      /* device address of frame0's first byte (the packer's output base is always null) */
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
