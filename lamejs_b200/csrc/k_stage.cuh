/* k_stage.cuh -- streaming handles fed from device memory (mp3b200_encode_device and its batch / Float32 twins).
 *
 * A handle keeps its retained samples in its device tail (k_handle.cuh); a device call's rows stay where the caller left
 * them.  Per launch, k_gather_rows puts, for every handle that encodes, [retained | caller's rows] into the contiguous rows
 * the launch reads, in the launch's input format (GatherDesc::pack is unused by the handle calls: NULL).
 * k_check_rows_f32 refuses a Float32 call before anything changes, with k_stage_f32's rule.
 *
 * Included after k_resample.cuh (MP3_F32_MAX_SAMPLE); defines no __constant__ data.
 */
#ifndef MP3B200_K_STAGE_CUH
#define MP3B200_K_STAGE_CUH
#include "k_resample.cuh"

#define GATHER_THREADS 256
#define GATHER_SPAN 4096          /* elements of each copy one block moves */

struct GatherDesc {
  const void* kept[2];      /* the retained samples, uploaded in the launch's format D; n_kept each */
  const void* row[2];       /* the caller's device rows, S (Int16 or Float32); n_row each (NULL when n_row = 0) */
  void* dst[2];             /* [kept | row] as D, n_kept + n_row each; NULL: the handle encodes nothing this round */
  void* pack[2];            /* row[pack_from, n_row) as S, for the host; NULL: nothing to keep */
  long long n_kept, n_row, pack_from;
  long long blk0;           /* its first block: the launch's blocks are the descriptors' spans back to back */
};

/* the descriptor block b of a launch belongs to: the last one whose first block is at most b (a descriptor with no blocks
 * shares its blk0 with the next one, so it is never the last such) */
template <class Desc>
__device__ __forceinline__ int desc_of(const Desc* __restrict__ descs, int nd, long long b) {
  int lo = 0, hi = nd - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (descs[mid].blk0 <= b) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

/* elements [blk, blk + 1) * GATHER_SPAN of dst[i] = D(src[i]), i < n (Int16 -> Float32 is exact).  16-byte loads (and
 * stores) from the first element at which src is 16-byte aligned, when dst is then too; the host places dst so. */
template <class S, class D>
__device__ __forceinline__ void gather_span(const S* __restrict__ src, D* __restrict__ dst, long long n, long long blk) {
  if (n <= 0) return;
  constexpr int V = 16 / sizeof(S);
  const int head = (int)(((16 - ((size_t)src & 15)) & 15) / sizeof(S));
  if (n < head + V || ((size_t)(dst + head) & 15) != 0) {
    const long long lo = blk * GATHER_SPAN, hi = lo + GATHER_SPAN < n ? lo + GATHER_SPAN : n;
    for (long long i = lo + threadIdx.x; i < hi; i += GATHER_THREADS) dst[i] = (D)src[i];
    return;
  }
  const long long nv = (n - head) / V, tail = head + nv * V;
  if (blk == 0) {
    for (int i = threadIdx.x; i < head; i += GATHER_THREADS) dst[i] = (D)src[i];
    for (long long i = tail + threadIdx.x; i < n; i += GATHER_THREADS) dst[i] = (D)src[i];
  }
  const long long c0 = blk * (GATHER_SPAN / V), c1 = c0 + GATHER_SPAN / V < nv ? c0 + GATHER_SPAN / V : nv;
  const uint4* __restrict__ s4 = reinterpret_cast<const uint4*>(src + head);
  for (long long k = c0 + threadIdx.x; k < c1; k += GATHER_THREADS) {
    const uint4 v = __ldg(s4 + k);
    if constexpr (sizeof(S) == sizeof(D)) {
      reinterpret_cast<uint4*>(dst + head)[k] = v;
    } else {                                          /* 8 Int16 -> 8 Float32 */
      float4* o = reinterpret_cast<float4*>(dst + head) + 2 * k;
      o[0] = make_float4((float)(short)(v.x & 0xffff), (float)(short)(v.x >> 16), (float)(short)(v.y & 0xffff), (float)(short)(v.y >> 16));
      o[1] = make_float4((float)(short)(v.z & 0xffff), (float)(short)(v.z >> 16), (float)(short)(v.w & 0xffff), (float)(short)(v.w >> 16));
    }
  }
}

/* grid (total blocks, nch): descriptor z owns blocks [blk0, blk0 + ceil(its longest copy / GATHER_SPAN)), so a batch that
 * mixes one long row with many short ones launches no empty blocks for the short ones.
 * S: the caller's rows (int16_t / float); D: the launch's input format (int16_t, or float when it holds a Float32 handle). */
template <class S, class D>
__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_rows(const GatherDesc* __restrict__ descs, int nd) {
  const int ch = blockIdx.y;
  const GatherDesc& d = descs[desc_of(descs, nd, (long long)blockIdx.x)];
  const long long blk = (long long)blockIdx.x - d.blk0;
  if (d.dst[ch]) {
    D* y = static_cast<D*>(d.dst[ch]);
    gather_span<D, D>(static_cast<const D*>(d.kept[ch]), y, d.n_kept, blk);
    gather_span<S, D>(static_cast<const S*>(d.row[ch]), y + d.n_kept, d.n_row, blk);
  }
  if (d.pack[ch])
    gather_span<S, S>(static_cast<const S*>(d.row[ch]) + d.pack_from, static_cast<S*>(d.pack[ch]), d.n_row - d.pack_from, blk);
}

/* one Float32 row of a device call and its configuration's scale */
struct CheckDesc {
  const float* x;
  long long n;
  double scale;
  int scale_applied;
  long long blk0;           /* its first block, as GatherDesc::blk0 */
};

/* grid (total blocks): row z owns blocks [blk0, blk0 + ceil(n / GATHER_SPAN)).  Sets *refused when a sample, scaled as
 * k_stage_f32 scales it, is not finite or beyond MP3_F32_MAX_SAMPLE (the rule of k_stage_f32 and of the host calls' check) */
__global__ void __launch_bounds__(GATHER_THREADS)
k_check_rows_f32(const CheckDesc* __restrict__ descs, int nd, int* __restrict__ refused) {
  const CheckDesc& d = descs[desc_of(descs, nd, (long long)blockIdx.x)];
  const long long lo = ((long long)blockIdx.x - d.blk0) * GATHER_SPAN, hi = lo + GATHER_SPAN < d.n ? lo + GATHER_SPAN : d.n;
  bool bad = false;
  for (long long i = lo + threadIdx.x; i < hi; i += GATHER_THREADS) {
    float v = __ldg(&d.x[i]);
    if (d.scale_applied) v = (float)((double)v * d.scale);
    if (!(fabsf(v) <= MP3_F32_MAX_SAMPLE)) bad = true;
  }
  if (bad) atomicOr(refused, 1);
}

#endif
