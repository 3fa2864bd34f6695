/* k_handle.cuh -- streaming handles inside an encode session (mp3b200_session_encode_batch and its twins, DESIGN.md 16).
 *
 * A handle bound to a session keeps its retained samples (the tail) and its carried sequential state on the device, in a
 * HandleRecord and two tail buffers beside it.  Per call: k_gather_rows (k_stage.cuh) puts [tail | caller's rows] into the
 * rows the launch reads; k_tail_store writes what each handle keeps into a tail buffer; k_handle_carry_in copies each
 * handle's carried scalars into the launch's descriptors before the psy analysis reads them; after the packer
 * k_handle_commit takes the end state back into the records, or, when the call is refused, marks its handles refused.
 *
 * Included after k_stage.cuh (GATHER_THREADS, GATHER_SPAN, desc_of) and mp3_device.cuh (StreamDesc).
 */
#ifndef MP3B200_K_HANDLE_CUH
#define MP3B200_K_HANDLE_CUH
#include "k_stage.cuh"

/* the device record of a bound handle */
struct HandleRecord {
  /* the sequential state at the start of the handle's next frame (StreamDesc's carried fields) */
  double ath_adjust, ath_adjust_limit;
  int blocktype_old[2], last_attacks[2], old_value[2], current_step[2];
  int refused;                      /* a call that named the handle was refused: nothing has been committed since */
  int words[3];                     /* that call's status words [0], [1] and [3] */
  unsigned long long call;          /* that call's index in its session */
};

/* one handle's tail of a call: dst[c][i] = src[c][i] for i < n_src, else 0 (flush zeros), i < n; nothing when rec is refused */
struct TailDesc {
  const void* src[2];               /* the gathered launch row (Float32) or the caller's row (Int16 or Float32) */
  float* dst[2];
  long long n, n_src;
  int src_f32;
  const HandleRecord* rec;
  long long blk0;                   /* as GatherDesc::blk0 */
};

/* one entry of a call for k_handle_commit: its record and its row in the launch (-1: it encodes nothing) */
struct CommitDesc {
  HandleRecord* rec;
  int z;
};

/* grid (total blocks, nch) */
__global__ void __launch_bounds__(GATHER_THREADS)
k_tail_store(const TailDesc* __restrict__ descs, int nd, int nch) {
  const int ch = blockIdx.y;
  const TailDesc& d = descs[desc_of(descs, nd, (long long)blockIdx.x)];
  if (ch >= nch || d.rec->refused) return;
  const long long lo = ((long long)blockIdx.x - d.blk0) * GATHER_SPAN, hi = lo + GATHER_SPAN < d.n ? lo + GATHER_SPAN : d.n;
  float* __restrict__ y = d.dst[ch];
  for (long long i = lo + threadIdx.x; i < hi; i += GATHER_THREADS) {
    float v = 0.0f;
    if (i < d.n_src) v = d.src_f32 ? static_cast<const float*>(d.src[ch])[i] : (float)static_cast<const int16_t*>(d.src[ch])[i];
    y[i] = v;
  }
}

/* after run_pipeline has uploaded the descriptors: stream z starts from the carried state of recs[z]; a handle already
 * refused writes its masking to `halo_scratch`, so that the halo it had before the refused call survives */
__global__ void k_handle_carry_in(StreamDesc* __restrict__ streams, int S, HandleRecord* const* __restrict__ recs,
                                  float* __restrict__ halo_scratch) {
  const int z = blockIdx.x * blockDim.x + threadIdx.x;
  if (z >= S) return;
  const HandleRecord& r = *recs[z];
  StreamDesc& sd = streams[z];
  sd.ath_adjust = r.ath_adjust; sd.ath_adjust_limit = r.ath_adjust_limit;
  for (int c = 0; c < 2; c++) {
    sd.blocktype_old[c] = r.blocktype_old[c]; sd.last_attacks[c] = r.last_attacks[c];
    sd.old_value[c] = r.old_value[c]; sd.current_step[c] = r.current_step[c];
  }
  if (r.refused) sd.halo_out = halo_scratch;
}

#define COMMIT_THREADS 256
/* One block, after the packer.  words: the session's ws.refusals ([0] a refused sample (k_stage_f32), [1] frames over
 * their budget, [3] a loop fault, [6] a refused sample of the caller's rows (k_check_rows_f32)).  The words of handles
 * already refused join the call's; then [0] |= [6], and the call is refused when [0], [1] or [3] is set.  A call that
 * stands commits each live handle's end state (streams[z], as k_qstate_commit left it) into its record; a refused one
 * commits nothing and marks every handle it names refused with its words.  words[7] = 1 for a refused call, else 0. */
__global__ void __launch_bounds__(COMMIT_THREADS)
k_handle_commit(const StreamDesc* __restrict__ streams, const CommitDesc* __restrict__ d, int n, int* __restrict__ words,
                unsigned long long call) {
  for (int i = threadIdx.x; i < n; i += COMMIT_THREADS) {
    const HandleRecord& r = *d[i].rec;
    if (!r.refused) continue;
    if (r.words[0]) atomicOr(&words[0], r.words[0]);
    if (r.words[1]) atomicOr(&words[1], r.words[1]);
    if (r.words[2]) atomicOr(&words[3], r.words[2]);
  }
  __syncthreads();
  __shared__ int w[3];
  if (threadIdx.x == 0) {
    words[0] |= words[6];
    w[0] = words[0]; w[1] = words[1]; w[2] = words[3];
    words[7] = (w[0] | w[1] | w[2]) ? 1 : 0;
  }
  __syncthreads();
  const bool bad = (w[0] | w[1] | w[2]) != 0;
  for (int i = threadIdx.x; i < n; i += COMMIT_THREADS) {
    HandleRecord& r = *d[i].rec;
    if (bad) {
      if (r.refused) continue;
      r.refused = 1; r.words[0] = w[0]; r.words[1] = w[1]; r.words[2] = w[2]; r.call = call;
    } else if (d[i].z >= 0) {
      const StreamDesc& sd = streams[d[i].z];
      r.ath_adjust = sd.ath_adjust; r.ath_adjust_limit = sd.ath_adjust_limit;
      for (int c = 0; c < 2; c++) {
        r.blocktype_old[c] = sd.blocktype_old[c]; r.last_attacks[c] = sd.last_attacks[c];
        r.old_value[c] = sd.old_value[c]; r.current_step[c] = sd.current_step[c];
      }
    }
  }
}

#endif
