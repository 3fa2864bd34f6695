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
  /* tagged handles (DESIGN.md 17): gfc.nMusicCRC, and the titles ended so far with the last one's gain (GetTitleGain) */
  unsigned music_crc;
  int titles;
  double title_db;
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

/* ---- tagged and ReplayGain handles (mp3b200_session_encode_batch_tagged and its twins, DESIGN.md 17) ----
 * These need k_tag.cuh (crc_append) and k_replaygain.cuh (RgCarry, RG_HIST), which mp3_encoder.cu includes first.
 * A call's refusal is known only after the packer, so nothing that analyses or checksums a call writes a handle's own state:
 * the analysis works on a copy of each handle's carry and histogram A (k_rg_stage_in), and the commit kernels below, which
 * run behind k_handle_commit, take the results into the handle only when words[7] says the call stood. */

/* one analysing handle of a call: its RgCarry + A (d_rg) and their copy in session workspace; q is its title in the job */
struct RgStageDesc {
  uint8_t* handle;
  uint8_t* stage;
  HandleRecord* rec;
  int q, title_end;
};
enum { RG_STAGE_BYTES = (int)sizeof(RgCarry) + 4 * RG_HIST, RG_STAGE_THREADS = 256 };
static_assert(RG_STAGE_BYTES % 16 == 0, "RgCarry + A copied as 16-byte words");

/* grid (handles): stage = the handle's carry and A */
__global__ void __launch_bounds__(RG_STAGE_THREADS) k_rg_stage_in(const RgStageDesc* __restrict__ d) {
  const RgStageDesc e = d[blockIdx.x];
  const uint4* src = reinterpret_cast<const uint4*>(e.handle);
  uint4* dst = reinterpret_cast<uint4*>(e.stage);
  for (int i = threadIdx.x; i < RG_STAGE_BYTES / 16; i += RG_STAGE_THREADS) dst[i] = src[i];
}

/* grid (handles), behind k_handle_commit: when the call stood, the staged carry and A become the handle's; at a title end
 * (GetTitleGain) A is added to B instead and cleared, and the record takes the title's gain (gain[q]) and counts it */
__global__ void __launch_bounds__(RG_STAGE_THREADS)
k_rg_commit(const RgStageDesc* __restrict__ d, const int* __restrict__ words, const double* __restrict__ gain) {
  if (words[7]) return;
  const RgStageDesc e = d[blockIdx.x];
  if (!e.title_end) {
    const uint4* src = reinterpret_cast<const uint4*>(e.stage);
    uint4* dst = reinterpret_cast<uint4*>(e.handle);
    for (int i = threadIdx.x; i < RG_STAGE_BYTES / 16; i += RG_STAGE_THREADS) dst[i] = src[i];
    return;
  }
  const int* a = reinterpret_cast<const int*>(e.stage + sizeof(RgCarry));
  int* ha = reinterpret_cast<int*>(e.handle + sizeof(RgCarry));
  int* hb = ha + RG_HIST;
  for (int b = threadIdx.x; b < RG_HIST; b += RG_STAGE_THREADS) { hb[b] += a[b]; ha[b] = 0; }
  const unsigned* cs = reinterpret_cast<const unsigned*>(e.stage);     /* the carry k_rg_finish zeroed */
  unsigned* ch = reinterpret_cast<unsigned*>(e.handle);
  for (int i = threadIdx.x; i < (int)(sizeof(RgCarry) / 4); i += RG_STAGE_THREADS) ch[i] = cs[i];
  if (threadIdx.x == 0) { e.rec->title_db = gain[e.q]; e.rec->titles++; }
}

/* one tagged handle whose frames a call encodes: k_music_crc's word crc[k] of its `bytes` audio bytes */
struct CrcCommitDesc {
  HandleRecord* rec;
  long long bytes;
};

/* behind k_handle_commit: when the call stood, each record's music CRC continues over the call's audio (copy_buffer's
 * running CRC, BitStream.js:924-928) */
__global__ void k_crc_commit(const CrcCommitDesc* __restrict__ d, int n, const unsigned* __restrict__ crc,
                             const CrcTables* __restrict__ tables, const int* __restrict__ words) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n || words[7]) return;
  HandleRecord& r = *d[k].rec;
  r.music_crc = crc_append(r.music_crc, crc[k] & 0xffffu, (unsigned long long)d[k].bytes, tables->pow);
}

/* the records' tag fields for k_tag_finish (crc, title_db: NULL to skip) and the refusals of the handles named, ORed into
 * status[0], [1], [3] (zeroed before) as k_handle_commit merges them */
__global__ void k_tag_gather(HandleRecord* const* __restrict__ recs, int n, unsigned* __restrict__ crc, double* __restrict__ title_db,
                             int* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const HandleRecord& r = *recs[i];
  if (crc) crc[i] = r.music_crc;
  if (title_db) title_db[i] = r.title_db;
  if (r.refused) {
    if (r.words[0]) atomicOr(&status[0], r.words[0]);
    if (r.words[1]) atomicOr(&status[1], r.words[1]);
    if (r.words[2]) atomicOr(&status[3], r.words[2]);
  }
}

#endif
