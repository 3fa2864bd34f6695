/* mp3_encoder.cu -- host orchestration + C ABI of libmp3b200.so (see include/mp3b200.h).
 *
 * One batch = S independent streams (lamejs Mp3Encoder instances) x their frames.  The pipeline is
 *   K2 psy_analysis -> K3a sequential scans -> K3b masking -> K1 filterbank+MDCT -> K4/K5 quantize+pack
 * launched on one CUDA stream; all intermediates live in HBM workspaces sized per batch.
 * No CPU fallback exists: if CUDA is unavailable every entry point returns MP3B200_ERR_CUDA.
 */
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/mp3b200.h"
#include "mp3_config.h"
#include "mp3_device.cuh"
#include "mp3_tables.h"
#include "k_filterbank.cuh"
#include "k_psy.cuh"
#include "k_quant.cuh"
#include "k_tag.cuh"
#include "mp3_tag.h"

namespace {

thread_local std::string g_err;
std::mutex g_mu;                          /* guards g_device, g_configs, the per-device flags below */
int g_device = 0;                         /* device of configurations / handles / batch calls created from now on */
std::atomic<long long> g_launches{0};
enum { MP3_MAX_DEVICES = 64 };
bool g_consts_ready[MP3_MAX_DEVICES] = {};   /* __constant__ / __device__ tables are per device */
bool g_fb_attr_done[MP3_MAX_DEVICES] = {};

#define CK(call)                                                                                  \
  do {                                                                                            \
    cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) {                                                                      \
      char b_[512];                                                                               \
      snprintf(b_, sizeof b_, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
      g_err = b_;                                                                                 \
      return MP3B200_ERR_CUDA;                                                                    \
    }                                                                                             \
  } while (0)

struct Config { Mp3Tables host; Mp3Tables* dev; int device; };
std::map<std::tuple<int, int, int, int>, Config*> g_configs;   /* (device, ch, sr, kbps) */
struct ByteGeom { int frame_bytes_nopad, frac_SpF, mode_gr; };
std::map<std::tuple<int, int, int>, ByteGeom> g_byte_geom;   /* (ch, sr, kbps) -> byte geometry; frame_bytes_nopad < 0: unsupported */

/* g_mu held.  Makes `dev` current for the calling thread and uploads the constant tables once per device. */
int ensure_device(int dev) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) { g_err = "no CUDA device available (libmp3b200 has no CPU fallback)"; return MP3B200_ERR_CUDA; }
  if (dev < 0 || dev >= n || dev >= MP3_MAX_DEVICES) { g_err = "invalid CUDA device"; return MP3B200_ERR_CUDA; }
  CK(cudaSetDevice(dev));
  if (!g_consts_ready[dev]) {
    CK(cudaMemcpyToSymbol(c_enwindow, MP3_ENWINDOW, sizeof(double) * 285));
    CK(cudaMemcpyToSymbol(c_mdct_win, MP3_MDCT_WIN, sizeof(double) * 144));
    CK(cudaMemcpyToSymbol(c_sb_order, MP3_SB_ORDER, sizeof(int) * 32));
    int rc = psy_upload_constants();
    if (rc) return rc;
    rc = quant_upload_constants();
    if (rc) return rc;
    g_consts_ready[dev] = true;
  }
  return 0;
}

int get_config(int ch, int sr, int kbps, Config** out) {
  std::lock_guard<std::mutex> lk(g_mu);
  const int dev = g_device;
  int rc = ensure_device(dev);
  if (rc) return rc;
  auto key = std::make_tuple(dev, ch, sr, kbps);
  auto it = g_configs.find(key);
  if (it != g_configs.end()) { *out = it->second; return 0; }
  Config* c = new Config();
  if (mp3_build_tables(ch, sr, kbps, &c->host) != 0) { delete c; g_err = "unsupported configuration"; return MP3B200_ERR_CONFIG; }
  c->device = dev;
  CK(cudaMalloc(&c->dev, sizeof(Mp3Tables)));
  CK(cudaMemcpy(c->dev, &c->host, sizeof(Mp3Tables), cudaMemcpyHostToDevice));
  g_configs[key] = c;
  *out = c;
  return 0;
}

/* frames produced by encodeBuffer(n samples) + flush()  (Lame.js:1592-1663 + :1393-1443 in closed form).
 * framesize = 576 * mode_gr; a frame is encoded whenever the FIFO holds framesize + 752 samples (calcNeeded, Lame.js:1516);
 * the FIFO starts with 528 zeros; ENCDELAY + POSTDELAY = 576 + 1152 regardless of the frame size. */
long long frames_for(long long n, int mode_gr) {
  const long long fs = 576LL * mode_gr, need = fs + 752;
  const long long f_enc = 528 + n >= need ? (528 + n - need) / fs + 1 : 0;
  long long mf_size = 528 + n - fs * f_enc;
  const long long ste = 576 + n - fs * f_enc;            /* mf_samples_to_encode - POSTDELAY */
  long long end_padding = fs - (ste % fs);
  if (end_padding < 576) end_padding += fs;
  long long frames_left = (ste + end_padding) / fs, frames = f_enc;
  /* lame_encode_flush feeds zero bunches of min(1152, need - mf_size) samples and counts ONE frame per bunch that completed
   * any (Lame.js:1416-1443); with 576-sample frames a bunch can complete two, so the loop is replayed, not closed-formed */
  while (frames_left > 0) {
    long long bunch = need - mf_size;
    if (bunch > 1152) bunch = 1152;
    if (bunch < 1) bunch = 1;
    int got = 0;
    while (bunch > 0) {
      const long long c = bunch < fs ? bunch : fs;
      bunch -= c; mf_size += c;
      if (mf_size >= need) { got++; mf_size -= fs; }
    }
    frames += got;
    frames_left -= got > 0 ? 1 : 0;
  }
  return frames;
}

/* ------------------------------------------------------------------------------------------------ */
/* Per-batch device workspace.                                                                         */
struct Workspace {
  int nstreams = 0, nch = 0;
  long long units = 0, frames = 0;        /* granule rows / frame rows */
  StreamDesc* d_streams = nullptr;
  signed char* d_bt_final = nullptr;      /* [units][2] final block type used by MDCT + quantizer */
  signed char* d_bt_prev = nullptr;       /* [units][2] blocktype_old seen by the masking of this granule */
  float* d_xr = nullptr;                  /* [units][nch][576] */
  float* d_slab = nullptr;                /* [units + nstreams][nch][18][32] subband samples (gfc.sb_sample), psy row numbering */
  PsyUnit* d_psy = nullptr;               /* [units + nstreams][nch]  (one halo unit per stream in front) */
  ScanIn* d_scan_in = nullptr;            /* [units + nstreams][nch] attack candidates + loudness for the scans */
  PsyRatioDev* d_ratio = nullptr;         /* [units + nstreams][nch]  masking of unit c (used by granule c+1) */
  double* d_ath_psy = nullptr;            /* [frames] ATH.adjust seen by the psy calls of the frame */
  double* d_ath_q = nullptr;              /* [frames] ATH.adjust after adjust_ATH (quantizer) */
  QuantFrameState* d_qstate = nullptr;    /* [frames] speculation bookkeeping */
  GranuleInfoDev* d_ginfo = nullptr;      /* [units][nch] side info of the final quantization */
  short* d_l3enc = nullptr;               /* [units][nch][576] quantised lines of a gc: after the search, parked best, final */
  float* d_xrq = nullptr;                 /* [units][nch][576] xr as the quantizer sees it (reordered, analog silence zeroed) */
  float* d_xrpow = nullptr;               /* [units][nch][576] |xr|^(3/4) */
  unsigned* d_neg = nullptr;              /* [units][nch][18] sign mask of d_xrq (what the packer needs of it) */
  GcPrep* d_prep = nullptr;               /* [units][nch] xmin + scalars of the prepared granule-channel */
  int* d_dirty = nullptr;                 /* [frames] work list for re-quantization passes */
  int* d_counter = nullptr;               /* [4] */
  ScanChunk* d_scan = nullptr;            /* [frames / SCAN_FRAMES + nstreams] */
  ~Workspace() { release(); }
  void release() {
    cudaFree(d_streams); cudaFree(d_bt_final); cudaFree(d_bt_prev); cudaFree(d_xr); cudaFree(d_slab); d_slab = nullptr; cudaFree(d_psy); cudaFree(d_scan_in); d_scan_in = nullptr;
    cudaFree(d_ratio); cudaFree(d_ath_psy); cudaFree(d_ath_q); cudaFree(d_qstate); cudaFree(d_ginfo);
    cudaFree(d_l3enc); cudaFree(d_xrq); d_xrq = nullptr; cudaFree(d_xrpow); d_xrpow = nullptr; cudaFree(d_neg); d_neg = nullptr; cudaFree(d_prep); d_prep = nullptr; cudaFree(d_dirty); cudaFree(d_counter); cudaFree(d_scan); d_scan = nullptr;
    d_streams = nullptr; d_bt_final = d_bt_prev = nullptr; d_xr = nullptr; d_psy = nullptr; d_ratio = nullptr;
    d_ath_psy = d_ath_q = nullptr; d_qstate = nullptr; d_ginfo = nullptr; d_l3enc = nullptr; d_dirty = nullptr; d_counter = nullptr;
  }
  int alloc(int S, int nch_, long long U, long long F, bool want_l3enc) {
    release();
    nstreams = S; nch = nch_; units = U; frames = F;
    CK(cudaMalloc(&d_streams, sizeof(StreamDesc) * S));
    CK(cudaMalloc(&d_bt_final, (size_t)U * 2 + 16));
    CK(cudaMalloc(&d_bt_prev, (size_t)U * 2 + 16));
    CK(cudaMalloc(&d_xr, sizeof(float) * (size_t)U * nch * 576));
    CK(cudaMalloc(&d_slab, sizeof(float) * (size_t)(U + S) * nch * 576));
    CK(cudaMalloc(&d_psy, sizeof(PsyUnit) * (size_t)(U + S) * nch));
    CK(cudaMalloc(&d_scan_in, sizeof(ScanIn) * (size_t)(U + S) * nch));
    CK(cudaMalloc(&d_ratio, sizeof(PsyRatioDev) * (size_t)(U + S) * nch));
    CK(cudaMalloc(&d_ath_psy, sizeof(double) * (size_t)(F + 1)));
    CK(cudaMalloc(&d_ath_q, sizeof(double) * (size_t)(F + 1)));
    CK(cudaMalloc(&d_qstate, sizeof(QuantFrameState) * (size_t)(F + 1)));
    CK(cudaMalloc(&d_ginfo, sizeof(GranuleInfoDev) * (size_t)U * nch));
    (void)want_l3enc;
    CK(cudaMalloc(&d_l3enc, sizeof(short) * (size_t)U * nch * 576));
    CK(cudaMalloc(&d_xrq, sizeof(float) * (size_t)U * nch * 576));
    CK(cudaMalloc(&d_xrpow, sizeof(float) * (size_t)U * nch * 576));
    CK(cudaMalloc(&d_neg, sizeof(unsigned) * (size_t)U * nch * 18));
    CK(cudaMalloc(&d_prep, sizeof(GcPrep) * (size_t)U * nch));
    CK(cudaMalloc(&d_dirty, sizeof(int) * 3 * (size_t)(F + 1)));
    CK(cudaMalloc(&d_counter, sizeof(int) * Q_NCOUNTERS));
    CK(cudaMalloc(&d_scan, sizeof(ScanChunk) * (size_t)(F / SCAN_FRAMES + S + 1)));
    return 0;
  }
};

/* Everything a host thread needs to drive the GPU: its own non-blocking stream (threads encoding through distinct handles
 * or batches never serialise on the legacy default stream), events, workspace and staging buffers.  Bound to one device;
 * re-created when the thread is used with a configuration of another device. */
enum { MP3_MAX_PCM_CHUNKS = 8 };
/* The stream index is a grid y / z coordinate of several kernels (CUDA limit 65535): larger batches run in groups */
enum { MP3_MAX_LAUNCH_STREAMS = 65535 };
struct ThreadCtx {
  int device = -1;
  cudaStream_t st = nullptr, up_st = nullptr, aux_st = nullptr;   /* main, PCM upload, quantizer repair chain */
  cudaEvent_t ev[8] = {}, evq[QE_COUNT] = {}, ev_in = nullptr, ev_fork = nullptr, ev_join = nullptr, ready[MP3_MAX_PCM_CHUNKS] = {};
  Workspace ws;
  int evq_pred[QE_COUNT] = {};
  int16_t* d_pcm = nullptr; size_t d_pcm_cap = 0;
  uint8_t* d_out = nullptr; size_t d_out_cap = 0;
  uint8_t* h_pin = nullptr; size_t h_pin_cap = 0;       /* pinned host staging */
  long long* d_crc_ranges = nullptr; unsigned* d_crc = nullptr; int crc_cap = 0;   /* music CRC: [2][cap] offsets / lengths, [cap] results */
  void release() {
    if (device < 0) return;
    cudaSetDevice(device);
    ws.release(); ws.units = ws.frames = 0; ws.nstreams = 0;
    cudaFree(d_pcm); d_pcm = nullptr; d_pcm_cap = 0;
    cudaFree(d_out); d_out = nullptr; d_out_cap = 0;
    cudaFreeHost(h_pin); h_pin = nullptr; h_pin_cap = 0;
    cudaFree(d_crc_ranges); d_crc_ranges = nullptr; cudaFree(d_crc); d_crc = nullptr; crc_cap = 0;
    for (auto& e : ev) if (e) { cudaEventDestroy(e); e = nullptr; }
    for (auto& e : evq) if (e) { cudaEventDestroy(e); e = nullptr; }
    for (auto& e : ready) if (e) { cudaEventDestroy(e); e = nullptr; }
    if (ev_in) { cudaEventDestroy(ev_in); ev_in = nullptr; }
    if (ev_fork) { cudaEventDestroy(ev_fork); ev_fork = nullptr; }
    if (ev_join) { cudaEventDestroy(ev_join); ev_join = nullptr; }
    if (aux_st) { cudaStreamDestroy(aux_st); aux_st = nullptr; }
    if (st) { cudaStreamDestroy(st); st = nullptr; }
    if (up_st) { cudaStreamDestroy(up_st); up_st = nullptr; }
    device = -1;
  }
  ~ThreadCtx() { release(); }
  int use(int dev) {
    CK(cudaSetDevice(dev));
    if (device == dev) return 0;
    release();
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&up_st, cudaStreamNonBlocking));
    for (auto& e : ev) CK(cudaEventCreate(&e));
    for (auto& e : evq) CK(cudaEventCreate(&e));
    for (auto& e : ready) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
    {
      int lo = 0, hi = 0;                  /* the repair chain is latency critical: highest priority */
      CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
      CK(cudaStreamCreateWithPriority(&aux_st, cudaStreamNonBlocking, hi));
    }
    device = dev;
    return 0;
  }
  int need_pcm(size_t samples) {
    if (d_pcm_cap >= samples) return 0;
    cudaFree(d_pcm); d_pcm = nullptr; d_pcm_cap = 0;
    CK(cudaMalloc(&d_pcm, sizeof(int16_t) * samples));
    d_pcm_cap = samples;
    return 0;
  }
  int need_out(size_t bytes) {
    if (d_out_cap >= bytes) return 0;
    cudaFree(d_out); d_out = nullptr; d_out_cap = 0;
    CK(cudaMalloc(&d_out, bytes));
    d_out_cap = bytes;
    return 0;
  }
  int need_crc(int ranges) {
    if (crc_cap >= ranges) return 0;
    cudaFree(d_crc_ranges); d_crc_ranges = nullptr; cudaFree(d_crc); d_crc = nullptr; crc_cap = 0;
    CK(cudaMalloc(&d_crc_ranges, sizeof(long long) * 2 * (size_t)ranges));
    CK(cudaMalloc(&d_crc, sizeof(unsigned) * (size_t)ranges));
    crc_cap = ranges;
    return 0;
  }
  int need_pin(size_t bytes) {
    if (h_pin_cap >= bytes) return 0;
    cudaFreeHost(h_pin); h_pin = nullptr; h_pin_cap = 0;
    CK(cudaMallocHost(&h_pin, bytes));
    h_pin_cap = bytes;
    return 0;
  }
};
thread_local ThreadCtx t_ctx;

/* MP3B200_DEBUG_SYNC=1: synchronise after every launch and name the failing kernel */
bool debug_sync() { static int v = -1; if (v < 0) { const char* e = getenv("MP3B200_DEBUG_SYNC"); v = (e && e[0] == '1') ? 1 : 0; } return v == 1; }
#define DBG(name)                                                                           \
  do {                                                                                      \
    if (debug_sync()) {                                                                     \
      cudaError_t e_ = cudaStreamSynchronize(st);                                           \
      if (e_ == cudaSuccess) e_ = cudaGetLastError();                                       \
      if (e_ != cudaSuccess) { g_err = std::string(name) + ": " + cudaGetErrorString(e_); return MP3B200_ERR_CUDA; } \
    }                                                                                       \
  } while (0)

struct Timings { float psy = 0, scan = 0, mask = 0, fb = 0, q1 = 0, qn = 0, total = 0; int passes = 0;
                 float q_prepare = 0, q_search = 0, q_outer = 0, q_finish = 0, q_pack = 0, q_mid = 0; };

/* Runs the whole pipeline for the streams described in `h_streams` (device pointers already set).
 * d_out: device output buffer.  force_bt: optional host array [units][nch] of block types (debug). */
/* pcm_chunks > 1: the caller uploads each stream's PCM in that many time slices on another stream and records
 * pcm_ready[j] after slice j; the psy analysis of slice j starts as soon as it has landed. */
struct PcmArrival { int chunks = 1; cudaEvent_t* ready = nullptr; };

/* All launches go to the calling thread's stream (t_ctx.st), which first waits for whatever the caller queued on the
 * legacy default stream (torch and plain CUDA callers produce their device buffers there); the call returns after the
 * stream has drained, so the results are visible to any stream afterwards. */
int run_pipeline(Config* cfg, Workspace& ws, std::vector<StreamDesc>& h_streams, uint8_t* d_out, const int32_t* force_bt,
                 bool stop_after_mdct, Timings* tm, const PcmArrival* arrival = nullptr, bool sync = true) {
  cudaStream_t st = t_ctx.st;
  cudaEvent_t* ev = t_ctx.ev;

  const int S = (int)h_streams.size();
  const int nch = cfg->host.nch;
  int max_frames = 0;
  long long total_frames = 0;          /* rows actually used this launch (the workspace may be larger) */
  int scan_rows = 0;
  int streams_with_frames = 0;
  for (auto& s : h_streams) {
    max_frames = s.nframes > max_frames ? s.nframes : max_frames;
    total_frames += s.nframes;
    streams_with_frames += s.nframes > 0 ? 1 : 0;
    s.scan_base = scan_rows;
    scan_rows += (s.nframes + SCAN_FRAMES - 1) / SCAN_FRAMES;
  }
  if (S == 0 || total_frames == 0) { if (tm) *tm = Timings(); return 0; }   /* empty batch: nothing to launch */
  if (S > MP3_MAX_LAUNCH_STREAMS) { g_err = "internal: more streams in one pipeline launch than a grid dimension holds"; return MP3B200_ERR_CUDA; }
  CK(cudaEventRecord(t_ctx.ev_in, cudaStreamLegacy));
  CK(cudaStreamWaitEvent(st, t_ctx.ev_in, 0));
  CK(cudaMemcpyAsync(ws.d_streams, h_streams.data(), sizeof(StreamDesc) * S, cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(ev[0], st));

  /* K2: psy analysis, one block per (granule incl. 1 halo, channel, stream) */
  {
    const int nchunks = arrival ? arrival->chunks : 1;
    /* units (relative index, -1 = halo) each upload slice completes, over all streams: the kernel's own rule
     * (k_psy_analysis) evaluated on the host, so that a slice's launch covers only its range of units */
    int u_lo[MP3_MAX_PCM_CHUNKS], u_hi[MP3_MAX_PCM_CHUNKS];
    const int G = cfg->host.mode_gr;     /* granules ("units") per frame */
    for (int j = 0; j < nchunks; j++) { u_lo[j] = G * max_frames; u_hi[j] = -1; }
    if (nchunks > 1) {
      for (const auto& sd : h_streams) {
        const long long n = sd.pcm_end - sd.pcm_base;
        for (int u = -1; u < G * sd.nframes; u++) {
          long long last = 576 * ((long long)G * sd.frame0 + u) - 224 + 1023 - sd.pcm_base;
          if (last > n - 1) last = n - 1;
          int mine = 0;
          while (mine < nchunks - 1 && last >= n * (mine + 1) / nchunks) mine++;
          if (u < u_lo[mine]) u_lo[mine] = u;
          if (u + 1 > u_hi[mine]) u_hi[mine] = u + 1;
        }
      }
    } else { u_lo[0] = -1; u_hi[0] = G * max_frames; }
    for (int j = 0; j < nchunks; j++) {
      if (arrival) CK(cudaStreamWaitEvent(st, arrival->ready[j], 0));
      if (u_hi[j] <= u_lo[j]) continue;
      dim3 gridj(u_hi[j] - u_lo[j], nch, S);
      k_psy_analysis<<<gridj, PSY_THREADS, 0, st>>>(cfg->dev, ws.d_streams, ws.d_psy, j, nchunks, u_lo[j]);
      g_launches++;
      DBG("k_psy_analysis");
    }
  }
  CK(cudaEventRecord(ev[1], st));
  /* K3a: attack pre-pass (parallel) + sequential per-stream scans */
  {
    dim3 grid((cfg->host.mode_gr * max_frames + 127) / 128, 1, S);
    k_attack_prepass<<<grid, 128, 0, st>>>(cfg->dev, ws.d_streams, ws.d_psy, ws.d_scan_in);
    DBG("k_attack_prepass");
    k_stream_scan<<<S, SCAN_THREADS, 0, st>>>(cfg->dev, ws.d_streams, S, ws.d_scan_in, ws.d_bt_final, ws.d_bt_prev, ws.d_ath_psy, ws.d_ath_q, ws.d_scan);
    g_launches += 2;
    DBG("k_stream_scan");
    /* K1a: subband analysis, programmatic dependent of the scan (reads nothing the scan writes; see k_stream_scan) */
    {
      const int G = cfg->host.mode_gr;
      const size_t smem = sizeof(double) * FB_PCM_WORDS + sizeof(float) * (FB_SLABS * 18 * FB_SLAB_STRIDE);
      {
        std::lock_guard<std::mutex> lk(g_mu);   /* the attribute is per device */
        if (!g_fb_attr_done[cfg->device]) { CK(cudaFuncSetAttribute(k_subband_analysis, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); g_fb_attr_done[cfg->device] = true; }
      }
      cudaLaunchConfig_t lc = {};
      lc.gridDim = dim3((G * max_frames + 1 + FB_SLABS - 1) / FB_SLABS, nch, S);
      lc.blockDim = dim3(FB_THREADS); lc.dynamicSmemBytes = smem; lc.stream = st;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      at[0].val.programmaticStreamSerializationAllowed = 1;
      lc.attrs = at; lc.numAttrs = 1;
      CK(cudaLaunchKernelEx(&lc, k_subband_analysis, (const Mp3Tables*)cfg->dev, (const StreamDesc*)ws.d_streams, ws.d_slab));
      g_launches++;
      DBG("k_subband_analysis");
    }
  }
  CK(cudaEventRecord(ev[2], st));
  if (force_bt) {   /* debug: override block decision for the filterbank */
    std::vector<signed char> bt((size_t)ws.units * 2, 0);
    for (long long u = 0; u < ws.units; u++)
      for (int c = 0; c < nch; c++) bt[u * 2 + c] = (signed char)force_bt[u * nch + c];
    CK(cudaMemcpyAsync(ws.d_bt_final, bt.data(), bt.size(), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
  }
  /* K3b: masking thresholds */
  {
    dim3 grid(cfg->host.mode_gr * max_frames + 1, 1, S);
    k_psy_masking<<<grid, MASK_THREADS, 0, st>>>(cfg->dev, ws.d_streams, ws.d_psy, ws.d_bt_prev, ws.d_ath_psy, ws.d_ratio);
    g_launches++;
    DBG("k_psy_masking");
  }
  CK(cudaEventRecord(ev[3], st));
  /* K1b: MDCT from the slabs and the block types.  (As a programmatic dependent of the masking kernel, running beside it:
   * it saves only a few microseconds for the pair -- not worth losing the per-kernel times.) */
  {
    dim3 grid((cfg->host.mode_gr * max_frames + FB_G - 1) / FB_G, nch, S);
    k_mdct<<<grid, FB_G * 32, 0, st>>>(cfg->dev, ws.d_streams, ws.d_slab, ws.d_bt_final, ws.d_xr);
    g_launches++;
    DBG("k_mdct");
  }
  CK(cudaEventRecord(ev[4], st));
  int passes = 0;
  if (!stop_after_mdct) {
    QuantBuffers qb;
    qb.xr = ws.d_xr; qb.ratio = ws.d_ratio; qb.bt = ws.d_bt_final; qb.ath_q = ws.d_ath_q; qb.qs = ws.d_qstate; qb.ginfo = ws.d_ginfo;
    qb.l3enc = ws.d_l3enc; qb.xrq = ws.d_xrq; qb.xrpow = ws.d_xrpow; qb.neg = ws.d_neg; qb.prep = ws.d_prep; qb.list = ws.d_dirty; qb.counter = ws.d_counter;
    int rc = quant_run(cfg->dev, cfg->host, ws.d_streams, S, streams_with_frames, max_frames, total_frames, qb, d_out, st, t_ctx.aux_st, t_ctx.ev_fork, t_ctx.ev_join, ev[5], t_ctx.evq, t_ctx.evq_pred, &passes, &g_launches);
    if (rc) { g_err = "quantizer stage failed: " + std::string(cudaGetErrorString(cudaGetLastError())); return rc; }
  } else {
    CK(cudaEventRecord(ev[5], st));
  }
  CK(cudaEventRecord(ev[6], st));
  if (!sync) return 0;                     /* the caller queues its copies behind the kernels and synchronises once */
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
  if (tm) {
    cudaEventElapsedTime(&tm->psy, ev[0], ev[1]);
    cudaEventElapsedTime(&tm->scan, ev[1], ev[2]);
    cudaEventElapsedTime(&tm->mask, ev[2], ev[3]);
    cudaEventElapsedTime(&tm->fb, ev[3], ev[4]);
    cudaEventElapsedTime(&tm->q1, ev[4], ev[5]);
    cudaEventElapsedTime(&tm->qn, ev[5], ev[6]);
    cudaEventElapsedTime(&tm->total, ev[0], ev[6]);
    tm->passes = passes;
    if (!stop_after_mdct && passes > 0) {
      auto span = [&](int slot) { float v = 0; const int p = t_ctx.evq_pred[slot]; if (p >= 0) cudaEventElapsedTime(&v, t_ctx.evq[p], t_ctx.evq[slot]); return v; };
      tm->q_prepare = span(QE_PREP);
      tm->q_search = span(QE_S0) + span(QE_S1);
      tm->q_outer = span(QE_O0) + span(QE_O1);
      tm->q_finish = span(QE_F0) + span(QE_F1);
      tm->q_pack = span(QE_PK);
      tm->q_mid = span(QE_MID);
    }
  }
  return 0;
}

void init_stream_state(StreamDesc& sd) {   /* lame_init_old + psymodel_init start values */
  sd.ath_adjust = 0.01; sd.ath_adjust_limit = 1.0;
  sd.blocktype_old[0] = sd.blocktype_old[1] = BT_NORM;
  sd.last_attacks[0] = sd.last_attacks[1] = 0;
  sd.old_value[0] = sd.old_value[1] = 180;
  sd.current_step[0] = sd.current_step[1] = 4;
}

long long bytes_for(const Mp3Tables& t, long long frames) {
  return frames * t.frame_bytes_nopad + pad_count(frames - 1, t.frac_SpF, t.samplerate);
}

}  // namespace

extern "C" {

const char* mp3b200_last_error(void) { return g_err.c_str(); }
#ifdef Q_STATS
int mp3b200_debug_qstats(unsigned long long* out16, int reset) {
  if (cudaMemcpyFromSymbol(out16, g_qstats, sizeof(unsigned long long) * 16) != cudaSuccess) return MP3B200_ERR_CUDA;
  if (reset) { unsigned long long z[16] = {0}; cudaMemcpyToSymbol(g_qstats, z, sizeof z); }
  return 0;
}
#endif
int64_t mp3b200_launch_count(void) { return g_launches; }

int mp3b200_set_device(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n || device >= MP3_MAX_DEVICES) { g_err = "invalid CUDA device"; return MP3B200_ERR_CUDA; }
  std::lock_guard<std::mutex> lk(g_mu);
  g_device = device;      /* existing handles keep the device they were created on */
  return 0;
}

int64_t mp3b200_stream_frames(int64_t nsamples) { return frames_for(nsamples, 2); }

namespace {
/* the byte geometry of a configuration is three integers; building the full tables costs ~1 ms, so it is done once */
ByteGeom byte_geom(int channels, int samplerate, int kbps) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto key = std::make_tuple(channels, samplerate, kbps);
  auto it = g_byte_geom.find(key);
  if (it != g_byte_geom.end()) return it->second;
  Mp3Tables* t = new Mp3Tables();
  const int rc = mp3_build_tables(channels, samplerate, kbps, t);
  ByteGeom g = rc == 0 ? ByteGeom{t->frame_bytes_nopad, t->frac_SpF, t->mode_gr} : ByteGeom{-1, 0, 2};
  delete t;
  g_byte_geom[key] = g;
  return g;
}
}  // namespace

int64_t mp3b200_stream_bytes(int channels, int samplerate, int kbps, int64_t nsamples) {
  const ByteGeom g = byte_geom(channels, samplerate, kbps);
  if (g.frame_bytes_nopad < 0 || nsamples < 0) return -1;
  const long long frames = frames_for(nsamples, g.mode_gr);
  return frames * g.frame_bytes_nopad + pad_count(frames - 1, g.frac_SpF, samplerate);
}

int64_t mp3b200_stream_frames_cfg(int channels, int samplerate, int kbps, int64_t nsamples) {
  const ByteGeom g = byte_geom(channels, samplerate, kbps);
  if (g.frame_bytes_nopad < 0 || nsamples < 0) return -1;
  return frames_for(nsamples, g.mode_gr);
}

int mp3b200_granules_per_frame(int channels, int samplerate, int kbps) {
  const ByteGeom g = byte_geom(channels, samplerate, kbps);
  return g.frame_bytes_nopad < 0 ? -1 : g.mode_gr;
}

}  // extern "C"

namespace {
int encode_streams_device_impl(Config* cfg, int channels, int nstreams, const int16_t* d_pcm, const int64_t* pcm_off,
                               const int64_t* nsamples, uint8_t* d_out, const int64_t* out_off, float* timings_ms,
                               const PcmArrival* arrival) {
  int rc = 0;
  if (timings_ms) for (int i = 0; i < 16; i++) timings_ms[i] = 0.0f;
  /* Streams are independent: a batch wider than one launch can hold runs as consecutive groups on the thread's stream.
   * The times add up over the groups; the pass count is the largest any group needed. */
  for (int g0 = 0; g0 < nstreams; g0 += MP3_MAX_LAUNCH_STREAMS) {
    const int n = nstreams - g0 < MP3_MAX_LAUNCH_STREAMS ? nstreams - g0 : MP3_MAX_LAUNCH_STREAMS;
    std::vector<StreamDesc> sds(n);
    long long U = 0, F = 0;
    for (int i = 0; i < n; i++) {
      const int s = g0 + i;
      StreamDesc& sd = sds[i];
      memset(&sd, 0, sizeof sd);
      sd.pcm[0] = d_pcm + pcm_off[s];
      sd.pcm[1] = channels == 2 ? d_pcm + pcm_off[s] + nsamples[s] : sd.pcm[0];
      sd.pcm_base = 0; sd.pcm_end = nsamples[s];
      sd.frame0 = 0; sd.nframes = (int)frames_for(nsamples[s], cfg->host.mode_gr);
      sd.unit_base = (int)U; sd.frame_base = (int)F;
      sd.out_base = out_off[s];
      init_stream_state(sd);
      U += (long long)cfg->host.mode_gr * sd.nframes; F += sd.nframes;
    }
    if (F == 0) continue;                     /* empty group: nothing to launch */
    Workspace& ws = t_ctx.ws;
    if (ws.units < U || ws.frames < F || ws.nstreams < n || ws.nch != cfg->host.nch) {
      rc = ws.alloc(n, cfg->host.nch, U, F, false);
      if (rc) return rc;
    }
    Timings tm;
    rc = run_pipeline(cfg, ws, sds, d_out, nullptr, false, &tm, arrival);
    if (rc) return rc;
    arrival = nullptr;                        /* the later groups run behind the first one, after every upload landed */
    if (timings_ms) {
      const float t[16] = {tm.psy, tm.scan, tm.mask, tm.fb, tm.q1, tm.qn, tm.total, 0.0f,
                           tm.q_prepare, tm.q_search, tm.q_outer, tm.q_finish, tm.q_pack, tm.q_mid, 0.0f, 0.0f};
      for (int i = 0; i < 16; i++) timings_ms[i] += t[i];
      if ((float)tm.passes > timings_ms[7]) timings_ms[7] = (float)tm.passes;
    }
  }
  return 0;
}

}  // namespace

extern "C" {

int mp3b200_encode_streams_device(int channels, int samplerate, int kbps, int nstreams, const int16_t* d_pcm,
                                  const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                  const int64_t* out_off, float* timings_ms) {
  if (nstreams < 0) { g_err = "negative stream count"; return MP3B200_ERR_HANDLE; }
  Config* cfg;
  int rc = get_config(channels, samplerate, kbps, &cfg);
  if (rc) return rc;
  rc = t_ctx.use(cfg->device);
  if (rc) return rc;
  return encode_streams_device_impl(cfg, channels, nstreams, d_pcm, pcm_off, nsamples, d_out, out_off, timings_ms, nullptr);
}

int mp3b200_encode_streams(int channels, int samplerate, int kbps, int nstreams, const int16_t* const* left,
                           const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                           const int64_t* cap, int64_t* out_bytes) {
  if (nstreams < 0) { g_err = "negative stream count"; return MP3B200_ERR_HANDLE; }
  Config* cfg;
  int rc = get_config(channels, samplerate, kbps, &cfg);
  if (rc) return rc;
  std::vector<int64_t> pcm_off(nstreams), out_off(nstreams);
  long long tot_samples = 0, tot_bytes = 0;
  for (int s = 0; s < nstreams; s++) {
    pcm_off[s] = tot_samples;
    tot_samples += nsamples[s] * channels;
    out_off[s] = tot_bytes;
    const long long b = bytes_for(cfg->host, frames_for(nsamples[s], cfg->host.mode_gr));
    if (cap[s] < b) { g_err = "output buffer too small"; return MP3B200_ERR_BUFFER; }
    out_bytes[s] = b;
    tot_bytes += b;
  }
  if (nstreams == 0) return MP3B200_OK;
  rc = t_ctx.use(cfg->device);
  if (rc) return rc;
  /* grow-only staging buffers: a steady stream of batches does not pay cudaMalloc/cudaFree per call */
  rc = t_ctx.need_pcm((size_t)tot_samples + 8);
  if (rc) return rc;
  rc = t_ctx.need_out((size_t)tot_bytes + 8);
  if (rc) return rc;
  int16_t* d_pcm = t_ctx.d_pcm;
  uint8_t* d_out = t_ctx.d_out;
  /* Upload in time slices on a copy stream; the psy analysis of a slice starts when it has landed, so only the first
   * slice's transfer is exposed.  Many small streams are uploaded whole (one slice): per-copy overhead would win. */
  PcmArrival arr;
  arr.chunks = (nstreams <= 8 && tot_samples >= (1 << 20)) ? MP3_MAX_PCM_CHUNKS : 1;
  arr.ready = t_ctx.ready;
  for (int j = 0; j < arr.chunks; j++) {
    for (int s = 0; s < nstreams; s++) {
      const int64_t lo = nsamples[s] * j / arr.chunks, hi = nsamples[s] * (j + 1) / arr.chunks;
      if (hi <= lo) continue;
      CK(cudaMemcpyAsync(d_pcm + pcm_off[s] + lo, left[s] + lo, sizeof(int16_t) * (hi - lo), cudaMemcpyHostToDevice, t_ctx.up_st));
      if (channels == 2)
        CK(cudaMemcpyAsync(d_pcm + pcm_off[s] + nsamples[s] + lo, right[s] + lo, sizeof(int16_t) * (hi - lo), cudaMemcpyHostToDevice, t_ctx.up_st));
    }
    CK(cudaEventRecord(t_ctx.ready[j], t_ctx.up_st));
  }
  rc = encode_streams_device_impl(cfg, channels, nstreams, d_pcm, pcm_off.data(), nsamples, d_out, out_off.data(), nullptr, &arr);
  if (rc == 0) {
    for (int s = 0; s < nstreams; s++)
      if (cudaMemcpyAsync(out[s], d_out + out_off[s], (size_t)out_bytes[s], cudaMemcpyDeviceToHost, t_ctx.st) != cudaSuccess) rc = MP3B200_ERR_CUDA;
    if (cudaStreamSynchronize(t_ctx.st) != cudaSuccess) rc = MP3B200_ERR_CUDA;
  }
  return rc;
}

int mp3b200_debug_stages(int channels, int samplerate, int kbps, const int16_t* left, const int16_t* right,
                         int64_t nsamples, const int32_t* force_blocktype, float* xr, int32_t* blocktype,
                         float* en_l, float* thm_l, float* en_s, float* thm_s, double* ath_adjust,
                         int32_t* l3_enc, int32_t* ginfo, uint8_t* bytes_out, int64_t bytes_cap) {
  mp3b200_debug_taps t;
  memset(&t, 0, sizeof t);
  t.size = (int32_t)sizeof t; t.channels = channels; t.samplerate = samplerate; t.kbps = kbps;
  t.left = left; t.right = right; t.nsamples = nsamples; t.force_blocktype = force_blocktype;
  t.xr = xr; t.blocktype = blocktype; t.en_l = en_l; t.thm_l = thm_l; t.en_s = en_s; t.thm_s = thm_s; t.ath_adjust = ath_adjust;
  t.l3_enc = l3_enc; t.ginfo = ginfo; t.bytes_out = bytes_out; t.bytes_cap = bytes_cap;
  return mp3b200_debug_stages_ex(&t);
}

int mp3b200_debug_stages_ex(const mp3b200_debug_taps* tp) {
  if (!tp || tp->size != (int32_t)sizeof(mp3b200_debug_taps)) { g_err = "mp3b200_debug_taps: size must be sizeof(mp3b200_debug_taps)"; return MP3B200_ERR_HANDLE; }
  const int channels = tp->channels;
  const int16_t *left = tp->left, *right = tp->right;
  const int64_t nsamples = tp->nsamples;
  const int32_t* force_blocktype = tp->force_blocktype;
  float *xr = tp->xr, *en_l = tp->en_l, *thm_l = tp->thm_l, *en_s = tp->en_s, *thm_s = tp->thm_s;
  int32_t *blocktype = tp->blocktype, *l3_enc = tp->l3_enc, *ginfo = tp->ginfo;
  double* ath_adjust = tp->ath_adjust;
  uint8_t* bytes_out = tp->bytes_out;
  const int64_t bytes_cap = tp->bytes_cap;
  Config* cfg;
  int rc = get_config(channels, tp->samplerate, tp->kbps, &cfg);
  if (rc) return rc;
  rc = t_ctx.use(cfg->device);
  if (rc) return rc;
  const int nch = cfg->host.nch;
  const int G = cfg->host.mode_gr;
  const long long F = frames_for(nsamples, G), U = G * F;
  int16_t* d_pcm = nullptr; uint8_t* d_out = nullptr;
  CK(cudaMalloc(&d_pcm, sizeof(int16_t) * (size_t)(nsamples * nch + 8)));
  CK(cudaMemcpy(d_pcm, left, sizeof(int16_t) * nsamples, cudaMemcpyHostToDevice));
  if (nch == 2) CK(cudaMemcpy(d_pcm + nsamples, right, sizeof(int16_t) * nsamples, cudaMemcpyHostToDevice));
  const long long nbytes = bytes_for(cfg->host, F);
  CK(cudaMalloc(&d_out, (size_t)nbytes + 8));
  CK(cudaMemset(d_out, 0, (size_t)nbytes + 8));
  std::vector<StreamDesc> sds(1);
  StreamDesc& sd = sds[0];
  memset(&sd, 0, sizeof sd);
  sd.pcm[0] = d_pcm; sd.pcm[1] = nch == 2 ? d_pcm + nsamples : d_pcm;
  sd.pcm_end = nsamples; sd.nframes = (int)F;
  init_stream_state(sd);
  Workspace ws;
  rc = ws.alloc(1, nch, U, F, true);
  if (rc) { cudaFree(d_pcm); cudaFree(d_out); return rc; }
  const bool want_gi = ginfo || tp->scalefac || tp->subblock_gain;
  const bool want_prep = tp->xmin || tp->max_nonzero_coeff || tp->xrpow_max;
  const bool want_q = tp->scfsi || tp->old_value || tp->cur_step;
  const bool only_mdct = !(l3_enc || bytes_out || want_gi || want_prep || want_q);
  rc = run_pipeline(cfg, ws, sds, d_out, force_blocktype, only_mdct, nullptr);
  if (rc == 0) {
    if (xr) CK(cudaMemcpy(xr, ws.d_xr, sizeof(float) * (size_t)U * nch * 576, cudaMemcpyDeviceToHost));
    if (blocktype) {
      std::vector<signed char> bt((size_t)U * 2);
      CK(cudaMemcpy(bt.data(), ws.d_bt_final, bt.size(), cudaMemcpyDeviceToHost));
      for (long long u = 0; u < U; u++) for (int c = 0; c < nch; c++) blocktype[u * nch + c] = bt[u * 2 + c];
    }
    if (en_l || thm_l || en_s || thm_s) {
      /* masking used by granule u is the ratio of psy unit u-1: row (u + 1 - 1) of the halo-shifted array */
      std::vector<PsyRatioDev> r((size_t)(U + 1) * nch);
      CK(cudaMemcpy(r.data(), ws.d_ratio, sizeof(PsyRatioDev) * r.size(), cudaMemcpyDeviceToHost));
      for (long long u = 0; u < U; u++) for (int c = 0; c < nch; c++) {
        const PsyRatioDev& q = r[(size_t)u * nch + c];
        if (en_l) memcpy(en_l + (u * nch + c) * 22, q.en_l, sizeof q.en_l);
        if (thm_l) memcpy(thm_l + (u * nch + c) * 22, q.thm_l, sizeof q.thm_l);
        if (en_s) memcpy(en_s + (u * nch + c) * 39, q.en_s, sizeof q.en_s);
        if (thm_s) memcpy(thm_s + (u * nch + c) * 39, q.thm_s, sizeof q.thm_s);
      }
    }
    if (ath_adjust) CK(cudaMemcpy(ath_adjust, ws.d_ath_q, sizeof(double) * (size_t)F, cudaMemcpyDeviceToHost));
    if (l3_enc) {
      std::vector<short> t((size_t)U * nch * 576);
      CK(cudaMemcpy(t.data(), ws.d_l3enc, sizeof(short) * t.size(), cudaMemcpyDeviceToHost));
      for (size_t i = 0; i < t.size(); i++) l3_enc[i] = t[i];
    }
    if (want_gi) {
      std::vector<GranuleInfoDev> g((size_t)U * nch);
      CK(cudaMemcpy(g.data(), ws.d_ginfo, sizeof(GranuleInfoDev) * g.size(), cudaMemcpyDeviceToHost));
      for (size_t i = 0; i < g.size(); i++) {
        if (ginfo) {
          int32_t* o = ginfo + i * 16;
          o[0] = g[i].global_gain; o[1] = g[i].part2_3_length; o[2] = g[i].part2_length; o[3] = g[i].big_values;
          o[4] = g[i].count1; o[5] = g[i].scalefac_compress; o[6] = g[i].table_select[0]; o[7] = g[i].table_select[1];
          o[8] = g[i].table_select[2]; o[9] = g[i].region0_count; o[10] = g[i].region1_count; o[11] = g[i].preflag;
          o[12] = g[i].scalefac_scale; o[13] = g[i].count1table_select; o[14] = g[i].block_type; o[15] = 0;
        }
        if (tp->scalefac) memcpy(tp->scalefac + i * MP3_SFBMAX, g[i].scalefac, sizeof(int32_t) * MP3_SFBMAX);
        if (tp->subblock_gain) for (int k = 0; k < 3; k++) tp->subblock_gain[i * 3 + k] = g[i].subblock_gain[k];
      }
    }
    if (want_prep) {
      /* the prepared granule-channel as k_q_prepare left it for the searches and rate loops; xmin is defined for the psymax
       * bands of granules with energy only (the others never reach calc_xmin) */
      std::vector<GcPrep> p((size_t)U * nch);
      CK(cudaMemcpy(p.data(), ws.d_prep, sizeof(GcPrep) * p.size(), cudaMemcpyDeviceToHost));
      for (size_t i = 0; i < p.size(); i++) {
        if (tp->xmin) {
          const int psymax = p[i].block_type == BT_SHORT ? 36 : 21;
          for (int k = 0; k < MP3_SFBMAX; k++) tp->xmin[i * MP3_SFBMAX + k] = (p[i].have && k < psymax) ? p[i].xmin[k] : 0.0f;
        }
        if (tp->max_nonzero_coeff) tp->max_nonzero_coeff[i] = p[i].mnz;
        if (tp->xrpow_max) tp->xrpow_max[i] = p[i].xrpow_max;
      }
    }
    if (want_q) {
      std::vector<QuantFrameState> q((size_t)F);
      CK(cudaMemcpy(q.data(), ws.d_qstate, sizeof(QuantFrameState) * q.size(), cudaMemcpyDeviceToHost));
      for (long long f = 0; f < F; f++) {
        const QuantFrameState& s = q[(size_t)f];
        for (int c = 0; c < nch; c++) {
          if (tp->scfsi) for (int b = 0; b < 4; b++) tp->scfsi[(f * nch + c) * 4 + b] = s.scfsi[c][b];
          /* [in, after gr0 (MPEG-1 only: bs_* is the state gr1's search started from), out] */
          const int ov[3] = {s.in_old[c], G == 2 ? s.bs_gain0[c] : 0, s.out_old[c]};
          const int cs[3] = {s.in_step[c], G == 2 ? s.bs_step0[c] : 0, s.out_step[c]};
          for (int k = 0; k < 3; k++) {
            if (tp->old_value) tp->old_value[(f * 3 + k) * nch + c] = ov[k];
            if (tp->cur_step) tp->cur_step[(f * 3 + k) * nch + c] = cs[k];
          }
        }
      }
    }
    if (bytes_out) {
      if (bytes_cap < nbytes) { g_err = "output buffer too small"; rc = MP3B200_ERR_BUFFER; }
      else CK(cudaMemcpy(bytes_out, d_out, (size_t)nbytes, cudaMemcpyDeviceToHost));
    }
  }
  cudaFree(d_pcm); cudaFree(d_out);
  return rc;
}

}  // extern "C"

/* ---- container / metadata step (SURVEY.md 8(f3)): music CRC on the device, tag frames on the host ---- */
namespace {
CrcTables g_crc_host;                              /* byte table + zero-byte powers (k_tag.cuh), built once */
bool g_crc_host_ready = false;
CrcTables* g_crc_dev[MP3_MAX_DEVICES] = {};        /* per device copy */

const CrcTables& crc_host() {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_crc_host_ready) { crc_host_tables(&g_crc_host); g_crc_host_ready = true; }
  return g_crc_host;
}

/* CRC-16 (start 0) of the byte ranges [off[i], off[i] + len[i]) of d_buf, one k_music_crc launch per 65535 ranges, on the
 * calling thread's stream behind whatever wrote the bytes.  crc[i] is valid when the call returns. */
int music_crc_ranges(int device, const uint8_t* d_buf, const std::vector<long long>& off, const std::vector<long long>& len, std::vector<unsigned>& crc) {
  const int R = (int)off.size();
  crc.assign((size_t)R, 0u);
  if (R == 0) return 0;
  const CrcTables& ht = crc_host();
  {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_crc_dev[device]) {
      CK(cudaMalloc(&g_crc_dev[device], sizeof(CrcTables)));
      CK(cudaMemcpy(g_crc_dev[device], &ht, sizeof(CrcTables), cudaMemcpyHostToDevice));
    }
  }
  ThreadCtx& sc = t_ctx;
  int rc = sc.need_crc(R);
  if (rc) return rc;
  std::vector<long long> ranges((size_t)2 * R);
  long long longest = 0;
  for (int i = 0; i < R; i++) { ranges[i] = off[i]; ranges[(size_t)R + i] = len[i]; longest = len[i] > longest ? len[i] : longest; }
  CK(cudaMemcpyAsync(sc.d_crc_ranges, ranges.data(), sizeof(long long) * ranges.size(), cudaMemcpyHostToDevice, sc.st));
  CK(cudaMemsetAsync(sc.d_crc, 0, sizeof(unsigned) * (size_t)R, sc.st));
  if (longest > 0) {
    const long long pieces = (longest + CRC_PIECE_BYTES - 1) / CRC_PIECE_BYTES;
    for (int r0 = 0; r0 < R; r0 += 65535) {
      const int nr = R - r0 < 65535 ? R - r0 : 65535;
      dim3 grid((unsigned)((pieces + CRC_WARPS - 1) / CRC_WARPS), (unsigned)nr);
      k_music_crc<<<grid, CRC_WARPS * 32, 0, sc.st>>>(d_buf, sc.d_crc_ranges + r0, sc.d_crc_ranges + R + r0, g_crc_dev[device], sc.d_crc + r0);
      g_launches++;
    }
  }
  CK(cudaMemcpyAsync(crc.data(), sc.d_crc, sizeof(unsigned) * (size_t)R, cudaMemcpyDeviceToHost, sc.st));
  CK(cudaStreamSynchronize(sc.st));
  CK(cudaGetLastError());
  return 0;
}
}  // namespace

extern "C" {

int mp3b200_wav_read_header(const uint8_t* data, int64_t len, mp3b200_wav_header* out) {
  if (!out || len < 0 || (len > 0 && !data)) return MP3B200_ERR_HANDLE;
  long long off = 0, dl = 0; int ch = 0; unsigned sr = 0;
  const int rc = mp3_wav_read_header(data, len, &off, &dl, &ch, &sr);
  out->data_offset = off; out->data_len = dl; out->channels = ch; out->sample_rate = sr;
  return rc;
}

/* CRC-16 of byte ranges of a DEVICE buffer (test / bench tap of k_music_crc): crc[i] for [off[i], off[i] + len[i]);
 * ms (optional) = CUDA-event time of the launch(es) on the library's stream, tables already resident. */
int mp3b200_debug_music_crc(const uint8_t* d_buf, const int64_t* off, const int64_t* len, int nranges, uint32_t* crc, float* ms) {
  if (nranges < 0 || (nranges > 0 && (!d_buf || !off || !len || !crc))) return MP3B200_ERR_HANDLE;
  int dev = 0;
  { std::lock_guard<std::mutex> lk(g_mu); dev = g_device; int rc = ensure_device(dev); if (rc) return rc; }
  int rc = t_ctx.use(dev);
  if (rc) return rc;
  std::vector<long long> o(off, off + nranges), l(len, len + nranges);
  std::vector<unsigned> c;
  CK(cudaEventRecord(t_ctx.ev_in, cudaStreamLegacy));
  CK(cudaStreamWaitEvent(t_ctx.st, t_ctx.ev_in, 0));
  rc = music_crc_ranges(dev, d_buf, o, l, c);              /* first call: uploads the tables */
  if (rc) return rc;
  if (ms) {
    CK(cudaEventRecord(t_ctx.ev[0], t_ctx.st));
    rc = music_crc_ranges(dev, d_buf, o, l, c);
    if (rc) return rc;
    CK(cudaEventRecord(t_ctx.ev[1], t_ctx.st));
    CK(cudaEventSynchronize(t_ctx.ev[1]));
    CK(cudaEventElapsedTime(ms, t_ctx.ev[0], t_ctx.ev[1]));
  }
  for (int i = 0; i < nranges; i++) crc[i] = c[i];
  return 0;
}

int mp3b200_get_vbr_tag(const uint8_t* frame, int64_t len, mp3b200_vbr_tag_data* out) {
  if (!out || len < 0 || (len > 0 && !frame)) return MP3B200_ERR_HANDLE;
  Mp3VbrTagData t;
  const int rc = mp3_tag_parse(frame, len, &t);
  out->h_id = t.h_id; out->samprate = t.samprate; out->flags = t.flags; out->frames = t.frames; out->bytes = t.bytes;
  out->vbr_scale = t.vbr_scale; out->headersize = t.headersize; out->enc_delay = t.enc_delay; out->enc_padding = t.enc_padding;
  memcpy(out->toc, t.toc, 100);
  return rc;
}

int mp3b200_crc16_combine(int crc_a, int crc_b, int64_t len_b) {
  if (len_b < 0) return MP3B200_ERR_HANDLE;
  return (int)crc_append((unsigned)crc_a & 0xffffu, (unsigned)crc_b & 0xffffu, (unsigned long long)len_b, crc_host().pow);
}

int mp3b200_lametag_size(int channels, int samplerate, int kbps) {
  Mp3TagParams p;
  if (mp3_tag_params(channels, samplerate, kbps, &p) != 0) return MP3B200_ERR_CONFIG;
  return p.fits ? p.frame_bytes : 0;
}

int mp3b200_lametag_build(int channels, int samplerate, int kbps, int64_t nframes, int64_t music_bytes, int music_crc, int encoder_padding,
                          uint8_t* buf, int cap) {
  Mp3TagParams p;
  if (mp3_tag_params(channels, samplerate, kbps, &p) != 0) { g_err = "unsupported configuration"; return MP3B200_ERR_CONFIG; }
  if (!p.fits || nframes <= 0) return 0;
  if (!buf || cap < p.frame_bytes) return p.frame_bytes;              /* like getLameTagFrame: the size it needs */
  Mp3SeekBag* bag = new Mp3SeekBag();
  bag->reset();
  bag->add_frames(nframes, p.kbps);
  const int n = mp3_tag_frame(p, *bag, music_bytes, (unsigned)music_crc, encoder_padding, buf);
  delete bag;
  return n;
}

int mp3b200_encode_streams_tagged(int channels, int samplerate, int kbps, int nstreams, const int16_t* const* left,
                                  const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                                  const int64_t* cap, int64_t* out_bytes) {
  if (nstreams < 0) { g_err = "negative stream count"; return MP3B200_ERR_HANDLE; }
  Config* cfg;
  int rc = get_config(channels, samplerate, kbps, &cfg);
  if (rc) return rc;
  Mp3TagParams p;
  if (mp3_tag_params(channels, samplerate, kbps, &p) != 0) { g_err = "unsupported configuration"; return MP3B200_ERR_CONFIG; }
  const int tfs = p.fits ? p.frame_bytes : 0;
  std::vector<int64_t> pcm_off(nstreams), out_off(nstreams);
  std::vector<long long> frames(nstreams), audio(nstreams);
  long long tot_samples = 0, tot_bytes = 0;
  for (int s = 0; s < nstreams; s++) {
    pcm_off[s] = tot_samples; tot_samples += nsamples[s] * channels;
    out_off[s] = tot_bytes;
    frames[s] = frames_for(nsamples[s], cfg->host.mode_gr);
    audio[s] = bytes_for(cfg->host, frames[s]);
    if (cap[s] < audio[s] + tfs) { g_err = "output buffer too small"; return MP3B200_ERR_BUFFER; }
    out_bytes[s] = audio[s] + tfs;
    tot_bytes += audio[s];
  }
  if (nstreams == 0) return MP3B200_OK;
  rc = t_ctx.use(cfg->device);
  if (rc) return rc;
  rc = t_ctx.need_pcm((size_t)tot_samples + 8);
  if (rc) return rc;
  rc = t_ctx.need_out((size_t)tot_bytes + 8);
  if (rc) return rc;
  for (int s = 0; s < nstreams; s++) {
    if (nsamples[s] <= 0) continue;
    CK(cudaMemcpyAsync(t_ctx.d_pcm + pcm_off[s], left[s], sizeof(int16_t) * nsamples[s], cudaMemcpyHostToDevice, t_ctx.up_st));
    if (channels == 2)
      CK(cudaMemcpyAsync(t_ctx.d_pcm + pcm_off[s] + nsamples[s], (right && right[s]) ? right[s] : left[s], sizeof(int16_t) * nsamples[s], cudaMemcpyHostToDevice, t_ctx.up_st));
  }
  PcmArrival arr;
  arr.chunks = 1; arr.ready = t_ctx.ready;
  CK(cudaEventRecord(t_ctx.ready[0], t_ctx.up_st));
  rc = encode_streams_device_impl(cfg, channels, nstreams, t_ctx.d_pcm, pcm_off.data(), nsamples, t_ctx.d_out, out_off.data(), nullptr, &arr);
  if (rc) return rc;
  /* the music CRC of every stream, where the bytes are */
  std::vector<long long> off(out_off.begin(), out_off.end());
  std::vector<unsigned> crc;
  rc = music_crc_ranges(cfg->device, t_ctx.d_out, off, audio, crc);
  if (rc) return rc;
  Mp3SeekBag* bag = new Mp3SeekBag();
  for (int s = 0; s < nstreams; s++) {
    int wrote = 0;
    if (tfs > 0 && frames[s] > 0) {
      bag->reset();
      bag->add_frames(frames[s], p.kbps);
      wrote = mp3_tag_frame(p, *bag, audio[s], crc[s], mp3_encoder_padding(nsamples[s], cfg->host.mode_gr), out[s]);
    }
    out_bytes[s] = audio[s] + wrote;
    if (audio[s] > 0 && cudaMemcpyAsync(out[s] + wrote, t_ctx.d_out + out_off[s], (size_t)audio[s], cudaMemcpyDeviceToHost, t_ctx.st) != cudaSuccess) rc = MP3B200_ERR_CUDA;
  }
  delete bag;
  if (cudaStreamSynchronize(t_ctx.st) != cudaSuccess) rc = MP3B200_ERR_CUDA;
  return rc;
}

}  // extern "C"

#include "mp3_handle.inc"

#ifdef Q_TASKSTAT
extern "C" int mp3b200_debug_taskstat(int* out, int rows) {
  if (rows > (1 << 16)) rows = 1 << 16;
  return cudaMemcpyFromSymbol(out, g_taskstat, sizeof(int) * 8 * (size_t)rows) == cudaSuccess ? 0 : -1;
}
#endif
