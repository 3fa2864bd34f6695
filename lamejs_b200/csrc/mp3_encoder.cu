/* mp3_encoder.cu -- host orchestration + C ABI of libmp3b200.so (see include/mp3b200.h).
 *
 * One batch = S independent streams (lamejs Mp3Encoder instances) x their frames.  The pipeline is
 *   K2 psy_analysis -> K3a sequential scans -> K3b masking -> K1 filterbank+MDCT -> K4/K5 quantize+pack
 * launched on one CUDA stream; all intermediates live in HBM workspaces sized per batch.
 * No CPU fallback exists: if CUDA is unavailable every entry point returns MP3B200_ERR_CUDA.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <algorithm>
#include <array>
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
#include "k_resample.cuh"
#include "k_replaygain.cuh"
#include "k_stage.cuh"
#include "k_handle.cuh"
#include "mp3_tag.h"

namespace {

thread_local std::string g_err;
std::mutex g_mu;                          /* guards g_device, g_configs, the per-device flags below */
int g_device = 0;                         /* device of configurations / handles / batch calls created from now on */
std::atomic<long long> g_launches{0};
enum { MP3_MAX_DEVICES = 64 };
bool g_consts_ready[MP3_MAX_DEVICES] = {};   /* __constant__ / __device__ tables are per device */
bool g_fb_attr_done[MP3_MAX_DEVICES][2] = {};   /* k_subband_analysis<false / true> */

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

/* One configuration as mp3_build_config derives it from the caller's (channels, samplerate, kbps, flags), built once on the
 * host.  host.samplerate is the rate lamejs encodes at; with resampling (rs.ratio > 1) the caller's samples arrive at
 * rs.in_rate and k_resample turns them into samples at host.samplerate on the device.  dev[d] is the tables' copy on device
 * d, uploaded by get_config on first use there. */
struct Config {
  Mp3Tables host;
  Mp3Resample rs;
  Mp3TagParams tag;
  bool encodable;                         /* rs.ratio <= RS_MAX_RATIO; the tag entry points describe the others too */
  Mp3Tables* dev[MP3_MAX_DEVICES];
};
std::map<std::tuple<int, int, int, int>, Config*> g_configs;   /* (ch, sr, kbps, flags) -> NULL: lamejs cannot encode it */

/* g_mu held.  The configuration, built on first use, or NULL (g_err set) when lamejs cannot encode it.  MP3B200_RESAMPLE only
 * matters where lamejs resamples, so a flagged configuration that encodes at its input rate is the unflagged one. */
Config* find_config(int ch, int sr, int kbps, int flags) {
  if (flags & ~MP3B200_RESAMPLE) { g_err = "unknown flags"; return nullptr; }
  if (flags && mp3_out_samplerate(ch, sr, kbps) == sr) flags = 0;
  const auto key = std::make_tuple(ch, sr, kbps, flags);
  auto it = g_configs.find(key);
  if (it == g_configs.end()) {
    Config* c = new Config();
    if (mp3_build_config(ch, sr, kbps, flags, &c->host, &c->rs, &c->tag) == 0) c->encodable = c->rs.ratio <= RS_MAX_RATIO;
    else { delete c; c = nullptr; }
    it = g_configs.emplace(key, c).first;
  }
  if (!it->second) g_err = "unsupported configuration";
  return it->second;
}

/* find_config for the entry points that need no device */
const Config* host_config(int ch, int sr, int kbps, int flags) {
  std::lock_guard<std::mutex> lk(g_mu);
  return find_config(ch, sr, kbps, flags);
}

/* the same for the entry points that size an encode: NULL also where k_resample cannot take the ratio */
const Config* encodable_config(int ch, int sr, int kbps, int flags) {
  const Config* c = host_config(ch, sr, kbps, flags);
  return c && c->encodable ? c : nullptr;
}

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
    CK(cudaMemcpyToSymbol(c_rg_yule, RG_YULE, sizeof RG_YULE));
    CK(cudaMemcpyToSymbol(c_rg_butter, RG_BUTTER, sizeof RG_BUTTER));
    int rc = psy_upload_constants();
    if (rc) return rc;
    rc = quant_upload_constants();
    if (rc) return rc;
    g_consts_ready[dev] = true;
  }
  return 0;
}

/* lamejs's input FIFO (gfc.mf_size / mf_samples_to_encode), counted without the samples.  framesize = 576 * mode_gr samples
 * enter per step of lame_encode_buffer_sample (Lame.js:1592-1663); a frame is encoded whenever the FIFO holds
 * framesize + 752 (calcNeeded, Lame.js:1516).  A fresh encoder's FIFO holds 576 - 48 zeros and has ENCDELAY + POSTDELAY =
 * 576 + 1152 samples to encode, whatever the frame size.
 * With an integer resampling ratio r (Config::rs) the FIFO fills with the resampler's outputs: after P input samples
 * lamejs has made outputs(P) = max(0, ceil((P - 16) / r)) of them (output m needs input r m + 16), however P was split
 * into calls.  Sample counts of feed() and flush() are input samples; mf_size and mf_samples_to_encode count outputs. */
struct FifoFlush { long long frames, zeros; int end_padding; };
struct LameFifo {
  static constexpr long long ENC_POST_DELAY = 576 + 1152;     /* ENCDELAY + POSTDELAY */
  long long framesize, mf_size = 576 - 48, mf_samples_to_encode = ENC_POST_DELAY;
  int ratio = 1;
  long long in_fed = 0;                   /* input samples fed so far (resampling only) */
  std::vector<long long>* pieces = nullptr;   /* when set: the sizes of the pieces AnalyzeSamples sees (ReplayGain), the
                                                 n_out of every fill_buffer step: up to framesize outputs each */
  explicit LameFifo(int mode_gr, int r = 1) : framesize(576LL * mode_gr), ratio(r) {}
  long long outputs(long long p) const {
    if (ratio == 1) return p;
    return p > MP3_RS_HALF ? (p - MP3_RS_HALF + ratio - 1) / ratio : 0;
  }
  /* frames completed by feeding n input samples.  Closed form of the step loop: a step adds at most framesize outputs and
   * takes at most one frame, so mf_size stays below framesize + 752 and the frames are the crossings of that level. */
  long long feed(long long n) {
    if (n <= 0) return 0;
    const long long k = outputs(in_fed + n) - outputs(in_fed);
    in_fed += n;
    if (pieces)
      for (long long i = 0; i < k; i += framesize) pieces->push_back(k - i < framesize ? k - i : framesize);
    const long long need = framesize + 752;
    const long long frames = mf_size + k >= need ? (mf_size + k - need) / framesize + 1 : 0;
    if (mf_samples_to_encode < 1) mf_samples_to_encode = ENC_POST_DELAY;
    mf_size += k - frames * framesize;
    mf_samples_to_encode += k - frames * framesize;
    return frames;
  }
  /* lame_encode_flush (Lame.js:1393-1443), in JS numbers: feeds zero bunches of min(1152, the input the next frame needs)
   * until the padded end is out; all zero once flushed (Lame.js:1397-1399).  end_padding is gfp.encoder_padding
   * (Lame.js:1412).  With resampling, samples_to_encode gains 16 * out / in (16 / r: the same correctly rounded quotient),
   * so end_padding and frames_left are fractional: frames_left = 3 + eps encodes a fourth frame, as lamejs does. */
  FifoFlush flush() {
    FifoFlush r = {0, 0, 0};
    if (mf_samples_to_encode < 1) return r;
    double samples_to_encode = (double)(mf_samples_to_encode - 1152);     /* POSTDELAY */
    if (ratio > 1) samples_to_encode += 16. / ratio;
    double end_padding = framesize - fmod(samples_to_encode, (double)framesize);
    if (end_padding < 576) end_padding += framesize;
    r.end_padding = (int)end_padding;                                    /* ToInt32 of a small positive number */
    double frames_left = (samples_to_encode + end_padding) / framesize;
    while (frames_left > 0) {
      double bunch = (double)(framesize + 752 - mf_size);
      bunch *= ratio;                                                    /* * in / out: exact for out | in */
      if (bunch > 1152) bunch = 1152;
      if (bunch < 1) bunch = 1;
      const long long got = feed((long long)bunch);                      /* an integer: (need) * r or a clamp bound */
      r.zeros += (long long)bunch;
      r.frames += got;
      frames_left -= got > 0 ? 1 : 0;     /* sic (Lame.js:1443): one per bunch that completed a frame, even when a 1152-sample
                                             bunch completed two 576-sample frames */
    }
    mf_samples_to_encode = 0;
    return r;
  }
};

/* frames produced by encodeBuffer(n samples) + flush() on a fresh encoder */
long long frames_for(long long n, int mode_gr, int ratio = 1) {
  LameFifo f(mode_gr, ratio);
  const long long fed = f.feed(n);
  return fed + f.flush().frames;
}

/* bytes of frames k0 .. k0 + n - 1 of a stream: frame k is padded when pad_count steps at k */
long long bytes_of_frames(const Mp3Tables& g, long long k0, long long n) {
  return n * g.frame_bytes_nopad + pad_count(k0 + n - 1, g.frac_SpF, g.samplerate) - pad_count(k0 - 1, g.frac_SpF, g.samplerate);
}

/* Grow-only buffer (device memory, or pinned host memory): when a call needs more than it holds, it is reallocated to
 * max(need, 2 x capacity) elements, so a steady run of calls of one shape allocates once.  Contents are not kept. */
template <class T, bool Pinned = false> struct Buf {
  T* p = nullptr;
  size_t cap = 0;
  void release() {
    if (Pinned) cudaFreeHost(p); else cudaFree(p);
    p = nullptr; cap = 0;
  }
  int fit(size_t n) {
    if (n <= cap) return 0;
    if (n < 2 * cap) n = 2 * cap;
    release();
    CK(Pinned ? cudaMallocHost((void**)&p, sizeof(T) * n) : cudaMalloc((void**)&p, sizeof(T) * n));
    cap = n;
    return 0;
  }
};

/* ------------------------------------------------------------------------------------------------ */
/* The status words of a call (Workspace::refusals): [0] a Float32 sample was refused (k_stage_f32), [1] frames over their
 * bit budget (k_q_pack), [2] the call's largest quantizer pass count, [3] a fixed-point loop hit its bound -- the four
 * status words, which a session's call copies to the caller's d_status -- [4] the pass count of the current launch group
 * (k_qstate_loop_cond), [5] the pass index of the ReplayGain repair loop (k_rg_loop_cond), and [6 .. 10) the four further
 * status words of a tagged call: the analysis's passes and reruns (k_rg_report) and two zeros.  A handle call uses [6] and
 * [7] itself (k_handle_commit), so the repair loop of a tagged handle call keeps its pass index, passes and reruns in
 * [10 .. 13). */
enum { MP3_SESSION_WORDS = 13, MP3_STATUS_WORDS = 4, MP3_TAGGED_WORDS_AT = 6, MP3_HANDLE_RG_WORDS_AT = 10 };

/* Per-launch device workspace (U granule rows, F frame rows, S streams of nch channels).                */
struct Workspace {
  Buf<StreamDesc> streams;
  Buf<signed char> bt_final;              /* [U][2] final block type used by MDCT + quantizer */
  Buf<signed char> bt_prev;               /* [U][2] blocktype_old seen by the masking of this granule */
  Buf<float> xr;                          /* [U][nch][576] */
  Buf<float> slab;                        /* [U + S][nch][18][32] subband samples (gfc.sb_sample), psy row numbering */
  Buf<PsyUnit> psy;                       /* [U + S][nch]  (one halo unit per stream in front) */
  Buf<PsyShort> psy_s;                    /* [U + S][nch]  short half of the units on the short list, psy row numbering */
  Buf<int2> short_list;                   /* [U + S][nch]  (stream, unit, channel) tasks of k_psy_short */
  Buf<int> short_count;                   /* [2]: the short list's length, k_psy_short's task counter */
  Buf<ScanIn> scan_in;                    /* [U + S][nch] attack candidates + loudness for the scans */
  Buf<PsyRatioDev> ratio;                 /* [U + S][nch]  masking of unit c (used by granule c+1) */
  Buf<double> ath_psy;                    /* [F] ATH.adjust seen by the psy calls of the frame */
  Buf<double> ath_q;                      /* [F] ATH.adjust after adjust_ATH (quantizer) */
  Buf<QuantFrameState> qstate;            /* [F] speculation bookkeeping */
  Buf<GranuleInfoDev> ginfo;              /* [U][nch] side info of the final quantization */
  Buf<short> l3enc;                       /* [U][nch][576] quantised lines of a gc: after the search, parked best, final */
  Buf<float> xrq;                         /* [U][nch][576] xr as the quantizer sees it (reordered, analog silence zeroed) */
  Buf<float> xrpow;                       /* [U][nch][576] |xr|^(3/4) */
  Buf<unsigned> neg;                      /* [U][nch][18] sign mask of xrq (what the packer needs of it) */
  Buf<GcPrep> prep;                       /* [U][nch] xmin + scalars of the prepared granule-channel */
  Buf<int> dirty;                         /* [3][F] work lists for re-quantization passes */
  Buf<int> counter;                       /* [Q_NCOUNTERS] */
  Buf<ScanChunk> scan;                    /* [F / SCAN_FRAMES + S] */
  Buf<ResampleDesc> rs_desc;              /* resampled batches: [S] */
  Buf<float> rs_y;                        /* resampled batches: the resampler's output rows, the PCM the pipeline reads */
  Buf<StageDesc> st_desc;                 /* Float32 input: [S] */
  Buf<float> st_y;                        /* Float32 input: the staged (scaled) rows */
  Buf<int> refusals;                      /* [MP3_SESSION_WORDS]: the call's status words (reset_words) */
  int fit(int S, int nch, long long U, long long F) {
    const size_t gc = (size_t)U * nch, rows = (size_t)(U + S) * nch, f = (size_t)F + 1;
    const bool failed = streams.fit(S) || bt_final.fit((size_t)U * 2 + 16) || bt_prev.fit((size_t)U * 2 + 16) ||
                        xr.fit(gc * 576) || slab.fit(rows * 576) || psy.fit(rows) || psy_s.fit(rows) || short_list.fit(rows) ||
                        short_count.fit(2) || scan_in.fit(rows) || ratio.fit(rows) ||
                        ath_psy.fit(f) || ath_q.fit(f) || qstate.fit(f) || ginfo.fit(gc) || l3enc.fit(gc * 576) ||
                        xrq.fit(gc * 576) || xrpow.fit(gc * 576) || neg.fit(gc * 18) || prep.fit(gc) || dirty.fit(3 * f) ||
                        counter.fit(Q_NCOUNTERS) || scan.fit((size_t)(F / SCAN_FRAMES + S + 1));
    return failed ? MP3B200_ERR_CUDA : 0;
  }
  /* the workspace's generation as far as the quantizer's buffers go: capacities only grow, so this sum changes exactly when
   * one of them has been reallocated (and a graph holding their addresses is stale) */
  size_t generation() const {
    return streams.cap + qstate.cap + ginfo.cap + l3enc.cap + xrq.cap + xrpow.cap + neg.cap + prep.cap + dirty.cap + counter.cap +
           refusals.cap;
  }
  void release() {
    streams.release(); bt_final.release(); bt_prev.release(); xr.release(); slab.release(); psy.release(); psy_s.release(); short_list.release();
    short_count.release(); scan_in.release();
    ratio.release(); ath_psy.release(); ath_q.release(); qstate.release(); ginfo.release(); l3enc.release(); xrq.release();
    xrpow.release(); neg.release(); prep.release(); dirty.release(); counter.release(); scan.release();
    rs_desc.release(); rs_y.release(); st_desc.release(); st_y.release(); refusals.release();
  }
};

/* Pinned host memory the descriptors of an asynchronous call are uploaded from (a slot of a session's ring): `used` bytes
 * of `cap` are taken. */
struct PinnedArena { uint8_t* p = nullptr; size_t cap = 0, used = 0; };

/* Everything a host thread needs to drive the GPU: its own non-blocking stream (threads encoding through distinct handles
 * or batches never serialise on the legacy default stream), events, workspace and staging buffers.  Bound to one device;
 * re-created when the thread is used with a configuration of another device.
 * An encode session (mp3b200_session) holds one too, bound to the caller's stream instead (session = true): its launches
 * are ordered by that stream alone, with no wait for the legacy default stream, and upload their descriptors from `arena`. */
enum { MP3_MAX_PCM_CHUNKS = 8 };
/* The graphs of a context's device loops: the quantizer's fixed-point loop (QuantLoop), one per launch shape (configuration,
 * streams, frames, longest stream's frames), and the ReplayGain repair loop (rg_finish), one per (configuration, Float32
 * rows, titles, longest title's chunks, chunk rows, loop words) -- what RgParams and the launch grids are made of.  They
 * hold the buffers' addresses, so the quantizer's are all dropped when the workspace's generation changes and the
 * ReplayGain ones when the context's rg_generation does.  A context sees arbitrary shapes: at most MP3_LOOP_GRAPHS graphs
 * are kept, the least recently used going first. */
enum { MP3_LOOP_GRAPHS = 32 };
struct LoopGraphs {
  /* (configuration, 0 for the quantizer or 1 + Float32 for the ReplayGain loop, then the shape), and the loop words */
  using Key = std::tuple<const Config*, int, long long, long long, long long, const int*>;
  struct Graph { cudaGraphExec_t exec = nullptr; unsigned long long used = 0; };
  cudaStream_t capture = nullptr;        /* only captured on */
  size_t generation = 0, rg_generation = 0;
  long long instantiated = 0;            /* graphs instantiated over the context's life (mp3b200_session_graph_instantiations) */
  unsigned long long tick = 0;
  std::map<Key, Graph> graphs;
  /* the cached graph of `key`, or null */
  cudaGraphExec_t find(const Key& key) {
    const auto e = graphs.find(key);
    if (e == graphs.end()) return nullptr;
    e->second.used = ++tick;
    return e->second.exec;
  }
  /* keeps the graph just instantiated for `key` */
  void put(const Key& key, cudaGraphExec_t exec) {
    if (graphs.size() >= MP3_LOOP_GRAPHS) {
      auto lru = graphs.begin();
      for (auto e = graphs.begin(); e != graphs.end(); ++e) if (e->second.used < lru->second.used) lru = e;
      cudaGraphExecDestroy(lru->second.exec);
      graphs.erase(lru);
    }
    graphs[key] = {exec, ++tick};
    instantiated++;
  }
  /* drops the graphs of one kind when the generation of the buffers they hold has changed */
  void renew(bool rg, size_t now) {
    size_t& gen = rg ? rg_generation : generation;
    if (gen == now) return;
    gen = now;
    for (auto e = graphs.begin(); e != graphs.end();) {
      if ((std::get<1>(e->first) != 0) != rg) { ++e; continue; }
      cudaGraphExecDestroy(e->second.exec);
      e = graphs.erase(e);
    }
  }
  void release() {
    for (auto& e : graphs) cudaGraphExecDestroy(e.second.exec);
    graphs.clear();
    if (capture) { cudaStreamDestroy(capture); capture = nullptr; }
  }
};
/* The stream index is a grid y / z coordinate of several kernels (CUDA limit 65535): larger batches run in groups */
enum { MP3_MAX_LAUNCH_STREAMS = 65535 };
struct ThreadCtx {
  int device = -1;
  bool session = false;                   /* st is the caller's stream (not owned) */
  PinnedArena* arena = nullptr;           /* sessions: where the current call's uploads are staged */
  cudaStream_t st = nullptr, up_st = nullptr, aux_st = nullptr;   /* main, PCM upload, quantizer repair chain */
  cudaEvent_t ev[8] = {}, evq[QE_COUNT] = {}, ev_in = nullptr, ev_fork = nullptr, ev_join = nullptr, ready[MP3_MAX_PCM_CHUNKS] = {};
  cudaEvent_t ev_rs[2] = {};              /* around k_resample */
  Workspace ws;
  LoopGraphs loops;
  int evq_pred[QE_COUNT] = {};
  Buf<uint8_t> pcm;                       /* staged PCM of host callers (Int16 or Float32 rows) */
  Buf<uint8_t> out;                       /* encoded bytes of host callers */
  Buf<uint8_t, true> pin;                 /* pinned host staging */
  Buf<long long> crc_ranges;              /* music CRC: [2][R] offsets / lengths */
  Buf<unsigned> crc;                      /* music CRC: [R] results */
  Buf<uint8_t> tags;                      /* tagged whole streams: the template frames and their destinations (k_tag_finish) */
  /* streaming handle calls (queue_handle_call): their device descriptors, the masking row of refused handles, the staged
   * ReplayGain carry and A of analysing handles; for host calls the pinned descriptor arena and the caller's rows */
  Buf<uint8_t> hdesc, rg_stage, hrows;
  Buf<float> halo_scratch;
  Buf<uint8_t, true> hpin;
  cudaStream_t rg_st = nullptr;           /* ReplayGain analysis, beside the encoder */
  cudaEvent_t ev_rg[3] = {};              /* fork, start, end */
  Buf<RgTitle> rg_titles;
  Buf<long long> rg_piece;
  Buf<double> rg_sum, rg_gain;
  Buf<RgState> rg_wstate, rg_cstart;
  Buf<RgEnd> rg_end_a, rg_end_b;
  Buf<RgCarry> rg_carry;
  Buf<int> rg_idx, rg_hist, rg_count;
  /* Workspace::generation for the buffers RgParams names (a graph of the repair loop holds their addresses) */
  size_t rg_generation() const {
    return rg_titles.cap + rg_sum.cap + rg_wstate.cap + rg_cstart.cap + rg_end_a.cap + rg_end_b.cap + rg_count.cap + ws.refusals.cap;
  }
  void release() {
    if (device < 0) return;
    cudaSetDevice(device);
    loops.release();
    ws.release(); pcm.release(); out.release(); pin.release(); crc_ranges.release(); crc.release(); tags.release();
    hdesc.release(); rg_stage.release(); hrows.release(); halo_scratch.release(); hpin.release();
    rg_titles.release(); rg_piece.release(); rg_sum.release(); rg_gain.release(); rg_wstate.release(); rg_cstart.release();
    rg_end_a.release(); rg_end_b.release(); rg_carry.release(); rg_idx.release(); rg_hist.release(); rg_count.release();
    for (auto& e : ev_rg) if (e) { cudaEventDestroy(e); e = nullptr; }
    if (rg_st) { cudaStreamDestroy(rg_st); rg_st = nullptr; }
    for (auto& e : ev) if (e) { cudaEventDestroy(e); e = nullptr; }
    for (auto& e : evq) if (e) { cudaEventDestroy(e); e = nullptr; }
    for (auto& e : ready) if (e) { cudaEventDestroy(e); e = nullptr; }
    for (auto& e : ev_rs) if (e) { cudaEventDestroy(e); e = nullptr; }
    if (ev_in) { cudaEventDestroy(ev_in); ev_in = nullptr; }
    if (ev_fork) { cudaEventDestroy(ev_fork); ev_fork = nullptr; }
    if (ev_join) { cudaEventDestroy(ev_join); ev_join = nullptr; }
    if (aux_st) { cudaStreamDestroy(aux_st); aux_st = nullptr; }
    if (st && !session) cudaStreamDestroy(st);
    st = nullptr;
    if (up_st) { cudaStreamDestroy(up_st); up_st = nullptr; }
    device = -1;
  }
  ~ThreadCtx() { release(); }
  int use(int dev) {
    CK(cudaSetDevice(dev));
    if (device == dev) return 0;
    release();
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    return create(dev);
  }
  /* a session's context on the current device `dev`, launching on the caller's stream `s` */
  int bind(int dev, cudaStream_t s) {
    release();
    session = true;
    st = s;
    return create(dev);
  }
  int create(int dev) {
    CK(cudaStreamCreateWithFlags(&up_st, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&rg_st, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&loops.capture, cudaStreamNonBlocking));
    for (auto& e : ev_rg) CK(cudaEventCreate(&e));
    for (auto& e : ev) CK(cudaEventCreate(&e));
    for (auto& e : evq) CK(cudaEventCreate(&e));
    for (auto& e : ready) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    for (auto& e : ev_rs) CK(cudaEventCreate(&e));
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
};
thread_local ThreadCtx t_ctx;

int config_on(int dev, int ch, int sr, int kbps, int flags, Config** out);

/* The configuration for a launch on the current device (g_device): uploads its tables there on first use and binds the
 * calling thread's context (t_ctx) to that device, so cfg->dev[t_ctx.device] holds them. */
int get_config(int ch, int sr, int kbps, int flags, Config** out) {
  int dev = 0;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    dev = g_device;
  }
  const int rc = config_on(dev, ch, sr, kbps, flags, out);
  return rc ? rc : t_ctx.use(dev);
}

/* get_config on device `dev`, binding no context (an encode session has its own) */
int config_on(int dev, int ch, int sr, int kbps, int flags, Config** out) {
  if (flags & ~MP3B200_RESAMPLE) { g_err = "unknown flags"; return MP3B200_ERR_CONFIG; }
  {
    std::lock_guard<std::mutex> lk(g_mu);
    int rc = ensure_device(dev);
    if (rc) return rc;
    Config* c = find_config(ch, sr, kbps, flags);
    if (!c || !c->encodable) { g_err = "unsupported configuration"; return MP3B200_ERR_CONFIG; }
    if (!c->dev[dev]) {
      if (c->rs.ratio > 1)     /* the ratio's filter row (the same taps for every configuration of that ratio) */
        CK(cudaMemcpyToSymbol(c_rs_h, c->rs.h, sizeof(float) * MP3_RS_TAPS, sizeof(float) * MP3_RS_TAPS * c->rs.ratio));
      Mp3Tables* d = nullptr;
      CK(cudaMalloc(&d, sizeof(Mp3Tables)));
      CK(cudaMemcpy(d, &c->host, sizeof(Mp3Tables), cudaMemcpyHostToDevice));
      c->dev[dev] = d;
    }
    *out = c;
  }
  return 0;
}

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

struct Timings { float psy = 0, scan = 0, mask = 0, fb = 0, q1 = 0, qn = 0, total = 0;
                 float q_prepare = 0, q_search = 0, q_outer = 0, q_finish = 0, q_pack = 0, q_mid = 0; };

/* chunks > 1: the caller uploads each stream's PCM in that many time slices on another stream and records ready[j] after
 * slice j; the psy analysis of slice j starts as soon as it has landed. */
struct PcmArrival { int chunks = 1; cudaEvent_t* ready = nullptr; };

/* The error of a call whose status words read refused / over_budget / fault (a device loop hit its bound), with g_err
 * set; 0 when the output stands. */
int refusal_error(int refused, int over_budget, int fault) {
  if (refused) { g_err = "non-finite input sample (or one beyond 2^40 once scaled)"; return MP3B200_ERR_CONFIG; }
  if (over_budget) { g_err = "frame over its bit budget (input too loud to encode)"; return MP3B200_ERR_CONFIG; }
  if (fault == RG_FAULT) { g_err = "ReplayGain repair did not converge"; return MP3B200_ERR_CUDA; }
  if (fault) { g_err = "quantizer stage failed: the fixed-point loop did not converge"; return MP3B200_ERR_CUDA; }
  return 0;
}

/* Once the call's work has joined c.st, one read-back of the status words: MP3B200_ERR_CONFIG when k_stage_f32 refused a
 * Float32 sample, or when a frame's bits did not fit its slot (k_q_pack left it unpacked), where lamejs throws out of the
 * call (BitStream.js:856-885); MP3B200_ERR_CUDA when a device loop hit its bound.  The call's output must not be used. */
int check_refusals(ThreadCtx& c) {
  int r[MP3_STATUS_WORDS] = {};
  CK(cudaMemcpyAsync(r, c.ws.refusals.p, sizeof r, cudaMemcpyDeviceToHost, c.st));
  CK(cudaStreamSynchronize(c.st));
  return refusal_error(r[0], r[1], r[3]);
}

/* Options of launch_streams */
struct LaunchOpts {
  const int32_t* force_bt = nullptr;     /* debug: host [units][nch] block types overriding the psy model's decision */
  bool stop_after_mdct = false;          /* debug: no quantizer, no bytes */
  bool all_short = false;                /* debug: the short-block psy half of every unit, as if each were read (stage taps) */
  const PcmArrival* arrival = nullptr;   /* PCM still landing on the upload stream */
  float* timings_ms = nullptr;           /* the 16 timing slots of include/mp3b200.h */
  bool sync = true;                      /* false: return with the work queued on the context's stream (no timings) */
  struct RgJob* rg = nullptr;            /* ReplayGain of every stream, beside the encoder (one launch group only) */
  bool f32_in = false;                   /* the descriptors point at the caller's Float32 rows (k_stage_f32 stages them); with
                                            sync, a non-finite sample makes the launch return MP3B200_ERR_CONFIG */
  const struct HandleCarry* carry = nullptr;   /* streaming handles: their carried state is on the device (k_handle_carry_in;
                                                  one launch group only) */
  int* rg_loop = nullptr;                /* the three words of the ReplayGain loop (rg_finish) of a handle call; NULL: ws.refusals + 5 */
  bool analyse_only = false;             /* stop after staging, resampling and the ReplayGain analysis of o.rg: no encoder
                                            kernels, no bytes, no workspace beyond the staged rows */
};

/* LaunchOpts::carry: recs[z] is the record of stream z (device array); halo_scratch takes the masking of refused handles */
struct HandleCarry { HandleRecord* const* recs; float* halo_scratch; };

/* Queues the copy of n bytes of host descriptors to dst on `on` (NULL: c.st).  A session's call stages them in its pinned
 * slot first, so the copy never waits for the device; a thread's context copies from `src` (pageable) as it is. */
int upload(ThreadCtx& c, void* dst, const void* src, size_t n, cudaStream_t on = nullptr) {
  if (c.arena) {
    PinnedArena& a = *c.arena;
    const size_t at = (a.used + 255) & ~(size_t)255;
    if (at + n > a.cap) { g_err = "descriptor staging overflow"; return MP3B200_ERR_CUDA; }
    memcpy(a.p + at, src, n);
    a.used = at + n;
    src = a.p + at;
  }
  CK(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, on ? on : c.st));
  return 0;
}

/* Resets the status words (ws.refusals) for a call of `nstreams` streams on c.st: [0 .. 2) zero, then the start words --
 * [2] is the pass count of launch groups that speculate nothing -- and zeros */
int reset_words(ThreadCtx& c, int nstreams) {
  int rc = c.ws.refusals.fit(MP3_SESSION_WORDS);
  if (rc) return rc;
  CK(cudaMemsetAsync(c.ws.refusals.p, 0, 2 * sizeof(int), c.st));
  const int start[MP3_SESSION_WORDS - 2] = {nstreams > 0 ? 2 : 0};
  return upload(c, c.ws.refusals.p + 2, start, sizeof start);
}

/* Makes c.st wait for the work the caller queued on the legacy default stream (torch and plain CUDA callers produce their
 * device buffers there).  A session's stream is the only ordering of its calls: nothing to do. */
int wait_legacy(ThreadCtx& c) {
  if (c.session) return 0;
  CK(cudaEventRecord(c.ev_in, cudaStreamLegacy));
  CK(cudaStreamWaitEvent(c.st, c.ev_in, 0));
  return 0;
}

/* The rows the descriptors of a launch point at: the caller's Int16 samples, {false, host.scale_applied}, or Float32 rows
 * already scaled by k_stage_f32 or k_resample, SCALED_F32.  The kernels that read them are instantiated for `f32`. */
struct Rows { bool f32; int scale_applied; };
constexpr Rows SCALED_F32 = {true, 0};

/* Debug psy-row capture (mp3b200_debug_psy_capture).  While it is on, every pipeline launch poisons the front-end and
 * quantizer rows it uses before k_psy_analysis, so that a row the launch forgets to write cannot pass for one written by an
 * earlier launch, and records them after k_attack_prepass (PsyUnit), after k_psy_short (the short list and its PsyShort
 * rows), after k_mdct (block types, ATH adjustments, masking and xr) and after the quantizer's fixed point (its frame states
 * and hand-over rows).  The launch synchronises its stream at those points; with capture off it does nothing at all. */
std::atomic<int> g_psy_capture{0};
std::mutex g_psy_mu;                      /* guards g_psy_rec, g_psy_launch */
std::vector<unsigned char> g_psy_rec;     /* records: int32[8] header + payload (include/mp3b200.h) */
int g_psy_launch = 0;

void psy_rec_append(const int32_t (&h)[8], const void* a, size_t na, const void* b = nullptr, size_t nb = 0) {
  std::lock_guard<std::mutex> lk(g_psy_mu);
  const unsigned char* hp = reinterpret_cast<const unsigned char*>(h);
  g_psy_rec.insert(g_psy_rec.end(), hp, hp + sizeof h);
  if (na) g_psy_rec.insert(g_psy_rec.end(), static_cast<const unsigned char*>(a), static_cast<const unsigned char*>(a) + na);
  if (nb) g_psy_rec.insert(g_psy_rec.end(), static_cast<const unsigned char*>(b), static_cast<const unsigned char*>(b) + nb);
}

/* The quantizer's rows of a launch (gcs granule-channels, nframes frame states), each value chosen so that a kernel reading
 * an unwritten row runs on and changes what the record or the bytes show, without indexing out of bounds or looping forever:
 *   xrq, xrpow  1.0f: finite and positive, so every adj43 index and every bin search stays in range; real rows are zeroed
 *               above the analog silence and are rarely exactly 1.0 anywhere else
 *   neg         0xAAAAAAAA: every other line negative, which flips the sign of half the packed lines
 *   l3enc       1 on every line: counted and packed like a real quantised row, never all zero as a silent granule's is
 *   prep        xmin 1.0f, have 1, mnz 575, block type NORM, xrpow_max 1.0: a granule with energy and valid long-block bands
 *   ginfo       gi_init_w's long-block template over that prep, but global_gain 1 where the template has 210; every other
 *               field 0, so part2_3_length 0 and table 0 everywhere (valid for the packer)
 *   qstate      stream 0, rel_frame 0 (k_qstate_verify skips a first frame instead of reading row -1), every carried state
 *               (180, 4) as at a stream's start, used0 0, valid 0, redo 0 */
int q_poison(ThreadCtx& c, size_t gcs, long long nframes) {
  if (!gcs) return 0;
  std::vector<float> one(gcs * 576, 1.0f);
  std::vector<unsigned> neg(gcs * 18, 0xAAAAAAAAu);
  std::vector<short> ix(gcs * 576, 1);
  GcPrep pr;
  memset(&pr, 0, sizeof pr);
  for (float& v : pr.xmin) v = 1.0f;
  pr.have = 1; pr.mnz = 575; pr.block_type = BT_NORM; pr.xrpow_max = 1.0;
  GranuleInfoDev gi;
  memset(&gi, 0, sizeof gi);
  gi.global_gain = 1; gi.block_type = BT_NORM;
  gi.sfb_lmax = 21; gi.sfb_smin = 12; gi.psy_lmax = 21; gi.psymax = 21; gi.sfbmax = 21; gi.sfbdivide = 11;
  gi.max_nonzero_coeff = 575; gi.xrpow_max = 1.0;
  QuantFrameState qs;
  memset(&qs, 0, sizeof qs);
  for (int ch = 0; ch < 2; ch++) {
    qs.in_old[ch] = qs.out_old[ch] = qs.bs_gain0[ch] = 180;
    qs.in_step[ch] = qs.out_step[ch] = qs.bs_step0[ch] = 4;
  }
  std::vector<GcPrep> prs(gcs, pr);
  std::vector<GranuleInfoDev> gis(gcs, gi);
  std::vector<QuantFrameState> qss((size_t)nframes, qs);
  CK(cudaMemcpyAsync(c.ws.xrq.p, one.data(), one.size() * sizeof(float), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.xrpow.p, one.data(), one.size() * sizeof(float), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.neg.p, neg.data(), neg.size() * sizeof(unsigned), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.l3enc.p, ix.data(), ix.size() * sizeof(short), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.prep.p, prs.data(), gcs * sizeof(GcPrep), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.ginfo.p, gis.data(), gcs * sizeof(GranuleInfoDev), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.qstate.p, qss.data(), qss.size() * sizeof(QuantFrameState), cudaMemcpyHostToDevice, c.st));
  CK(cudaStreamSynchronize(c.st));
  return 0;
}

/* Fills the launch's rows: front-end floats with a quiet NaN, bytes with values that stay valid table indices (mask_idx 8,
 * attack 0, block types BT_START), so that reading an unwritten row changes results without ever indexing out of bounds.
 * bt_prev never holds BT_START when written (the scan stores NORM, STOP or SHORT there).
 * The quantizer's rows get finite values its kernels can run on (q_poison): a NaN or negative xrpow would index adj43 out of
 * range, and a zero search step would never end a bin search. */
int psy_poison(ThreadCtx& c, int G, long long total_frames, int S, int nch, int* launch) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CK(cudaStreamIsCapturing(c.st, &cs));
  if (cs != cudaStreamCaptureStatusNone) { g_err = "psy-row capture inside CUDA stream capture"; return MP3B200_ERR_CUDA; }
  {
    std::lock_guard<std::mutex> lk(g_psy_mu);
    *launch = g_psy_launch++;
  }
  const uint32_t qbits = 0x7fc00000u;
  float qnan;
  memcpy(&qnan, &qbits, sizeof qnan);
  PsyUnit pu;
  for (float& v : pu.eb_l) v = qnan;
  for (float& v : pu.peaks) v = qnan;
  pu.loudness = qnan;
  memset(pu.mask_idx, 8, sizeof pu.mask_idx);
  memset(pu.attack, 0, sizeof pu.attack);
  pu.pad_ = 0;
  PsyShort ps;
  for (int s = 0; s < 3; s++)
    for (int b = 0; b < MP3_CBANDS; b++) { ps.ecb_s[s][b] = (double)qnan; ps.eb_s[s][b] = qnan; }
  const size_t units = (size_t)G * total_frames, rows = (units + S) * nch;
  std::vector<PsyUnit> u(rows, pu);
  std::vector<PsyShort> sh(rows, ps);
  std::vector<float> f(rows * 576, qnan);             /* slab rows; the ratio and xr rows take a prefix */
  const uint64_t dbits = 0x7ff8000000000000ull;
  double dnan;
  memcpy(&dnan, &dbits, sizeof dnan);
  std::vector<double> d((size_t)total_frames, dnan);
  CK(cudaMemcpyAsync(c.ws.psy.p, u.data(), rows * sizeof(PsyUnit), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.psy_s.p, sh.data(), rows * sizeof(PsyShort), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.ratio.p, f.data(), rows * sizeof(PsyRatioDev), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.slab.p, f.data(), rows * 576 * sizeof(float), cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyAsync(c.ws.xr.p, f.data(), units * nch * 576 * sizeof(float), cudaMemcpyHostToDevice, c.st));
  if (total_frames) {
    CK(cudaMemcpyAsync(c.ws.ath_psy.p, d.data(), d.size() * sizeof(double), cudaMemcpyHostToDevice, c.st));
    CK(cudaMemcpyAsync(c.ws.ath_q.p, d.data(), d.size() * sizeof(double), cudaMemcpyHostToDevice, c.st));
  }
  CK(cudaMemsetAsync(c.ws.bt_final.p, BT_START, units * 2, c.st));
  CK(cudaMemsetAsync(c.ws.bt_prev.p, BT_START, units * 2, c.st));
  CK(cudaStreamSynchronize(c.st));
  return q_poison(c, units * nch, total_frames);
}

/* After k_attack_prepass: each stream's rows u = -1 .. G nframes - 1 */
int psy_record_units(ThreadCtx& c, const StreamDesc* sds, int S, int nch, int G, int launch) {
  CK(cudaStreamSynchronize(c.st));
  for (int z = 0; z < S; z++) {
    const StreamDesc& sd = sds[z];
    const size_t n = ((size_t)G * sd.nframes + 1) * nch;
    std::vector<PsyUnit> rows(n);
    CK(cudaMemcpyAsync(rows.data(), c.ws.psy.p + ((size_t)sd.unit_base + z) * nch, n * sizeof(PsyUnit), cudaMemcpyDeviceToHost, c.st));
    CK(cudaStreamSynchronize(c.st));
    const int32_t h[8] = {1, launch, z, sd.frame0, sd.nframes, nch, G, (int32_t)sizeof(PsyUnit)};
    psy_rec_append(h, rows.data(), n * sizeof(PsyUnit));
  }
  return 0;
}

/* After k_psy_short: the short list in list order and the PsyShort row of each entry */
int psy_record_short(ThreadCtx& c, const StreamDesc* sds, int nch, int G, int launch, int k2_launches) {
  CK(cudaStreamSynchronize(c.st));
  int count = 0;
  CK(cudaMemcpyAsync(&count, c.ws.short_count.p, sizeof count, cudaMemcpyDeviceToHost, c.st));
  CK(cudaStreamSynchronize(c.st));
  std::vector<int2> list((size_t)count);
  std::vector<PsyShort> rows((size_t)count);
  if (count) CK(cudaMemcpyAsync(list.data(), c.ws.short_list.p, count * sizeof(int2), cudaMemcpyDeviceToHost, c.st));
  CK(cudaStreamSynchronize(c.st));
  for (int i = 0; i < count; i++) {
    const int z = list[i].x, u = (list[i].y >> 1) - 1, ch = list[i].y & 1;
    const size_t row = ((size_t)sds[z].unit_base + z + u + 1) * nch + ch;
    CK(cudaMemcpyAsync(&rows[i], c.ws.psy_s.p + row, sizeof(PsyShort), cudaMemcpyDeviceToHost, c.st));
  }
  CK(cudaStreamSynchronize(c.st));
  const int32_t h[8] = {2, launch, count, nch, G, k2_launches, 0, (int32_t)sizeof(PsyShort)};
  psy_rec_append(h, list.data(), count * sizeof(int2), rows.data(), count * sizeof(PsyShort));
  return 0;
}

/* After k_mdct: per stream, ath_psy and ath_q of its frames, the ratio rows u = -1 .. G nframes - 1, the xr rows, bt_final
 * and bt_prev of its units (two per unit, as the workspace holds them), zero bytes up to a multiple of 8 */
int psy_record_front(ThreadCtx& c, const StreamDesc* sds, int S, int nch, int G, int launch) {
  CK(cudaStreamSynchronize(c.st));
  for (int z = 0; z < S; z++) {
    const StreamDesc& sd = sds[z];
    const size_t F = (size_t)sd.nframes, n = (size_t)G * sd.nframes;
    const size_t b_ath = 2 * F * sizeof(double), b_ratio = (n + 1) * nch * sizeof(PsyRatioDev);
    const size_t b_xr = n * nch * 576 * sizeof(float), b_bt = 2 * n * 2;
    std::vector<unsigned char> p(b_ath + b_ratio + b_xr + ((b_bt + 7) & ~(size_t)7), 0);
    unsigned char* q = p.data();
    if (F) {
      CK(cudaMemcpyAsync(q, c.ws.ath_psy.p + sd.frame_base, F * sizeof(double), cudaMemcpyDeviceToHost, c.st));
      CK(cudaMemcpyAsync(q + F * sizeof(double), c.ws.ath_q.p + sd.frame_base, F * sizeof(double), cudaMemcpyDeviceToHost, c.st));
    }
    q += b_ath;
    CK(cudaMemcpyAsync(q, c.ws.ratio.p + ((size_t)sd.unit_base + z) * nch, b_ratio, cudaMemcpyDeviceToHost, c.st));
    q += b_ratio;
    if (n) {
      CK(cudaMemcpyAsync(q, c.ws.xr.p + (size_t)sd.unit_base * nch * 576, b_xr, cudaMemcpyDeviceToHost, c.st));
      CK(cudaMemcpyAsync(q + b_xr, c.ws.bt_final.p + (size_t)sd.unit_base * 2, n * 2, cudaMemcpyDeviceToHost, c.st));
      CK(cudaMemcpyAsync(q + b_xr + n * 2, c.ws.bt_prev.p + (size_t)sd.unit_base * 2, n * 2, cudaMemcpyDeviceToHost, c.st));
    }
    CK(cudaStreamSynchronize(c.st));
    const int32_t h[8] = {3, launch, z, sd.frame0, sd.nframes, nch, G, (int32_t)sizeof(PsyRatioDev)};
    psy_rec_append(h, p.data(), p.size());
  }
  return 0;
}

/* After the quantizer's fixed point and k_qstate_commit: per stream, the row sizes int32[4] {QuantFrameState, GcPrep,
 * GranuleInfoDev, 0}, its frames' QuantFrameState rows, then for its n nch granule-channels (n = G nframes) the GcPrep and
 * GranuleInfoDev rows, l3enc short[576], xrq and xrpow float[576] and neg unsigned[18] of each (every size a multiple of 8).
 * k_q_prepare's rows are never rewritten, so this one record sees what every later kernel read. */
int q_record(ThreadCtx& c, const StreamDesc* sds, int S, int nch, int G, int launch) {
  CK(cudaStreamSynchronize(c.st));
  const int32_t sizes[4] = {(int32_t)sizeof(QuantFrameState), (int32_t)sizeof(GcPrep), (int32_t)sizeof(GranuleInfoDev), 0};
  for (int z = 0; z < S; z++) {
    const StreamDesc& sd = sds[z];
    const size_t F = (size_t)sd.nframes, g = (size_t)G * sd.nframes * nch, g0 = (size_t)sd.unit_base * nch;
    const size_t b_qs = F * sizeof(QuantFrameState), b_prep = g * sizeof(GcPrep), b_gi = g * sizeof(GranuleInfoDev);
    const size_t b_ix = g * 576 * sizeof(short), b_row = g * 576 * sizeof(float), b_neg = g * 18 * sizeof(unsigned);
    std::vector<unsigned char> p(sizeof sizes + b_qs + b_prep + b_gi + b_ix + 2 * b_row + b_neg);
    unsigned char* q = p.data();
    memcpy(q, sizes, sizeof sizes);
    q += sizeof sizes;
    if (F) {
      CK(cudaMemcpyAsync(q, c.ws.qstate.p + sd.frame_base, b_qs, cudaMemcpyDeviceToHost, c.st));
      q += b_qs;
      CK(cudaMemcpyAsync(q, c.ws.prep.p + g0, b_prep, cudaMemcpyDeviceToHost, c.st));
      q += b_prep;
      CK(cudaMemcpyAsync(q, c.ws.ginfo.p + g0, b_gi, cudaMemcpyDeviceToHost, c.st));
      q += b_gi;
      CK(cudaMemcpyAsync(q, c.ws.l3enc.p + g0 * 576, b_ix, cudaMemcpyDeviceToHost, c.st));
      q += b_ix;
      CK(cudaMemcpyAsync(q, c.ws.xrq.p + g0 * 576, b_row, cudaMemcpyDeviceToHost, c.st));
      q += b_row;
      CK(cudaMemcpyAsync(q, c.ws.xrpow.p + g0 * 576, b_row, cudaMemcpyDeviceToHost, c.st));
      q += b_row;
      CK(cudaMemcpyAsync(q, c.ws.neg.p + g0 * 18, b_neg, cudaMemcpyDeviceToHost, c.st));
    }
    CK(cudaStreamSynchronize(c.st));
    const int32_t h[8] = {4, launch, z, sd.frame0, sd.nframes, nch, G, 0};
    psy_rec_append(h, p.data(), p.size());
  }
  return 0;
}

/* One pipeline launch for the streams sds[0 .. S) (at most MP3_MAX_LAUNCH_STREAMS, unit / frame bases set, the workspace
 * large enough).  All launches go to the context's stream (c.st: the calling thread's, t_ctx.st, or a session's), which
 * first waits for whatever the caller queued on the legacy default stream (wait_legacy); with o.sync the call returns after
 * the stream has drained, so the results are visible to any stream afterwards. */
int run_pipeline(ThreadCtx& c, Config* cfg, StreamDesc* h_streams, int S, const LaunchOpts& o,
                 const PcmArrival* arrival, Rows rows, Timings* tm) {
  cudaStream_t st = c.st;
  cudaEvent_t* ev = c.ev;
  Workspace& ws = c.ws;

  const Mp3Tables* const tab = cfg->dev[c.device];
  const int nch = cfg->host.nch;
  const bool f32_pcm = rows.f32;
  int max_frames = 0;
  long long total_frames = 0;          /* rows actually used this launch (the workspace may be larger) */
  int scan_rows = 0;
  int streams_with_frames = 0;
  for (int i = 0; i < S; i++) {
    StreamDesc& s = h_streams[i];
    max_frames = s.nframes > max_frames ? s.nframes : max_frames;
    total_frames += s.nframes;
    streams_with_frames += s.nframes > 0 ? 1 : 0;
    s.scan_base = scan_rows;
    scan_rows += (s.nframes + SCAN_FRAMES - 1) / SCAN_FRAMES;
  }
  int rc = wait_legacy(c);
  if (rc || (rc = upload(c, ws.streams.p, h_streams, sizeof(StreamDesc) * S))) return rc;
  if (o.carry) {
    k_handle_carry_in<<<(S + 127) / 128, 128, 0, st>>>(ws.streams.p, S, o.carry->recs, o.carry->halo_scratch);
    g_launches++;
    DBG("k_handle_carry_in");
  }
  int psy_launch = -1, k2_launches = 0;
  if (g_psy_capture.load(std::memory_order_relaxed) &&
      (rc = psy_poison(c, cfg->host.mode_gr, total_frames, S, nch, &psy_launch))) return rc;
  CK(cudaEventRecord(ev[0], st));

  /* K2: psy analysis, one block per (PSY_UNITS consecutive granules incl. 1 halo, channel, stream) */
  {
    const int nchunks = arrival ? arrival->chunks : 1;
    /* units (relative index, -1 = halo) each upload slice completes, over all streams: the kernel's own rule
     * (k_psy_analysis) evaluated on the host, so that a slice's launch covers only its range of units */
    int u_lo[MP3_MAX_PCM_CHUNKS], u_hi[MP3_MAX_PCM_CHUNKS];
    const int G = cfg->host.mode_gr;     /* granules ("units") per frame */
    for (int j = 0; j < nchunks; j++) { u_lo[j] = G * max_frames; u_hi[j] = -1; }
    if (nchunks > 1) {
      for (int s = 0; s < S; s++) {
        const StreamDesc& sd = h_streams[s];
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
      dim3 gridj((u_hi[j] - u_lo[j] + PSY_UNITS - 1) / PSY_UNITS, nch, S);
      if (f32_pcm) k_psy_analysis<true><<<gridj, PSY_A_THREADS, 0, st>>>(tab, ws.streams.p, ws.psy.p, j, nchunks, u_lo[j]);
      else k_psy_analysis<false><<<gridj, PSY_A_THREADS, 0, st>>>(tab, ws.streams.p, ws.psy.p, j, nchunks, u_lo[j]);
      g_launches++;
      k2_launches++;
      DBG("k_psy_analysis");
    }
  }
  CK(cudaEventRecord(ev[1], st));
  /* K3a: attack pre-pass (parallel) + sequential per-stream scans */
  {
    dim3 grid((cfg->host.mode_gr * max_frames + 127) / 128, 1, S);
    k_attack_prepass<<<grid, 128, 0, st>>>(tab, ws.streams.p, ws.psy.p, ws.scan_in.p);
    DBG("k_attack_prepass");
    if (psy_launch >= 0 && (rc = psy_record_units(c, h_streams, S, nch, cfg->host.mode_gr, psy_launch))) return rc;
    k_stream_scan<<<S, SCAN_THREADS, 0, st>>>(tab, ws.streams.p, S, ws.scan_in.p, ws.bt_final.p, ws.bt_prev.p, ws.ath_psy.p, ws.ath_q.p, ws.scan.p);
    g_launches += 2;
    DBG("k_stream_scan");
    /* K1a: subband analysis, programmatic dependent of the scan (reads nothing the scan writes; see k_stream_scan) */
    {
      const int G = cfg->host.mode_gr;
      const size_t smem = sizeof(double) * FB_PCM_WORDS + sizeof(float) * (FB_SLABS * 18 * FB_SLAB_STRIDE);
      void (*const k_fb)(const Mp3Tables*, const StreamDesc*, float*) = f32_pcm ? k_subband_analysis<true> : k_subband_analysis<false>;
      {
        std::lock_guard<std::mutex> lk(g_mu);   /* the attribute is per device */
        if (!g_fb_attr_done[c.device][f32_pcm]) { CK(cudaFuncSetAttribute(k_fb, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); g_fb_attr_done[c.device][f32_pcm] = true; }
      }
      cudaLaunchConfig_t lc = {};
      lc.gridDim = dim3((G * max_frames + 1 + FB_SLABS - 1) / FB_SLABS, nch, S);
      lc.blockDim = dim3(FB_THREADS); lc.dynamicSmemBytes = smem; lc.stream = st;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      at[0].val.programmaticStreamSerializationAllowed = 1;
      lc.attrs = at; lc.numAttrs = 1;
      CK(cudaLaunchKernelEx(&lc, k_fb, tab, (const StreamDesc*)ws.streams.p, ws.slab.p));
      g_launches++;
      DBG("k_subband_analysis");
    }
  }
  CK(cudaEventRecord(ev[2], st));
  if (o.force_bt) {   /* debug: override block decision for the filterbank */
    const long long units = (long long)cfg->host.mode_gr * total_frames;
    std::vector<signed char> bt((size_t)units * 2, 0);
    for (long long u = 0; u < units; u++)
      for (int c = 0; c < nch; c++) bt[u * 2 + c] = (signed char)o.force_bt[u * nch + c];
    CK(cudaMemcpyAsync(ws.bt_final.p, bt.data(), bt.size(), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
  }
  /* K2b: the short-block psy half of the units whose short thresholds are read, listed from the final block types (after
   * force_bt); persistent blocks that leave at once when the list is empty */
  {
    CK(cudaMemsetAsync(ws.short_count.p, 0, 2 * sizeof(int), st));
    dim3 grid((cfg->host.mode_gr * max_frames + 1 + 127) / 128, S);
    k_psy_short_list<<<grid, 128, 0, st>>>(tab, ws.streams.p, ws.bt_final.p, o.all_short ? 1 : 0, ws.short_list.p, ws.short_count.p);
    DBG("k_psy_short_list");
    int sms = 132;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c.device));
    const long long tasks = ((long long)cfg->host.mode_gr * total_frames + S) * nch;
    const int blocks = (int)std::min<long long>(std::max<long long>(tasks, 1), (long long)sms * PSY_SHORT_BLOCKS);
    if (f32_pcm) k_psy_short<true><<<blocks, PSY_THREADS, 0, st>>>(tab, ws.streams.p, ws.psy_s.p, ws.short_list.p, ws.short_count.p);
    else k_psy_short<false><<<blocks, PSY_THREADS, 0, st>>>(tab, ws.streams.p, ws.psy_s.p, ws.short_list.p, ws.short_count.p);
    g_launches += 2;
    DBG("k_psy_short");
    if (psy_launch >= 0 && (rc = psy_record_short(c, h_streams, nch, cfg->host.mode_gr, psy_launch, k2_launches))) return rc;
  }
  /* K3b: masking thresholds */
  {
    dim3 grid(cfg->host.mode_gr * max_frames + 1, 1, S);
    k_psy_masking<<<grid, MASK_THREADS, 0, st>>>(tab, ws.streams.p, ws.psy.p, ws.psy_s.p, ws.bt_prev.p, ws.bt_final.p,
                                                 o.all_short ? 1 : 0, ws.ath_psy.p, ws.ratio.p);
    g_launches++;
    DBG("k_psy_masking");
  }
  CK(cudaEventRecord(ev[3], st));
  /* K1b: MDCT from the slabs and the block types.  (As a programmatic dependent of the masking kernel, running beside it:
   * it saves only a few microseconds for the pair -- not worth losing the per-kernel times.) */
  {
    dim3 grid((cfg->host.mode_gr * max_frames + FB_G - 1) / FB_G, nch, S);
    k_mdct<<<grid, FB_G * 32, 0, st>>>(tab, ws.streams.p, ws.slab.p, ws.bt_final.p, ws.xr.p);
    g_launches++;
    DBG("k_mdct");
    if (psy_launch >= 0 && (rc = psy_record_front(c, h_streams, S, nch, cfg->host.mode_gr, psy_launch))) return rc;
  }
  CK(cudaEventRecord(ev[4], st));
  if (!o.stop_after_mdct) {
    QuantBuffers qb;
    qb.xr = ws.xr.p; qb.ratio = ws.ratio.p; qb.bt = ws.bt_final.p; qb.ath_q = ws.ath_q.p; qb.qs = ws.qstate.p; qb.ginfo = ws.ginfo.p;
    qb.l3enc = ws.l3enc.p; qb.xrq = ws.xrq.p; qb.xrpow = ws.xrpow.p; qb.neg = ws.neg.p; qb.prep = ws.prep.p; qb.list = ws.dirty.p; qb.counter = ws.counter.p;
    qb.over_budget = ws.refusals.p + 1;
    LoopGraphs& lg = c.loops;              /* the graph for this shape, captured by quant_run if there is none */
    lg.renew(false, ws.generation());
    const LoopGraphs::Key key = {cfg, 0, S, total_frames, max_frames, nullptr};
    QuantLoop loop;
    loop.capture = lg.capture; loop.st = ws.refusals.p + 2; loop.exec = lg.find(key);
    const bool cached = loop.exec != nullptr;
    rc = quant_run(tab, cfg->host, ws.streams.p, S, streams_with_frames, max_frames, total_frames, qb, st, c.aux_st, c.ev_fork, c.ev_join,
                   ev[5], c.evq, c.evq_pred, &g_launches, loop);
    if (!cached && loop.exec) lg.put(key, loop.exec);
    if (rc) { g_err = "quantizer stage failed: " + std::string(cudaGetErrorString(cudaGetLastError())); return rc; }
    if (psy_launch >= 0 && (rc = q_record(c, h_streams, S, nch, cfg->host.mode_gr, psy_launch))) return rc;
  } else {
    CK(cudaEventRecord(ev[5], st));
  }
  CK(cudaEventRecord(ev[6], st));
  if (!o.sync) return 0;                   /* the caller queues its copies behind the kernels and synchronises once */
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
    if (!o.stop_after_mdct) {
      auto span = [&](int slot) { float v = 0; const int p = c.evq_pred[slot]; if (p >= 0) cudaEventElapsedTime(&v, c.evq[p], c.evq[slot]); return v; };
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

/* first sample (at the encoding rate) that frame `frame` and later frames read: the filterbank slab of the granule before
 * frame k starts at framesize * k - 1104 */
long long hist_base_at(int mode_gr, long long frame) {
  const long long b = 576LL * mode_gr * frame - 1104;
  return b > 0 ? b : 0;
}

/* Float32 input: the descriptors sds[0 .. S) point at the caller's Float32 rows.  Queues k_stage_f32, which writes them
 * scaled into the workspace (ws.refusals[0] flags a refused sample), and points the descriptors at the staged rows; the
 * sample indices stay as they were. */
int stage_streams(ThreadCtx& c, Config* cfg, StreamDesc* sds, int S) {
  const int nch = cfg->host.nch;
  Workspace& ws = c.ws;
  std::vector<StageDesc> d((size_t)S);
  long long tot = 0, max_n = 0;
  for (int i = 0; i < S; i++) {
    const long long n = sds[i].pcm_end > sds[i].pcm_base ? sds[i].pcm_end - sds[i].pcm_base : 0;
    for (int c = 0; c < 2; c++) d[i].x[c] = static_cast<const float*>(sds[i].pcm[c]);
    d[i].n = n;
    tot += n * nch;
    max_n = n > max_n ? n : max_n;
  }
  int rc = ws.st_desc.fit((size_t)S);
  if (rc) return rc;
  rc = ws.st_y.fit((size_t)tot + 1);
  if (rc) return rc;
  long long off = 0;
  for (int i = 0; i < S; i++) {
    d[i].y[0] = ws.st_y.p + off; d[i].y[1] = nch == 2 ? d[i].y[0] + d[i].n : d[i].y[0];
    off += d[i].n * nch;
    for (int c = 0; c < 2; c++) sds[i].pcm[c] = d[i].y[c];
  }
  cudaStream_t st = c.st;
  if ((rc = wait_legacy(c)) || (rc = upload(c, ws.st_desc.p, d.data(), sizeof(StageDesc) * S))) return rc;
  if (max_n > 0) {
    const long long per = (long long)STAGE_THREADS * STAGE_PER_THREAD;
    dim3 grid((unsigned)((max_n + per - 1) / per), nch, S);
    k_stage_f32<<<grid, STAGE_THREADS, 0, st>>>(ws.st_desc.p, cfg->host.scale_applied, cfg->host.scale, ws.refusals.p);
    g_launches++;
    DBG("k_stage_f32");
  }
  return 0;
}

/* Queues k_resample for the S descriptors rd (uploaded here), whose input rows `in` describes; ev_rs[0 / 1] bracket the
 * kernel (timing slot 14). */
int queue_resample(ThreadCtx& c, const Config* cfg, const ResampleDesc* rd, int S, long long max_ny, Rows in) {
  Workspace& ws = c.ws;
  cudaStream_t st = c.st;
  int rc = ws.rs_desc.fit((size_t)S);
  if (rc || (rc = upload(c, ws.rs_desc.p, rd, sizeof(ResampleDesc) * S))) return rc;
  CK(cudaEventRecord(c.ev_rs[0], st));
  if (max_ny > 0) {
    dim3 grid((unsigned)((max_ny + RS_THREADS - 1) / RS_THREADS), cfg->host.nch, S);
    if (in.f32) k_resample<float><<<grid, RS_THREADS, 0, st>>>(ws.rs_desc.p, cfg->rs.ratio, in.scale_applied, cfg->host.scale);
    else k_resample<int16_t><<<grid, RS_THREADS, 0, st>>>(ws.rs_desc.p, cfg->rs.ratio, in.scale_applied, cfg->host.scale);
    g_launches++;
    DBG("k_resample");
  }
  CK(cudaEventRecord(c.ev_rs[1], st));
  return 0;
}

/* Resampled launches: the descriptors sds[0 .. S) hold the caller's input as `in` describes (pcm_base / pcm_end count
 * input samples, and pcm_base is at most max(0, r * hist_base_at(frame0) - 16), the first input the outputs below read).
 * Queues k_resample for the outputs the streams' frames read -- from hist_base_at(frame0) up to the last output the input
 * reaches; later outputs are 0 -- into the workspace, and points the descriptors at them: from then on pcm_base / pcm_end
 * count outputs, and the stream reads like PCM at the output rate. */
int resample_streams(ThreadCtx& c, Config* cfg, StreamDesc* sds, int S, Rows in) {
  const int r = cfg->rs.ratio, nch = cfg->host.nch;
  Workspace& ws = c.ws;
  std::vector<ResampleDesc> rd((size_t)S);
  long long tot = 0, max_ny = 0;
  for (int i = 0; i < S; i++) {
    const StreamDesc& sd = sds[i];
    const long long yb = hist_base_at(cfg->host.mode_gr, sd.frame0);
    const long long xb = r * yb - MP3_RS_HALF > 0 ? r * yb - MP3_RS_HALF : 0;
    if (sd.pcm_base > xb) { g_err = "resampler input starts after the first sample it reads"; return MP3B200_ERR_HANDLE; }
    long long ye = (sd.pcm_end + MP3_RS_HALF - 1) / r + 1;      /* y[m] reads input up to r m + 16 */
    if (sd.nframes == 0 || ye < yb) ye = yb;
    ResampleDesc& d = rd[i];
    d.x[0] = sd.pcm[0]; d.x[1] = sd.pcm[1]; d.x_base = sd.pcm_base; d.x_end = sd.pcm_end;
    d.y_base = yb; d.ny = ye - yb;
    tot += d.ny * nch;
    max_ny = d.ny > max_ny ? d.ny : max_ny;
  }
  int rc = ws.rs_y.fit((size_t)tot + 1);
  if (rc) return rc;
  long long off = 0;
  for (int i = 0; i < S; i++) {
    ResampleDesc& d = rd[i];
    d.y[0] = ws.rs_y.p + off; d.y[1] = nch == 2 ? d.y[0] + d.ny : d.y[0];
    off += d.ny * nch;
    for (int c = 0; c < 2; c++) sds[i].pcm[c] = d.y[c];
    sds[i].pcm_base = d.y_base; sds[i].pcm_end = d.y_base + d.ny;
  }
  if ((rc = wait_legacy(c))) return rc;                     /* the input may come from the legacy default stream */
  return queue_resample(c, cfg, rd.data(), S, max_ny, in);
}

/* ---- ReplayGain (lamejs findReplayGain; k_replaygain.cuh) ----
 * A launch analyses, for each stream listed in the job, the samples [g0, g0 + sum(pieces)) of its current title (which
 * started at t0), reading the PCM its descriptor points at once the launch has resampled it (stream sample indices: Int16 as
 * mfbuf holds it, or the resampler's Float32 rows); `pieces` are the AnalyzeSamples calls lamejs makes for them. */
struct RgSpec {
  int stream = 0;                                /* index in the launch */
  std::vector<long long> pieces;                 /* piece sizes (LameFifo::pieces) */
  long long t0 = 0, g0 = 0;
  RgCarry* carry = nullptr;                      /* device; NULL: a fresh title in launch workspace */
  int* hist = nullptr;                           /* device A; NULL: launch workspace */
  int* hist_b = nullptr;                         /* device B of a handle (GetTitleGain moves A into it); NULL: none */
  int title_end = 1;
};
struct RgJob {
  std::vector<RgSpec> specs;
  /* results */
  std::vector<double> title_db;                  /* per spec (RG_NOT_ENOUGH_SAMPLES where the title does not end) */
  double album_db = 0;                           /* analyzeResult of the specs' summed A */
  int passes = 0, reruns = 0;
  float ms = 0;                                  /* CUDA-event time of the analysis on its stream */
  /* debug: spec 0's windows */
  bool want_windows = false;
  std::vector<double> win_sum;                   /* [windows][2] */
  std::vector<int> win_idx;
  std::vector<int> hist0;
  /* filled by rg_queue */
  long long chunk_rows = 0;
  int max_chunks = 0, max_win = 0, nwin0 = 0;
  RgParams prm;
};

int rg_req_index(int sr) {
  static const int rates[9] = {48000, 44100, 32000, 24000, 22050, 16000, 12000, 11025, 8000};
  for (int i = 0; i < 9; i++) if (rates[i] == sr) return i;
  return -1;
}

/* queues pass 1 and the first RG_QUEUED_PASSES repair passes on c.rg_st, after the PCM (the upload slices in `arrival`,
 * or everything queued on c.st so far: uploads and the resampler) */
int rg_queue(ThreadCtx& c, Config* cfg, const StreamDesc* sds, RgJob& job, const PcmArrival* arrival, Rows rows) {
  const int sr = cfg->host.samplerate, W = (sr + 19) / 20, nch = cfg->host.nch, req = rg_req_index(sr);
  if (req < 0) { g_err = "no ReplayGain filter for this rate"; return MP3B200_ERR_CONFIG; }
  const int T = (int)job.specs.size();
  std::vector<RgTitle> t((size_t)T);
  long long npiece = 0, nwin = 0, nchunk = 0;
  for (const RgSpec& sp : job.specs) npiece += (long long)sp.pieces.size();
  int rc = 0;
  if ((rc = c.rg_piece.fit((size_t)npiece + 1)) || (rc = c.rg_carry.fit((size_t)T + 1)) || (rc = c.rg_hist.fit((size_t)(T + 1) * RG_HIST)))
    return rc;
  std::vector<long long> starts((size_t)npiece + 1);
  long long po = 0;
  job.max_chunks = job.max_win = 0;
  for (int i = 0; i < T; i++) {
    const RgSpec& sp = job.specs[i];
    const StreamDesc& sd = sds[sp.stream];
    RgTitle& ti = t[i];
    ti.x[0] = sd.pcm[0]; ti.x[1] = sd.pcm[1];
    ti.x_base = sd.pcm_base; ti.x_end = sd.pcm_end;
    long long at = sp.g0;
    ti.piece = c.rg_piece.p + po;
    for (long long k : sp.pieces) { starts[po++] = at; at += k; }
    ti.npieces = (int)sp.pieces.size();
    ti.t0 = sp.t0; ti.g0 = sp.g0; ti.g1 = at;
    ti.wa = (int)((sp.g0 - sp.t0) / W);
    ti.nwin = (int)((at - sp.t0) / W) - ti.wa;
    const int pseudo = ti.nwin + (at > sp.t0 + (long long)(ti.wa + ti.nwin) * W ? 1 : 0);   /* + the partial window at g1 */
    ti.win0 = (int)nwin;
    ti.nchunks = (pseudo + RG_CHUNK_WINDOWS - 1) / RG_CHUNK_WINDOWS;
    ti.chunk0 = (int)nchunk;
    ti.carry = sp.carry ? sp.carry : c.rg_carry.p + i;
    ti.hist = sp.hist ? sp.hist : c.rg_hist.p + (size_t)i * RG_HIST;
    ti.hist_b = sp.hist_b;
    ti.title_end = sp.title_end;
    nwin += ti.nwin; nchunk += ti.nchunks;
    job.max_chunks = ti.nchunks > job.max_chunks ? ti.nchunks : job.max_chunks;
    job.max_win = ti.nwin > job.max_win ? ti.nwin : job.max_win;
  }
  job.nwin0 = T > 0 ? t[0].nwin : 0;
  job.chunk_rows = nchunk * nch;
  const int max_passes = job.max_chunks + RG_QUEUED_PASSES + 2;
  if ((rc = c.rg_titles.fit((size_t)T + 1)) || (rc = c.rg_sum.fit((size_t)nwin * 2 + 2)) || (rc = c.rg_wstate.fit((size_t)nwin * nch + 1)) ||
      (rc = c.rg_cstart.fit((size_t)job.chunk_rows + 1)) || (rc = c.rg_end_a.fit((size_t)job.chunk_rows + 1)) ||
      (rc = c.rg_end_b.fit((size_t)job.chunk_rows + 1)) || (rc = c.rg_idx.fit((size_t)nwin + 1)) ||
      (rc = c.rg_count.fit((size_t)max_passes + 2)) || (rc = c.rg_gain.fit((size_t)T + 1)))
    return rc;
  cudaStream_t st = c.rg_st;
  if (arrival) for (int j = 0; j < arrival->chunks; j++) CK(cudaStreamWaitEvent(st, arrival->ready[j], 0));
  CK(cudaEventRecord(c.ev_rg[0], c.st));
  CK(cudaStreamWaitEvent(st, c.ev_rg[0], 0));
  CK(cudaEventRecord(c.ev_rg[1], st));
  if ((rc = upload(c, c.rg_piece.p, starts.data(), sizeof(long long) * (size_t)(npiece + 1), st)) ||
      (rc = upload(c, c.rg_titles.p, t.data(), sizeof(RgTitle) * (size_t)T, st)))
    return rc;
  CK(cudaMemsetAsync(c.rg_count.p, 0, sizeof(int) * (size_t)(max_passes + 2), st));
  CK(cudaMemsetAsync(c.rg_hist.p, 0, sizeof(int) * (size_t)(T + 1) * RG_HIST, st));
  CK(cudaMemsetAsync(c.rg_carry.p, 0, sizeof(RgCarry) * (size_t)(T + 1), st));
  RgParams& p = job.prm;
  p.titles = c.rg_titles.p; p.nch = nch; p.W = W; p.req = req; p.f32 = rows.f32;
  p.scale_applied = rows.scale_applied;
  p.scale = cfg->host.scale;
  p.win_sum = c.rg_sum.p; p.win_state = c.rg_wstate.p; p.chunk_start = c.rg_cstart.p; p.end_in = c.rg_end_a.p; p.end_out = c.rg_end_b.p;
  p.done = c.rg_count.p; p.reruns = c.rg_count.p + 1; p.pass_changed = c.rg_count.p + 2;
  job.passes = 0;
  if (job.max_chunks > 0) {
    dim3 grid((unsigned)((job.max_chunks * nch + RG_THREADS - 1) / RG_THREADS), (unsigned)T);
    k_rg_pass1<<<grid, RG_THREADS, 0, st>>>(p);
    g_launches++;
    for (int q = 0; q < RG_QUEUED_PASSES; q++) {
      k_rg_repair<<<grid, RG_THREADS, 0, st>>>(p, job.passes);
      k_rg_check<<<(unsigned)((job.chunk_rows + 255) / 256), 256, 0, st>>>(p, job.passes, job.chunk_rows);
      job.passes++;
      g_launches += 2;
    }
  }
  CK(cudaGetLastError());
  return 0;
}

/* once the repair passes have ended: queues the titles' histograms, the album's, and the gains (c.rg_gain: [t] of the
 * titles that end, [T] the album's) on c.rg_st */
int rg_queue_results(ThreadCtx& c, RgJob& job) {
  cudaStream_t st = c.rg_st;
  const RgParams& p = job.prm;
  const int T = (int)job.specs.size();
  if (job.max_win > 0) {
    k_rg_hist<<<dim3((unsigned)((job.max_win + 255) / 256), (unsigned)T), 256, 0, st>>>(p.titles, p.W, p.win_sum, c.rg_idx.p);
    g_launches++;
  }
  int* album = c.rg_hist.p + (size_t)T * RG_HIST;
  k_rg_album<<<(RG_HIST + 255) / 256, 256, 0, st>>>(p.titles, T, album);
  CK(cudaMemsetAsync(c.rg_gain.p, 0, sizeof(double) * (size_t)(T + 1), st));
  k_rg_result<<<T + 1, 256, 0, st>>>(p.titles, T, album, c.rg_gain.p);
  g_launches += 2;
  return 0;
}

/* After the encoder has been queued: the repair loop runs as a graph on c.rg_st (k_rg_loop_cond), kept in c.loops per
 * shape and captured here when there is none; then the histograms, the gains of the titles that end (c.rg_gain) and the
 * carries.  `loop` is three words of device memory: the pass index, and what k_rg_report leaves there (the passes the
 * analysis needed and the chunks it ran again); *fault is set to RG_FAULT if the loop hits its bound.  Nothing is read
 * back (rg_read). */
int rg_finish(ThreadCtx& c, Config* cfg, RgJob& job, int* loop, int* fault) {
  cudaStream_t st = c.rg_st;
  RgParams& p = job.prm;
  const int nch = cfg->host.nch, T = (int)job.specs.size();
  if (job.max_chunks > 0) {
    LoopGraphs& lg = c.loops;
    lg.renew(true, c.rg_generation());
    const LoopGraphs::Key key = {cfg, 1 + (p.f32 != 0), T, job.max_chunks, job.chunk_rows, loop};
    cudaGraphExec_t exec = lg.find(key);
    if (!exec) {
      cudaGraph_t g = nullptr;
      cudaGraphConditionalHandle cond;
      cudaGraphNode_t node;
      cudaGraphNodeParams cp = {};
      cp.type = cudaGraphNodeTypeConditional;
      bool ok = cudaGraphCreate(&g, 0) == cudaSuccess;
      ok = ok && cudaGraphConditionalHandleCreate(&cond, g, 1, cudaGraphCondAssignDefault) == cudaSuccess;
      cp.conditional.handle = cond; cp.conditional.type = cudaGraphCondTypeWhile; cp.conditional.size = 1;
      ok = ok && cudaGraphAddNode(&node, g, nullptr, 0, &cp) == cudaSuccess;
      cudaGraph_t body = ok ? cp.conditional.phGraph_out[0] : nullptr;
      if (ok && cudaStreamBeginCaptureToGraph(lg.capture, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
        dim3 grid((unsigned)((job.max_chunks * nch + RG_THREADS - 1) / RG_THREADS), (unsigned)T);
        k_rg_repair_at<<<grid, RG_THREADS, 0, lg.capture>>>(p, loop);
        k_rg_check_at<<<(unsigned)((job.chunk_rows + 255) / 256), 256, 0, lg.capture>>>(p, loop, job.chunk_rows);
        k_rg_loop_cond<<<1, 1, 0, lg.capture>>>(cond, loop, p.done, job.max_chunks + RG_QUEUED_PASSES + 1, fault);
        cudaGraph_t captured = nullptr;
        ok = cudaStreamEndCapture(lg.capture, &captured) == cudaSuccess && captured == body &&
             cudaGraphInstantiate(&exec, g, 0) == cudaSuccess;
      } else {
        ok = false;
      }
      if (g) cudaGraphDestroy(g);
      if (!ok) {
        g_err = "ReplayGain loop graph failed: " + std::string(cudaGetErrorString(cudaGetLastError()));
        return MP3B200_ERR_CUDA;
      }
      lg.put(key, exec);
    }
    const int first = RG_QUEUED_PASSES;              /* the pass index the graph starts at */
    int rc = upload(c, loop, &first, sizeof first, st);
    if (rc) return rc;
    CK(cudaGraphLaunch(exec, st));
    k_rg_report<<<1, 1, 0, st>>>(loop, p.pass_changed, p.reruns);
    g_launches += 2;
  }
  const int rc = rg_queue_results(c, job);
  if (rc) return rc;
  k_rg_finish<<<T, 256, 0, st>>>(p.titles, p.end_in, nch);
  g_launches++;
  CK(cudaGetLastError());
  return 0;
}

/* A synchronous call's results of the analysis, once rg_finish's work has drained: the gains, the passes and reruns from
 * the loop words `loop`, the analysis's time and (want_windows) spec 0's windows and histogram A. */
int rg_read(ThreadCtx& c, RgJob& job, const int* loop) {
  const int T = (int)job.specs.size();
  auto fetch = [&](void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c.st); };
  std::vector<double> g((size_t)T + 1);
  int counts[2] = {0, 0};
  CK(fetch(g.data(), c.rg_gain.p, sizeof(double) * (size_t)(T + 1)));
  if (job.max_chunks > 0) CK(fetch(counts, loop + 1, sizeof counts));
  if (job.want_windows) {                          /* a whole stream's A is the workspace's (RgSpec::hist NULL) */
    job.win_sum.assign((size_t)job.nwin0 * 2, 0.0);
    job.win_idx.assign((size_t)job.nwin0, 0);
    if (job.nwin0 > 0) {
      CK(fetch(job.win_sum.data(), c.rg_sum.p, sizeof(double) * 2 * (size_t)job.nwin0));
      CK(fetch(job.win_idx.data(), c.rg_idx.p, sizeof(int) * (size_t)job.nwin0));
    }
    if (T > 0) {
      job.hist0.assign(RG_HIST, 0);
      CK(fetch(job.hist0.data(), c.rg_hist.p, sizeof(int) * RG_HIST));
    }
  }
  CK(cudaStreamSynchronize(c.st));
  CK(cudaEventElapsedTime(&job.ms, c.ev_rg[1], c.ev_rg[2]));
  job.passes = counts[0];
  job.reruns = counts[1];
  job.title_db.assign((size_t)T, (double)RG_NOT_ENOUGH_SAMPLES);
  for (int i = 0; i < T; i++) if (job.specs[i].title_end) job.title_db[i] = g[i];
  job.album_db = g[T];
  return 0;
}

/* Encodes the streams `sds`: the caller sets each descriptor's PCM, pcm_base / pcm_end, frame0, nframes, out_base (the
 * device address of its bytes) and carried state; this assigns unit_base / frame_base, grows the context's workspace and runs the pipeline.
 * The stream index is a grid y / z coordinate of several kernels (CUDA limit 65535): a larger batch runs as consecutive
 * launches of at most MP3_MAX_LAUNCH_STREAMS streams on the context's stream, the later ones behind every PCM upload.
 * Timings add up over the launches; the pass count (ws.refusals[2]) is the largest any of them needed.  The caller has
 * reset the status words (reset_words); with o.sync the call returns with its work drained and the words checked.
 * With resampling (cfg->rs.ratio > 1) the descriptors hold the caller's input as resample_streams describes; each launch
 * first resamples it (timing slot 14). */
int launch_streams(ThreadCtx& c, Config* cfg, std::vector<StreamDesc>& sds, const LaunchOpts& o) {
  if (o.timings_ms) for (int i = 0; i < 16; i++) o.timings_ms[i] = 0.0f;
  const PcmArrival* arrival = o.arrival;
  const int nstreams = (int)sds.size();
  if (o.rg && nstreams > MP3_MAX_LAUNCH_STREAMS) { g_err = "ReplayGain batches hold at most 65535 streams"; return MP3B200_ERR_HANDLE; }
  /* Before anything reads the descriptors' rows: the caller's device rows may come from the legacy default stream, and
   * rg_queue forks the analysis stream from c.st ahead of run_pipeline's own wait (Int16 rows that are neither staged
   * nor resampled are read by k_rg_pass1 where the caller left them). */
  {
    const int rc = wait_legacy(c);
    if (rc) return rc;
  }
  for (int g0 = 0; g0 < nstreams; g0 += MP3_MAX_LAUNCH_STREAMS) {
    const int n = nstreams - g0 < MP3_MAX_LAUNCH_STREAMS ? nstreams - g0 : MP3_MAX_LAUNCH_STREAMS;
    StreamDesc* group = sds.data() + g0;
    long long U = 0, F = 0;
    for (int i = 0; i < n; i++) {
      group[i].unit_base = (int)U; group[i].frame_base = (int)F;
      U += (long long)cfg->host.mode_gr * group[i].nframes; F += group[i].nframes;
    }
    if (F == 0) continue;                     /* empty group: nothing to launch */
    int rc = o.analyse_only ? 0 : c.ws.fit(n, cfg->host.nch, U, F);
    if (rc) return rc;
    const bool resampled = cfg->rs.ratio > 1;
    if (resampled || o.f32_in) {
      if (arrival)                              /* the resampler / stager reads all of the input: wait for every slice */
        for (int j = 0; j < arrival->chunks; j++) CK(cudaStreamWaitEvent(c.st, arrival->ready[j], 0));
      arrival = nullptr;
    }
    Rows rows = {false, cfg->host.scale_applied};
    if (o.f32_in) {
      rc = stage_streams(c, cfg, group, n);
      if (rc) return rc;
      rows = SCALED_F32;
    }
    if (resampled) {
      rc = resample_streams(c, cfg, group, n, rows);
      if (rc) return rc;
      rows = SCALED_F32;
    }
    if (o.rg) {
      rc = rg_queue(c, cfg, group, *o.rg, arrival, rows);
      if (rc) return rc;
    }
    Timings tm;
    rc = o.analyse_only ? 0 : run_pipeline(c, cfg, group, n, o, arrival, rows, &tm);
    if (rc) return rc;
    if (o.rg) {                                /* ws.refusals[3] is the fault word, [5 .. 8) the loop's words */
      rc = rg_finish(c, cfg, *o.rg, o.rg_loop ? o.rg_loop : c.ws.refusals.p + 5, c.ws.refusals.p + 3);
      if (rc) return rc;
      /* the analysis joins the call before anything reads what it wrote */
      CK(cudaEventRecord(c.ev_rg[2], c.rg_st));
      CK(cudaStreamWaitEvent(c.st, c.ev_rg[2], 0));
    }
    arrival = nullptr;
    float rs_ms = 0.0f;
    if (resampled && o.timings_ms && o.sync) CK(cudaEventElapsedTime(&rs_ms, c.ev_rs[0], c.ev_rs[1]));
    if (o.timings_ms) {
      const float t[16] = {tm.psy, tm.scan, tm.mask, tm.fb, tm.q1, tm.qn, tm.total, 0.0f,
                           tm.q_prepare, tm.q_search, tm.q_outer, tm.q_finish, tm.q_pack, tm.q_mid, rs_ms, 0.0f};
      for (int i = 0; i < 16; i++) o.timings_ms[i] += t[i];
    }
  }
  if (o.timings_ms && o.sync && !o.stop_after_mdct && !o.analyse_only) {
    int passes = 0;
    CK(cudaMemcpyAsync(&passes, c.ws.refusals.p + 2, sizeof passes, cudaMemcpyDeviceToHost, c.st));
    CK(cudaStreamSynchronize(c.st));
    o.timings_ms[7] = (float)passes;
  }
  return o.sync && (o.f32_in || !o.stop_after_mdct) ? check_refusals(c) : 0;
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
int mp3b200_debug_psy_capture(int on) {
  std::lock_guard<std::mutex> lk(g_psy_mu);
  if (on) { g_psy_rec.clear(); g_psy_launch = 0; }
  g_psy_capture.store(on ? 1 : 0);
  return 0;
}
int64_t mp3b200_debug_psy_take(void* buf, int64_t cap) {
  std::lock_guard<std::mutex> lk(g_psy_mu);
  const int64_t n = (int64_t)g_psy_rec.size();
  if (buf && cap >= n) {
    memcpy(buf, g_psy_rec.data(), (size_t)n);
    g_psy_rec.clear();
  }
  return n;
}

int mp3b200_set_device(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n || device >= MP3_MAX_DEVICES) { g_err = "invalid CUDA device"; return MP3B200_ERR_CUDA; }
  std::lock_guard<std::mutex> lk(g_mu);
  g_device = device;      /* existing handles keep the device they were created on */
  return 0;
}

int64_t mp3b200_stream_frames(int64_t nsamples) { return frames_for(nsamples, 2); }

int64_t mp3b200_stream_bytes(int channels, int samplerate, int kbps, int64_t nsamples) {
  return mp3b200_stream_bytes_ex(channels, samplerate, kbps, 0, nsamples);
}

int64_t mp3b200_stream_bytes_ex(int channels, int samplerate, int kbps, int flags, int64_t nsamples) {
  const Config* c = encodable_config(channels, samplerate, kbps, flags);
  if (!c || nsamples < 0) return -1;
  return bytes_of_frames(c->host, 0, frames_for(nsamples, c->host.mode_gr, c->rs.ratio));
}

int64_t mp3b200_stream_frames_cfg(int channels, int samplerate, int kbps, int64_t nsamples) {
  return mp3b200_stream_frames_ex(channels, samplerate, kbps, 0, nsamples);
}

int64_t mp3b200_stream_frames_ex(int channels, int samplerate, int kbps, int flags, int64_t nsamples) {
  const Config* c = encodable_config(channels, samplerate, kbps, flags);
  if (!c || nsamples < 0) return -1;
  return frames_for(nsamples, c->host.mode_gr, c->rs.ratio);
}

int mp3b200_granules_per_frame(int channels, int samplerate, int kbps) {
  return mp3b200_granules_per_frame_ex(channels, samplerate, kbps, 0);
}

int mp3b200_granules_per_frame_ex(int channels, int samplerate, int kbps, int flags) {
  const Config* c = encodable_config(channels, samplerate, kbps, flags);
  return c ? c->host.mode_gr : -1;
}

int mp3b200_out_samplerate(int channels, int samplerate, int kbps) { return mp3_out_samplerate(channels, samplerate, kbps); }

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

/* uploads the CRC tables to `device` on first use there (g_crc_dev) */
int crc_tables_on(int device) {
  const CrcTables& ht = crc_host();
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_crc_dev[device]) {
    CK(cudaMalloc(&g_crc_dev[device], sizeof(CrcTables)));
    CK(cudaMemcpy(g_crc_dev[device], &ht, sizeof(CrcTables), cudaMemcpyHostToDevice));
  }
  return 0;
}

/* Queues on c.st, behind whatever wrote the bytes, the music CRC (CRC-16, start 0) of the byte ranges [at[r], at[r] + len[r])
 * (absolute device addresses, like the packer's output offsets) into c.crc[r]: one k_music_crc launch per 65535 ranges.
 * The ranges go up through upload(); the CRC tables must already be on the device (crc_tables_on). */
int queue_music_crc(ThreadCtx& c, const std::vector<long long>& at, const std::vector<long long>& len) {
  const int R = (int)at.size();
  if (R == 0) return 0;
  std::vector<long long> ranges((size_t)2 * R);
  long long longest = 0;
  for (int i = 0; i < R; i++) { ranges[i] = at[i]; ranges[(size_t)R + i] = len[i]; longest = len[i] > longest ? len[i] : longest; }
  int rc = 0;
  if ((rc = c.crc_ranges.fit((size_t)2 * R)) || (rc = c.crc.fit((size_t)R)) ||
      (rc = upload(c, c.crc_ranges.p, ranges.data(), sizeof(long long) * ranges.size())))
    return rc;
  CK(cudaMemsetAsync(c.crc.p, 0, sizeof(unsigned) * (size_t)R, c.st));
  const long long pieces = (longest + CRC_PIECE_BYTES - 1) / CRC_PIECE_BYTES;
  for (int r0 = 0; r0 < R && longest > 0; r0 += 65535) {
    const int nr = R - r0 < 65535 ? R - r0 : 65535;
    dim3 grid((unsigned)((pieces + CRC_WARPS - 1) / CRC_WARPS), (unsigned)nr);
    k_music_crc<<<grid, CRC_WARPS * 32, 0, c.st>>>(nullptr, c.crc_ranges.p + r0, c.crc_ranges.p + R + r0, g_crc_dev[c.device], c.crc.p + r0);
    g_launches++;
  }
  return 0;
}

/* mp3b200_lametag_build(_ex): `field` is the tag's Radio Replay Gain field, 0 for a stream nobody analysed */
int build_lametag(int channels, int samplerate, int kbps, int flags, int64_t nframes, int64_t music_bytes, int music_crc,
                  int encoder_padding, int field, uint8_t* buf, int cap) {
  const Config* c = host_config(channels, samplerate, kbps, flags);
  if (!c) return MP3B200_ERR_CONFIG;
  const Mp3TagParams& p = c->tag;
  if (!p.fits || nframes <= 0) return 0;
  if (!buf || cap < p.frame_bytes) return p.frame_bytes;              /* like getLameTagFrame: the size it needs */
  Mp3SeekBag* bag = new Mp3SeekBag();
  bag->reset();
  bag->add_frames(nframes, p.kbps);
  const int n = mp3_tag_frame(p, *bag, music_bytes, (unsigned)music_crc, encoder_padding, buf, field);
  delete bag;
  return n;
}
}  // namespace

namespace {
/* ---- whole streams: encodeBuffer(everything) + flush() on fresh encoders of one configuration ----
 * Every whole-stream entry point fills in one WholeCall and hands it to one of two drivers: whole_sync (the calling
 * thread's context, returns with the results on the host) or whole_async (an encode session, mp3_session.inc).  Both check
 * the arguments (whole_args), get the configuration, plan the streams (stream_plan) and run the one body, whole_run. */
template <class T>     /* the rows' samples: int16_t or float (uint8_t: the encoded files the tag step alone reads) */
struct WholeCall {
  int channels, samplerate, kbps, flags, nstreams;
  /* the rows, nsamples[s] samples per channel: host rows left[s] / right[s] (right or right[s] NULL: left[s] on both
   * channels), or device rows at d_pcm + pcm_off[s] (stereo: the right channel follows the left) */
  const T* const* left = nullptr;
  const T* const* right = nullptr;
  const T* d_pcm = nullptr;
  const int64_t* pcm_off = nullptr;
  const int64_t* nsamples = nullptr;
  /* what the call does */
  bool encode = true;                    /* false: no encoder, the analysis alone or the tag step alone */
  bool tagged = false;                   /* files: the Info/LAME tag frame, then the audio */
  bool analyse = false;                  /* the ReplayGain analysis (a tagged call's only where its tag is written) */
  /* where the results go: device files at d_out + out_off[s], or host files out[s] of cap[s] bytes; out_bytes[s] each
   * file's length; title_db / album_db (optional) the analysis's gains; timings_ms (optional) the 16 timing slots */
  uint8_t* d_out = nullptr;
  const int64_t* out_off = nullptr;
  uint8_t* const* out = nullptr;
  const int64_t* cap = nullptr;
  int64_t* out_bytes = nullptr;
  double* title_db = nullptr;
  double* album_db = nullptr;
  float* timings_ms = nullptr;
  const double* title_in = nullptr;      /* the tag step alone: the title gains the tags carry (host; NULL: none) */
  RgJob* job = nullptr;                  /* debug: the caller's job, to read the analysis's windows */
  /* sessions: the gains ([nstreams] titles, then the album's) and the status words, on the device */
  bool session = false;
  double* d_gain = nullptr;
  int32_t* d_status = nullptr;
};

/* The argument rules of every whole-stream call (include/mp3b200.h, "Whole-stream calls"), checked before the
 * configuration and before any CUDA call.  MP3B200_REPLAYGAIN is a flag of the tagged encodes; the analysis alone implies it. */
template <class T>
int whole_args(const WholeCall<T>& k) {
  auto refuse = [](const char* why) { g_err = why; return MP3B200_ERR_HANDLE; };
  if (k.nstreams < 0) return refuse("negative stream count");
  if (k.flags & ~(MP3B200_RESAMPLE | (k.encode && k.tagged ? MP3B200_REPLAYGAIN : 0))) { g_err = "unknown flags"; return MP3B200_ERR_CONFIG; }
  if (k.analyse && k.nstreams > MP3_MAX_LAUNCH_STREAMS) return refuse("ReplayGain batches hold at most 65535 streams");
  if (k.session) {                       /* written by every call: the album's gain and the status words */
    if (k.analyse && !k.d_gain) return refuse("d_gain is NULL");
    if (!k.d_status) return refuse("d_status is NULL");
    if (k.tagged && !k.out_bytes) return refuse("out_bytes is NULL");
  }
  if (k.nstreams == 0) return MP3B200_OK;
  const bool files = k.encode || k.tagged;
  if (!k.nsamples || !(k.left || (k.d_pcm && k.pcm_off)) || (files && (k.left ? !k.out || !k.cap : !k.out_off)))
    return refuse("null array");
  if (!k.out_bytes && (k.left ? k.encode : k.tagged)) return refuse(k.encode ? "out_bytes is NULL" : "file_bytes is NULL");
  for (int s = 0; s < k.nstreams; s++) {
    if (k.left && !k.left[s]) return refuse("null row");
    if (k.nsamples[s] < 0) return refuse("negative sample count");
  }
  return MP3B200_OK;
}

/* What is known about whole streams before anything runs, in closed form from the lamejs FIFO: each stream's frames, audio
 * bytes and end padding, the room of its tag frame (tag[s]: tfs, or 0 where no tag is written: untagged calls, a tag that
 * does not fit, a stream without frames), and with the analysis (rg) the pieces it sees (rg->specs).  A tagged stream is
 * analysed only when its tag is written (Lame.js:911-916): rg is then NULL where the tag does not fit. */
struct StreamPlan {
  int tfs = 0;
  RgJob* rg = nullptr;
  std::vector<long long> frames, audio;
  std::vector<int> padding, tag;
};
StreamPlan stream_plan(const Config* cfg, int nstreams, const int64_t* nsamples, bool tagged, RgJob* rg) {
  StreamPlan pl;
  pl.tfs = tagged && cfg->tag.fits ? cfg->tag.frame_bytes : 0;
  pl.rg = tagged && !cfg->tag.fits ? nullptr : rg;
  if (pl.rg) pl.rg->specs.assign((size_t)nstreams, RgSpec());
  pl.frames.resize((size_t)nstreams); pl.audio.resize((size_t)nstreams); pl.padding.resize((size_t)nstreams); pl.tag.resize((size_t)nstreams);
  for (int s = 0; s < nstreams; s++) {
    LameFifo fifo(cfg->host.mode_gr, cfg->rs.ratio);
    if (pl.rg) { pl.rg->specs[s].stream = s; fifo.pieces = &pl.rg->specs[s].pieces; }
    const long long fed = fifo.feed(nsamples[s]);
    const FifoFlush fl = fifo.flush();
    pl.frames[s] = fed + fl.frames;
    pl.audio[s] = bytes_of_frames(cfg->host, 0, pl.frames[s]);
    pl.padding[s] = fl.end_padding;
    pl.tag[s] = pl.tfs > 0 && pl.frames[s] > 0 ? pl.tfs : 0;
  }
  return pl;
}

/* The descriptors of whole streams: stream s reads nsamples[s] samples per channel at d_pcm + pcm_off[s] (stereo: the right
 * channel follows the left) and writes its audio at d_out + out_off[s] + plan.tag[s], behind the room of its tag frame
 * (out_off NULL: the analysis alone, which writes no bytes). */
template <class T>     /* int16_t, or float (the launch stages the rows: LaunchOpts::f32_in) */
std::vector<StreamDesc> whole_streams(const Config* cfg, const StreamPlan& pl, int nstreams, const T* d_pcm, const int64_t* pcm_off,
                                      const int64_t* nsamples, uint8_t* d_out, const int64_t* out_off) {
  std::vector<StreamDesc> sds(nstreams);
  for (int s = 0; s < nstreams; s++) {
    StreamDesc& sd = sds[s];
    memset(&sd, 0, sizeof sd);
    const T* x = d_pcm + pcm_off[s];
    sd.pcm[0] = x;
    sd.pcm[1] = cfg->host.nch == 2 ? x + nsamples[s] : x;
    sd.pcm_base = 0; sd.pcm_end = nsamples[s];
    sd.frame0 = 0; sd.nframes = (int)pl.frames[s];
    sd.out_base = out_off ? (long long)(uintptr_t)(d_out + out_off[s] + pl.tag[s]) : 0;
    init_stream_state(sd);
  }
  return sds;
}

/* Queues, behind the packer on c.st, what turns the audio of tagged whole streams into files: the music CRC of each stream
 * where its audio lies (sds[i].out_base), and k_tag_finish, which completes each template frame with it and with the field
 * of gain[i] (device; NULL: the field is 0) and writes it to d_out + out_off[i].  The templates are mp3_tag_frame with music
 * CRC 0 and gain field 0.  Every upload goes through upload(). */
int finish_tagged(ThreadCtx& c, Config* cfg, const StreamPlan& plan, const std::vector<StreamDesc>& sds, uint8_t* d_out,
                  const int64_t* out_off, const double* gain) {
  const int S = (int)sds.size();
  const Mp3TagParams& p = cfg->tag;
  int ntags = 0;
  for (int i = 0; i < S; i++) ntags += plan.tag[i] ? 1 : 0;
  if (ntags == 0) return 0;
  std::vector<long long> at((size_t)S);
  for (int i = 0; i < S; i++) at[i] = sds[i].out_base;
  int rc = queue_music_crc(c, at, plan.audio);
  if (rc) return rc;
  /* the template frames: everything but the music CRC, the gain field and the frame's own CRC */
  const size_t tfs = (size_t)plan.tfs;
  std::vector<TagDest> dst((size_t)ntags);
  std::vector<uint8_t> frames(tfs * (size_t)ntags);
  Mp3SeekBag* bag = new Mp3SeekBag();
  for (int i = 0, k = 0; i < S; i++) {
    if (!plan.tag[i]) continue;
    bag->reset();
    bag->add_frames(plan.frames[i], p.kbps);
    mp3_tag_frame(p, *bag, plan.audio[i], 0, plan.padding[i], frames.data() + tfs * (size_t)k, 0);
    dst[k].at = d_out + out_off[i]; dst[k].stream = i;
    k++;
  }
  delete bag;
  const size_t dst_bytes = (sizeof(TagDest) * (size_t)ntags + 255) & ~(size_t)255;
  if ((rc = c.tags.fit(dst_bytes + frames.size())) || (rc = upload(c, c.tags.p, dst.data(), sizeof(TagDest) * dst.size())) ||
      (rc = upload(c, c.tags.p + dst_bytes, frames.data(), frames.size())))
    return rc;
  k_tag_finish<<<ntags, TAG_FINISH_THREADS, 0, c.st>>>(reinterpret_cast<const TagDest*>(c.tags.p), c.tags.p + dst_bytes, p, c.crc.p, gain);
  g_launches++;
  CK(cudaGetLastError());
  return 0;
}

/* the thread's device buffer for n samples of host PCM of type T; NULL (g_err set) when it cannot grow */
template <class T> T* staging_pcm(size_t n) { return t_ctx.pcm.fit(sizeof(T) * n) ? nullptr : reinterpret_cast<T*>(t_ctx.pcm.p); }

/* the right row of stream s: stereo input with right == NULL or right[s] == NULL encodes left[s] on both channels */
template <class T> const T* right_row(const T* const* left, const T* const* right, int s) { return right && right[s] ? right[s] : left[s]; }

/* Float32 input (lamejs's store and scale): true when every sample, scaled like k_stage_f32 scales it, is finite and
 * within MP3_F32_MAX_SAMPLE */
bool finite_after_scale(const Mp3Tables& T, const float* x, long long n) {
  for (long long i = 0; i < n; i++) {
    float v = x[i];
    if (T.scale_applied) v = (float)((double)v * T.scale);
    if (!(std::fabs(v) <= MP3_F32_MAX_SAMPLE)) return false;   /* also false for NaN */
  }
  return true;
}

/* The input gate of the host entry points: the caller's rows are checked before anything runs, and refused with
 * MP3B200_ERR_CONFIG.  Int16 rows always pass; Float32 rows must stay finite through lamejs's store and scale. */
template <class T> int check_input(const Config*, int, const T* const*, const T* const*, const int64_t*) { return MP3B200_OK; }
int check_input(const Config* cfg, int nstreams, const float* const* left, const float* const* right, const int64_t* nsamples) {
  for (int s = 0; s < nstreams; s++)
    if (!finite_after_scale(cfg->host, left[s], nsamples[s]) ||
        (cfg->host.nch == 2 && !finite_after_scale(cfg->host, right_row(left, right, s), nsamples[s]))) {
      g_err = "non-finite input sample (or one beyond 2^40 once scaled)"; return MP3B200_ERR_CONFIG;
    }
  return MP3B200_OK;
}

/* Host PCM is uploaded in time slices on a copy stream; the psy analysis of a slice starts when it has landed, so only the
 * first slice's transfer is exposed.  Many small streams are uploaded whole (one slice): per-copy overhead would win. */
int upload_slices(int nstreams, long long tot_samples) {
  return (nstreams <= 8 && tot_samples >= (1 << 20)) ? MP3_MAX_PCM_CHUNKS : 1;
}

/* Stages the rows of host streams (Int16 or Float32) in the thread's buffer, stream s at d_pcm + pcm_off[s] laid out as
 * whole_streams reads it, and fills the upload's arrival `arr`.  Stereo input with right == NULL or right[s] == NULL takes
 * left[s] for both channels. */
template <class T>
int upload_host_rows(const Config* cfg, int nstreams, const T* const* left, const T* const* right, const int64_t* nsamples,
                     std::vector<int64_t>& pcm_off, T*& d_pcm, PcmArrival& arr) {
  const int nch = cfg->host.nch;
  pcm_off.assign(nstreams, 0);
  long long tot_samples = 0;
  for (int s = 0; s < nstreams; s++) {
    pcm_off[s] = tot_samples;
    tot_samples += nsamples[s] * nch;
  }
  d_pcm = staging_pcm<T>((size_t)tot_samples + 8);
  if (!d_pcm) return MP3B200_ERR_CUDA;
  arr.chunks = upload_slices(nstreams, tot_samples);
  arr.ready = t_ctx.ready;
  for (int j = 0; j < arr.chunks; j++) {
    for (int s = 0; s < nstreams; s++) {
      const int64_t lo = nsamples[s] * j / arr.chunks, hi = nsamples[s] * (j + 1) / arr.chunks;
      if (hi <= lo) continue;
      CK(cudaMemcpyAsync(d_pcm + pcm_off[s] + lo, left[s] + lo, sizeof(T) * (hi - lo), cudaMemcpyHostToDevice, t_ctx.up_st));
      if (nch == 2)
        CK(cudaMemcpyAsync(d_pcm + pcm_off[s] + nsamples[s] + lo, right_row(left, right, s) + lo, sizeof(T) * (hi - lo),
                           cudaMemcpyHostToDevice, t_ctx.up_st));
    }
    CK(cudaEventRecord(t_ctx.ready[j], t_ctx.up_st));
  }
  return MP3B200_OK;
}

/* The body of every whole-stream call, on context c once it is planned (pl): stages host rows (upload_host_rows), describes
 * the streams (whole_streams), resets the status words, encodes and / or analyses them (launch_streams; o.arrival, o.rg and
 * o.analyse_only are set here) and writes the tag frames (finish_tagged).  The files lie at k.d_out + k.out_off[s] on the device; k.out_bytes[s]
 * (optional) receives each file's length. */
template <class T>
int whole_run(ThreadCtx& c, Config* cfg, const WholeCall<T>& k, const StreamPlan& pl, LaunchOpts o) {
  const int S = k.nstreams;
  std::vector<int64_t> staged_off;
  T* staged = nullptr;
  PcmArrival arr;
  if (k.left) {
    const int rc = upload_host_rows(cfg, S, k.left, k.right, k.nsamples, staged_off, staged, arr);
    if (rc) return rc;
    o.arrival = &arr;
  }
  std::vector<StreamDesc> sds = whole_streams(cfg, pl, S, k.left ? staged : k.d_pcm, k.left ? staged_off.data() : k.pcm_off,
                                              k.nsamples, k.d_out, k.out_off);
  for (int s = 0; k.out_bytes && s < S; s++) k.out_bytes[s] = pl.audio[s] + pl.tag[s];
  o.rg = pl.rg;
  o.analyse_only = !k.encode;
  /* launch_streams returns with the refusals checked when it synchronises: no tag for a refused call.  The tag step alone
   * waits for the caller's files as a launch waits for its rows. */
  int rc = reset_words(c, S);
  if (!rc) rc = k.encode || pl.rg ? launch_streams(c, cfg, sds, o) : wait_legacy(c);
  if (rc || !k.tagged) return rc;
  const double* gain = pl.rg ? c.rg_gain.p : nullptr;
  if (k.title_in && S > 0) {
    if ((rc = c.rg_gain.fit((size_t)S)) || (rc = upload(c, c.rg_gain.p, k.title_in, sizeof(double) * (size_t)S))) return rc;
    gain = c.rg_gain.p;
  }
  return finish_tagged(c, cfg, pl, sds, k.d_out, k.out_off, gain);
}

template <class T>
int whole_sync_run(WholeCall<T> k, Config* cfg, const PcmArrival* arrival = nullptr, int* album_hist = nullptr);

/* The synchronous driver, on the calling thread's context: host files are laid out in t_ctx.out and copied into out[s];
 * returns with every result on the host. */
template <class T>
int whole_sync(WholeCall<T> k) {
  Config* cfg = nullptr;
  int rc = whole_args(k);
  if (rc || (rc = get_config(k.channels, k.samplerate, k.kbps, k.flags & MP3B200_RESAMPLE, &cfg))) return rc;
  return whole_sync_run(k, cfg);
}

/* whole_sync once the arguments are checked and the configuration is bound.  Device rows (k.d_pcm) may be written to host
 * files (k.out): the WAV calls stage their rows themselves and pass the upload's `arrival`.  album_hist (optional, RG_HIST
 * ints) receives the album histogram of the streams analysed (zeros where none were). */
template <class T>
int whole_sync_run(WholeCall<T> k, Config* cfg, const PcmArrival* arrival, int* album_hist) {
  int rc = 0;
  if ((k.left && (rc = check_input(cfg, k.nstreams, k.left, k.right, k.nsamples))) || (k.tagged && (rc = crc_tables_on(t_ctx.device))))
    return rc;
  const int S = k.nstreams;
  RgJob job;
  const StreamPlan pl = stream_plan(cfg, S, k.nsamples, k.tagged, k.analyse ? (k.job ? k.job : &job) : nullptr);
  std::vector<int64_t> file_off;
  if (k.out) {
    long long tot = 0;
    file_off.resize((size_t)S);
    for (int s = 0; s < S; s++) {
      if (k.cap[s] < pl.audio[s] + pl.tag[s]) { g_err = "output buffer too small"; return MP3B200_ERR_BUFFER; }
      file_off[s] = tot;
      tot += pl.audio[s] + pl.tag[s];
    }
    if ((rc = t_ctx.out.fit((size_t)tot + 8))) return rc;
    k.d_out = t_ctx.out.p;
    k.out_off = file_off.data();
  }
  LaunchOpts o;
  o.f32_in = std::is_same_v<T, float>;
  o.timings_ms = k.timings_ms;
  o.arrival = arrival;
  if ((rc = whole_run(t_ctx, cfg, k, pl, o))) return rc;
  if (k.out || k.tagged) {               /* the copies and the tag step are still queued */
    for (int s = 0; k.out && s < S; s++)
      CK(cudaMemcpyAsync(k.out[s], k.d_out + k.out_off[s], (size_t)k.out_bytes[s], cudaMemcpyDeviceToHost, t_ctx.st));
    CK(cudaStreamSynchronize(t_ctx.st));
    CK(cudaGetLastError());
  }
  if (pl.rg && S > 0 && (rc = rg_read(t_ctx, *pl.rg, t_ctx.ws.refusals.p + 5))) return rc;
  const bool ran = pl.rg && (int)pl.rg->title_db.size() == S && S > 0;
  for (int s = 0; k.title_db && s < S; s++) k.title_db[s] = ran ? pl.rg->title_db[s] : RG_NOT_ENOUGH_SAMPLES;
  if (k.album_db) *k.album_db = ran ? pl.rg->album_db : RG_NOT_ENOUGH_SAMPLES;
  if (album_hist) {                      /* rg_queue_results left the album's histogram behind the titles' */
    if (ran) CK(cudaMemcpy(album_hist, t_ctx.rg_hist.p + (size_t)S * RG_HIST, sizeof(int) * RG_HIST, cudaMemcpyDeviceToHost));
    else memset(album_hist, 0, sizeof(int) * RG_HIST);
  }
  return MP3B200_OK;
}
}  // namespace

extern "C" {

int mp3b200_encode_streams(int channels, int samplerate, int kbps, int nstreams, const int16_t* const* left,
                           const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                           const int64_t* cap, int64_t* out_bytes) {
  return mp3b200_encode_streams_ex(channels, samplerate, kbps, 0, nstreams, left, right, nsamples, out, cap, out_bytes);
}

int mp3b200_encode_streams_ex(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* const* left,
                              const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                              const int64_t* cap, int64_t* out_bytes) {
  return whole_sync<int16_t>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                              .left = left, .right = right, .nsamples = nsamples, .out = out, .cap = cap, .out_bytes = out_bytes});
}

int mp3b200_encode_streams_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* const* left,
                               const float* const* right, const int64_t* nsamples, uint8_t* const* out,
                               const int64_t* cap, int64_t* out_bytes) {
  return whole_sync<float>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                            .left = left, .right = right, .nsamples = nsamples, .out = out, .cap = cap, .out_bytes = out_bytes});
}

int mp3b200_encode_streams_device(int channels, int samplerate, int kbps, int nstreams, const int16_t* d_pcm,
                                  const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                  const int64_t* out_off, float* timings_ms) {
  return mp3b200_encode_streams_device_ex(channels, samplerate, kbps, 0, nstreams, d_pcm, pcm_off, nsamples, d_out, out_off, timings_ms);
}

int mp3b200_encode_streams_device_ex(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* d_pcm,
                                     const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                     const int64_t* out_off, float* timings_ms) {
  return whole_sync<int16_t>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                              .d_pcm = d_pcm, .pcm_off = pcm_off, .nsamples = nsamples, .d_out = d_out, .out_off = out_off,
                              .timings_ms = timings_ms});
}

int mp3b200_encode_streams_device_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* d_pcm,
                                      const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                      const int64_t* out_off, float* timings_ms) {
  return whole_sync<float>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                            .d_pcm = d_pcm, .pcm_off = pcm_off, .nsamples = nsamples, .d_out = d_out, .out_off = out_off,
                            .timings_ms = timings_ms});
}

int mp3b200_encode_streams_tagged(int channels, int samplerate, int kbps, int nstreams, const int16_t* const* left,
                                  const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                                  const int64_t* cap, int64_t* out_bytes) {
  return mp3b200_encode_streams_tagged_ex(channels, samplerate, kbps, 0, nstreams, left, right, nsamples, out, cap, out_bytes,
                                          nullptr, nullptr);
}

int mp3b200_encode_streams_tagged_ex(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* const* left,
                                     const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                                     const int64_t* cap, int64_t* out_bytes, double* title_db, double* album_db) {
  return whole_sync<int16_t>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                              .left = left, .right = right, .nsamples = nsamples, .tagged = true,
                              .analyse = (flags & MP3B200_REPLAYGAIN) != 0, .out = out, .cap = cap, .out_bytes = out_bytes,
                              .title_db = title_db, .album_db = album_db});
}

int mp3b200_encode_streams_tagged_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* const* left,
                                      const float* const* right, const int64_t* nsamples, uint8_t* const* out,
                                      const int64_t* cap, int64_t* out_bytes, double* title_db, double* album_db) {
  return whole_sync<float>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                            .left = left, .right = right, .nsamples = nsamples, .tagged = true,
                            .analyse = (flags & MP3B200_REPLAYGAIN) != 0, .out = out, .cap = cap, .out_bytes = out_bytes,
                            .title_db = title_db, .album_db = album_db});
}

int mp3b200_encode_streams_tagged_device(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* d_pcm,
                                         const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out, const int64_t* out_off,
                                         int64_t* out_bytes, double* title_db, double* album_db) {
  return whole_sync<int16_t>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                              .d_pcm = d_pcm, .pcm_off = pcm_off, .nsamples = nsamples, .tagged = true,
                              .analyse = (flags & MP3B200_REPLAYGAIN) != 0, .d_out = d_out, .out_off = out_off,
                              .out_bytes = out_bytes, .title_db = title_db, .album_db = album_db});
}

int mp3b200_encode_streams_tagged_device_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* d_pcm,
                                             const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out, const int64_t* out_off,
                                             int64_t* out_bytes, double* title_db, double* album_db) {
  return whole_sync<float>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                            .d_pcm = d_pcm, .pcm_off = pcm_off, .nsamples = nsamples, .tagged = true,
                            .analyse = (flags & MP3B200_REPLAYGAIN) != 0, .d_out = d_out, .out_off = out_off,
                            .out_bytes = out_bytes, .title_db = title_db, .album_db = album_db});
}

int mp3b200_replaygain_streams(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* const* left,
                               const int16_t* const* right, const int64_t* nsamples, double* title_db, double* album_db) {
  return whole_sync<int16_t>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                              .left = left, .right = right, .nsamples = nsamples, .encode = false, .analyse = true,
                              .title_db = title_db, .album_db = album_db});
}
int mp3b200_replaygain_streams_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* const* left,
                                   const float* const* right, const int64_t* nsamples, double* title_db, double* album_db) {
  return whole_sync<float>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                            .left = left, .right = right, .nsamples = nsamples, .encode = false, .analyse = true,
                            .title_db = title_db, .album_db = album_db});
}
int mp3b200_replaygain_streams_device(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* d_pcm,
                                      const int64_t* pcm_off, const int64_t* nsamples, double* title_db, double* album_db) {
  return whole_sync<int16_t>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                              .d_pcm = d_pcm, .pcm_off = pcm_off, .nsamples = nsamples, .encode = false, .analyse = true,
                              .title_db = title_db, .album_db = album_db});
}
int mp3b200_replaygain_streams_device_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* d_pcm,
                                          const int64_t* pcm_off, const int64_t* nsamples, double* title_db, double* album_db) {
  return whole_sync<float>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                            .d_pcm = d_pcm, .pcm_off = pcm_off, .nsamples = nsamples, .encode = false, .analyse = true,
                            .title_db = title_db, .album_db = album_db});
}

/* the tag step alone: the encoded files are the call's rows, and its output */
int mp3b200_finish_tags_device(int channels, int samplerate, int kbps, int flags, int nstreams, uint8_t* d_files,
                               const int64_t* file_off, const int64_t* nsamples, const double* title_db, int64_t* file_bytes) {
  return whole_sync<uint8_t>({.channels = channels, .samplerate = samplerate, .kbps = kbps, .flags = flags, .nstreams = nstreams,
                              .d_pcm = d_files, .pcm_off = file_off, .nsamples = nsamples, .encode = false, .tagged = true,
                              .d_out = d_files, .out_off = file_off, .out_bytes = file_bytes, .title_in = title_db});
}

}  // extern "C"

extern "C" {

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

}  // extern "C"

namespace {
/* mp3b200_debug_stages_ex with the input `left` / `right` (Int16 or Float32) instead of the struct's */
template <class T>
int debug_stages(const mp3b200_debug_taps* tp, const T* left, const T* right) {
  if (!tp || tp->size != (int32_t)sizeof(mp3b200_debug_taps)) { g_err = "mp3b200_debug_taps: size must be sizeof(mp3b200_debug_taps)"; return MP3B200_ERR_HANDLE; }
  const int channels = tp->channels;
  const int64_t nsamples = tp->nsamples;
  const int32_t* force_blocktype = tp->force_blocktype;
  float *xr = tp->xr, *en_l = tp->en_l, *thm_l = tp->thm_l, *en_s = tp->en_s, *thm_s = tp->thm_s;
  int32_t *blocktype = tp->blocktype, *l3_enc = tp->l3_enc, *ginfo = tp->ginfo;
  double* ath_adjust = tp->ath_adjust;
  uint8_t* bytes_out = tp->bytes_out;
  const int64_t bytes_cap = tp->bytes_cap;
  Config* cfg;
  int rc = get_config(channels, tp->samplerate, tp->kbps, tp->flags, &cfg);
  if (rc || (rc = check_input(cfg, 1, &left, &right, &nsamples))) return rc;
  const int nch = cfg->host.nch;
  const int G = cfg->host.mode_gr;
  /* one whole stream, staged and encoded like a batch of host streams of one.  nsamples are the caller's (input) samples;
   * frames and granules are those of the rate the configuration encodes at. */
  const StreamPlan pl = stream_plan(cfg, 1, &nsamples, false, nullptr);
  const long long F = pl.frames[0], U = G * F, nbytes = pl.audio[0];
  std::vector<int64_t> pcm_off;
  T* d_pcm = nullptr;
  PcmArrival arr;
  if ((rc = upload_host_rows(cfg, 1, &left, &right, &nsamples, pcm_off, d_pcm, arr)) || (rc = t_ctx.out.fit((size_t)nbytes + 8))) return rc;
  uint8_t* d_out = t_ctx.out.p;
  const int64_t zero = 0;
  std::vector<StreamDesc> sds = whole_streams(cfg, pl, 1, d_pcm, pcm_off.data(), &nsamples, d_out, &zero);
  const bool want_gi = ginfo || tp->scalefac || tp->subblock_gain;
  const bool want_prep = tp->xmin || tp->max_nonzero_coeff || tp->xrpow_max;
  const bool want_q = tp->scfsi || tp->old_value || tp->cur_step;
  LaunchOpts opts;
  opts.f32_in = std::is_same_v<T, float>;
  opts.force_bt = force_blocktype;
  opts.all_short = true;
  opts.stop_after_mdct = !(l3_enc || bytes_out || want_gi || want_prep || want_q);
  opts.arrival = &arr;
  rc = reset_words(t_ctx, 1);
  if (!rc) rc = launch_streams(t_ctx, cfg, sds, opts);
  /* read-back on the thread's stream (the launch has drained it) */
  auto fetch = [](void* dst, const void* src, size_t bytes) {
    const cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, t_ctx.st);
    return e != cudaSuccess ? e : cudaStreamSynchronize(t_ctx.st);
  };
  const Workspace& ws = t_ctx.ws;
  if (rc == 0) {
    if (xr) CK(fetch(xr, ws.xr.p, sizeof(float) * (size_t)U * nch * 576));
    if (blocktype) {
      std::vector<signed char> bt((size_t)U * 2);
      CK(fetch(bt.data(), ws.bt_final.p, bt.size()));
      for (long long u = 0; u < U; u++) for (int c = 0; c < nch; c++) blocktype[u * nch + c] = bt[u * 2 + c];
    }
    if (en_l || thm_l || en_s || thm_s) {
      /* masking used by granule u is the ratio of psy unit u-1: row (u + 1 - 1) of the halo-shifted array */
      std::vector<PsyRatioDev> r((size_t)(U + 1) * nch);
      CK(fetch(r.data(), ws.ratio.p, sizeof(PsyRatioDev) * r.size()));
      for (long long u = 0; u < U; u++) for (int c = 0; c < nch; c++) {
        const PsyRatioDev& q = r[(size_t)u * nch + c];
        if (en_l) memcpy(en_l + (u * nch + c) * 22, q.en_l, sizeof q.en_l);
        if (thm_l) memcpy(thm_l + (u * nch + c) * 22, q.thm_l, sizeof q.thm_l);
        if (en_s) memcpy(en_s + (u * nch + c) * 39, q.en_s, sizeof q.en_s);
        if (thm_s) memcpy(thm_s + (u * nch + c) * 39, q.thm_s, sizeof q.thm_s);
      }
    }
    if (ath_adjust) CK(fetch(ath_adjust, ws.ath_q.p, sizeof(double) * (size_t)F));
    if (l3_enc) {
      std::vector<short> t((size_t)U * nch * 576);
      CK(fetch(t.data(), ws.l3enc.p, sizeof(short) * t.size()));
      for (size_t i = 0; i < t.size(); i++) l3_enc[i] = t[i];
    }
    if (want_gi) {
      std::vector<GranuleInfoDev> g((size_t)U * nch);
      CK(fetch(g.data(), ws.ginfo.p, sizeof(GranuleInfoDev) * g.size()));
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
      CK(fetch(p.data(), ws.prep.p, sizeof(GcPrep) * p.size()));
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
      CK(fetch(q.data(), ws.qstate.p, sizeof(QuantFrameState) * q.size()));
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
      else CK(fetch(bytes_out, d_out, (size_t)nbytes));
    }
  }
  return rc;
}

template <class T>
int debug_resample(int channels, int samplerate, int kbps, const T* left, const T* right, int64_t nsamples, float* y, int64_t ny) {
  if (nsamples < 0 || ny < 0 || (nsamples > 0 && !left) || (ny > 0 && !y)) { g_err = "bad buffers"; return MP3B200_ERR_HANDLE; }
  Config* cfg;
  int rc = get_config(channels, samplerate, kbps, MP3B200_RESAMPLE, &cfg);
  if (rc) return rc;
  if (cfg->rs.ratio == 1) { g_err = "this configuration does not resample"; return MP3B200_ERR_CONFIG; }
  if ((rc = check_input(cfg, 1, &left, &right, &nsamples))) return rc;
  if (ny == 0) return 0;
  const int nch = cfg->host.nch;
  std::vector<int64_t> pcm_off;
  T* d_pcm = nullptr;
  PcmArrival arr;
  if ((rc = upload_host_rows(cfg, 1, &left, &right, &nsamples, pcm_off, d_pcm, arr)) || (rc = t_ctx.ws.rs_y.fit((size_t)(ny * nch))))
    return rc;
  for (int j = 0; j < arr.chunks; j++) CK(cudaStreamWaitEvent(t_ctx.st, arr.ready[j], 0));   /* the resampler reads all of it */
  StreamDesc sd;
  memset(&sd, 0, sizeof sd);
  sd.pcm[0] = d_pcm;
  sd.pcm[1] = nch == 2 ? d_pcm + nsamples : d_pcm;
  sd.pcm_end = nsamples;
  Rows rows = {false, cfg->host.scale_applied};
  if (std::is_same_v<T, float>) {                   /* the launch path's staging: Float32(x * scale) rows */
    rc = t_ctx.ws.refusals.fit(MP3_SESSION_WORDS);
    if (rc) return rc;
    rc = stage_streams(t_ctx, cfg, &sd, 1);
    if (rc) return rc;
    rows = SCALED_F32;
  }
  ResampleDesc d;
  d.x[0] = sd.pcm[0]; d.x[1] = sd.pcm[1]; d.x_base = 0; d.x_end = nsamples;
  d.y[0] = t_ctx.ws.rs_y.p; d.y[1] = d.y[0] + (nch == 2 ? ny : 0); d.y_base = 0; d.ny = ny;
  rc = queue_resample(t_ctx, cfg, &d, 1, ny, rows);
  if (rc) return rc;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(y, t_ctx.ws.rs_y.p, sizeof(float) * (size_t)(ny * nch), cudaMemcpyDeviceToHost, t_ctx.st));
  CK(cudaStreamSynchronize(t_ctx.st));
  return 0;
}

/* one tagged whole stream with the analysis, and the analysis's windows */
template <class T>
int debug_replaygain(int channels, int samplerate, int kbps, int flags, const T* left, const T* right, int64_t nsamples,
                     double* win_sums, int32_t* win_idx, int64_t nwin_cap, int32_t* hist, double* title_db, int32_t* stats) {
  RgJob job;
  job.want_windows = true;
  const Config* c = encodable_config(channels, samplerate, kbps, flags & MP3B200_RESAMPLE);
  if (!c) { g_err = "unsupported configuration"; return MP3B200_ERR_CONFIG; }
  if (!c->tag.fits) { g_err = "the tag does not fit: no ReplayGain"; return MP3B200_ERR_CONFIG; }
  const int64_t cap = bytes_of_frames(c->host, 0, frames_for(nsamples, c->host.mode_gr, c->rs.ratio)) + c->tag.frame_bytes;
  std::vector<uint8_t> out((size_t)cap);
  uint8_t* outp = out.data();
  int64_t ob = 0;
  const int rc = whole_sync<T>({.channels = channels, .samplerate = samplerate, .kbps = kbps,
                                .flags = (flags & MP3B200_RESAMPLE) | MP3B200_REPLAYGAIN, .nstreams = 1, .left = &left, .right = &right,
                                .nsamples = &nsamples, .tagged = true, .analyse = true, .out = &outp, .cap = &cap, .out_bytes = &ob,
                                .job = &job});
  if (rc) return rc;
  const long long n = (long long)job.win_idx.size();
  for (long long w = 0; w < n && w < nwin_cap; w++) {
    if (win_sums) { win_sums[2 * w] = job.win_sum[2 * w]; win_sums[2 * w + 1] = job.win_sum[2 * w + 1]; }
    if (win_idx) win_idx[w] = job.win_idx[w];
  }
  if (hist && !job.hist0.empty()) memcpy(hist, job.hist0.data(), sizeof(int32_t) * RG_HIST);
  if (title_db) *title_db = job.title_db[0];
  if (stats) { stats[0] = (int32_t)n; stats[1] = job.passes; stats[2] = job.reruns; memcpy(stats + 3, &job.ms, sizeof(float)); }
  return 0;
}
}  // namespace

extern "C" {

int mp3b200_debug_stages_ex(const mp3b200_debug_taps* tp) { return debug_stages(tp, tp ? tp->left : nullptr, tp ? tp->right : nullptr); }
int mp3b200_debug_stages_f32(const mp3b200_debug_taps* tp, const float* left, const float* right) { return debug_stages(tp, left, right); }

int mp3b200_debug_resample(int channels, int samplerate, int kbps, const int16_t* left, const int16_t* right, int64_t nsamples,
                           float* y, int64_t ny) {
  return debug_resample(channels, samplerate, kbps, left, right, nsamples, y, ny);
}
int mp3b200_debug_resample_f32(int channels, int samplerate, int kbps, const float* left, const float* right, int64_t nsamples,
                               float* y, int64_t ny) {
  return debug_resample(channels, samplerate, kbps, left, right, nsamples, y, ny);
}

int mp3b200_debug_replaygain(int channels, int samplerate, int kbps, int flags, const int16_t* left, const int16_t* right,
                             int64_t nsamples, double* win_sums, int32_t* win_idx, int64_t nwin_cap, int32_t* hist,
                             double* title_db, int32_t* stats) {
  return debug_replaygain(channels, samplerate, kbps, flags, left, right, nsamples, win_sums, win_idx, nwin_cap, hist, title_db, stats);
}
int mp3b200_debug_replaygain_f32(int channels, int samplerate, int kbps, int flags, const float* left, const float* right,
                                 int64_t nsamples, double* win_sums, int32_t* win_idx, int64_t nwin_cap, int32_t* hist,
                                 double* title_db, int32_t* stats) {
  return debug_replaygain(channels, samplerate, kbps, flags, left, right, nsamples, win_sums, win_idx, nwin_cap, hist, title_db, stats);
}
}  // extern "C"

namespace {
/* ---- WAV files (include/mp3b200.h "WAV files in, MP3 files out", DESIGN.md 18) ---- */

/* One file's outcome from its bytes alone (host arithmetic): lamejs's header, view and split, then the 16-bit PCM rule and
 * the configuration. */
mp3b200_wav_plan_entry wav_plan_file(int kbps, int flags, bool tagged, const uint8_t* f, long long len) {
  mp3b200_wav_plan_entry e;
  memset(&e, 0, sizeof e);
  long long off = 0, dl = 0;
  int ch = 0;
  unsigned sr = 0;
  const int hdr = mp3_wav_read_header(f, len, &off, &dl, &ch, &sr);
  if (hdr == 0) { e.status = MP3B200_WAV_NOT_WAV; return e; }
  if (hdr == -1) { e.status = MP3B200_WAV_EXTENDED_FMT; return e; }
  if (hdr != 1) { e.status = MP3B200_WAV_RANGE_ERROR; return e; }
  e.channels = ch;
  e.sample_rate = sr > 0x7fffffffu ? -1 : (int32_t)sr;
  e.data_offset = off;
  /* new Int16Array(buffer, dataOffset, dataLen / 2): the length truncates; an odd offset or a view past the end throws.
   * new Int16Array(dataLen / (2 channels)) throws for 0 channels with data (length Infinity; 0 / 0 is NaN, length 0). */
  const long long view = dl / 2;
  if ((off & 1) || off + 2 * view > len || (ch == 0 && dl > 0)) { e.status = MP3B200_WAV_RANGE_ERROR; return e; }
  e.nsamples = ch == 1 ? view : ch == 0 ? 0 : dl / (2LL * ch);
  const unsigned tag = (unsigned)f[20] | ((unsigned)f[21] << 8), bits = (unsigned)f[34] | ((unsigned)f[35] << 8);
  if (tag != 1 || bits != 16) { e.status = MP3B200_WAV_NOT_PCM16; return e; }
  const Config* c = e.sample_rate > 0 ? encodable_config(ch, e.sample_rate, kbps, flags & MP3B200_RESAMPLE) : nullptr;
  if (!c) { e.status = MP3B200_WAV_UNSUPPORTED; return e; }
  e.status = MP3B200_WAV_ENCODED;
  e.out_samplerate = c->host.samplerate;
  e.out_bytes = bytes_of_frames(c->host, 0, frames_for(e.nsamples, c->host.mode_gr, c->rs.ratio));
  if (tagged && c->tag.fits) e.out_bytes += c->tag.frame_bytes;
  return e;
}

/* The argument rules of the WAV calls, the whole-stream calls' rules on their arrays, before any CUDA call */
int wav_args(int flags, int allowed, int nfiles, const uint8_t* const* files, const int64_t* file_len, bool encode,
             uint8_t* const* out, const int64_t* cap, const int64_t* out_bytes, const int32_t* status) {
  auto refuse = [](const char* why) { g_err = why; return MP3B200_ERR_HANDLE; };
  if (nfiles < 0) return refuse("negative stream count");
  if (flags & ~allowed) { g_err = "unknown flags"; return MP3B200_ERR_CONFIG; }
  if ((flags & MP3B200_REPLAYGAIN) && nfiles > MP3_MAX_LAUNCH_STREAMS) return refuse("ReplayGain batches hold at most 65535 streams");
  if (nfiles == 0) return MP3B200_OK;
  if (!files || !file_len || (encode && (!out || !cap || !out_bytes || !status))) return refuse("null array");
  for (int s = 0; s < nfiles; s++) {
    if (!files[s]) return refuse("null file");
    if (file_len[s] < 0) return refuse("negative file length");
  }
  return MP3B200_OK;
}

/* Uploads the data regions of the files `idx` (one configuration: cfg) as they are, one copy per file and upload slice on
 * t_ctx.up_st, and stages them as the rows whole_streams reads: file i's left row at rows + pcm_off[i], its right row behind
 * it.  Mono regions are copied straight into their rows; stereo regions land in a raw area behind the rows and k_stage_wav
 * splits each slice on the copy stream once it has landed, so arr.ready[j] means slice j's rows are there. */
int upload_wav_rows(const Config* cfg, const uint8_t* const* files, const std::vector<mp3b200_wav_plan_entry>& plan,
                    const std::vector<int>& idx, std::vector<int64_t>& pcm_off, int16_t*& rows, PcmArrival& arr, bool poison = false) {
  const int n = (int)idx.size(), nch = cfg->host.nch;
  pcm_off.assign((size_t)n, 0);
  std::vector<long long> raw_off((size_t)n, 0);
  long long tot = 0, raw = 0;
  for (int i = 0; i < n; i++) {
    const long long ns = plan[idx[i]].nsamples;
    pcm_off[i] = tot;
    tot += (ns * nch + 7) & ~7LL;                    /* rows 16-byte aligned: k_stage_wav's 8-byte left stores */
    if (nch == 2) { raw_off[i] = raw; raw += (4 * ns + 15) & ~15LL; }
  }
  const size_t rows_bytes = ((size_t)tot * 2 + 16 + 255) & ~(size_t)255, raw_bytes = ((size_t)raw + 255) & ~(size_t)255;
  const size_t desc_bytes = nch == 2 ? sizeof(WavStageDesc) * (size_t)n : 0;
  if (t_ctx.pcm.fit(rows_bytes + raw_bytes + desc_bytes)) return MP3B200_ERR_CUDA;
  rows = reinterpret_cast<int16_t*>(t_ctx.pcm.p);
  uint8_t* d_raw = t_ctx.pcm.p + rows_bytes;
  WavStageDesc* d_desc = reinterpret_cast<WavStageDesc*>(d_raw + raw_bytes);
  if (poison) CK(cudaMemsetAsync(rows, 0x7f, rows_bytes, t_ctx.up_st));   /* debug tap: rows of 0x7f7f until written */
  long long max_n = 0;
  if (nch == 2) {
    std::vector<WavStageDesc> d((size_t)n);
    for (int i = 0; i < n; i++) {
      d[i].x = d_raw + raw_off[i];
      d[i].y[0] = rows + pcm_off[i];
      d[i].y[1] = d[i].y[0] + plan[idx[i]].nsamples;
      d[i].n = plan[idx[i]].nsamples;
      max_n = d[i].n > max_n ? d[i].n : max_n;
    }
    const int rc = upload(t_ctx, d_desc, d.data(), desc_bytes, t_ctx.up_st);
    if (rc) return rc;
  }
  arr.chunks = upload_slices(n, tot);
  arr.ready = t_ctx.ready;
  for (int j = 0; j < arr.chunks; j++) {
    long long max_groups = 0;
    for (int i = 0; i < n; i++) {
      const mp3b200_wav_plan_entry& e = plan[idx[i]];
      const long long lo = e.nsamples * j / arr.chunks, hi = e.nsamples * (j + 1) / arr.chunks;
      if (hi <= lo) continue;
      const uint8_t* src = files[idx[i]] + e.data_offset;
      if (nch == 1) CK(cudaMemcpyAsync(rows + pcm_off[i] + lo, src + 2 * lo, 2 * (hi - lo), cudaMemcpyHostToDevice, t_ctx.up_st));
      else CK(cudaMemcpyAsync(d_raw + raw_off[i] + 4 * lo, src + 4 * lo, 4 * (hi - lo), cudaMemcpyHostToDevice, t_ctx.up_st));
      const long long groups = ((hi + 3) >> 2) - (lo >> 2);
      max_groups = groups > max_groups ? groups : max_groups;
    }
    for (int f0 = 0; nch == 2 && max_groups > 0 && f0 < n; f0 += MP3_MAX_LAUNCH_STREAMS) {
      const int nf = n - f0 < MP3_MAX_LAUNCH_STREAMS ? n - f0 : MP3_MAX_LAUNCH_STREAMS;
      dim3 grid((unsigned)((max_groups + WAV_STAGE_THREADS - 1) / WAV_STAGE_THREADS), (unsigned)nf);
      k_stage_wav<<<grid, WAV_STAGE_THREADS, 0, t_ctx.up_st>>>(d_desc + f0, j, arr.chunks);
      g_launches++;
      CK(cudaGetLastError());
    }
    CK(cudaEventRecord(t_ctx.ready[j], t_ctx.up_st));
  }
  return MP3B200_OK;
}

/* The body of mp3b200_encode_wav / _tagged: plan every file, then one whole-stream encode per (channels, sampleRate) on the
 * rows upload_wav_rows stages.  Output order is input order whatever the group order. */
int encode_wav(int kbps, int flags, bool tagged, int nfiles, const uint8_t* const* files, const int64_t* file_len,
               uint8_t* const* out, const int64_t* cap, int64_t* out_bytes, int32_t* status, double* title_db, double* album_db) {
  int rc = wav_args(flags, MP3B200_RESAMPLE | (tagged ? MP3B200_REPLAYGAIN : 0), nfiles, files, file_len, true, out, cap, out_bytes,
                    status);
  if (rc) return rc;
  std::vector<mp3b200_wav_plan_entry> plan((size_t)nfiles);
  std::map<std::pair<int, int>, std::vector<int>> groups;
  for (int s = 0; s < nfiles; s++) {
    plan[s] = wav_plan_file(kbps, flags, tagged, files[s], file_len[s]);
    if (plan[s].status == MP3B200_WAV_ENCODED) {
      if (cap[s] < plan[s].out_bytes) { g_err = "output buffer too small"; return MP3B200_ERR_BUFFER; }
      groups[{plan[s].channels, plan[s].sample_rate}].push_back(s);
    }
  }
  for (int s = 0; s < nfiles; s++) {
    status[s] = plan[s].status;
    out_bytes[s] = 0;
    if (title_db) title_db[s] = RG_NOT_ENOUGH_SAMPLES;
  }
  const bool analyse = tagged && (flags & MP3B200_REPLAYGAIN);
  std::vector<int> album(RG_HIST, 0), hist(RG_HIST);
  for (const auto& g : groups) {
    const std::vector<int>& idx = g.second;
    const int n = (int)idx.size();
    Config* cfg = nullptr;
    if ((rc = get_config(g.first.first, g.first.second, kbps, flags & MP3B200_RESAMPLE, &cfg))) return rc;
    std::vector<int64_t> pcm_off, ns((size_t)n), caps((size_t)n), nb((size_t)n);
    std::vector<uint8_t*> outs((size_t)n);
    std::vector<double> title((size_t)n);
    for (int i = 0; i < n; i++) { ns[i] = plan[idx[i]].nsamples; outs[i] = out[idx[i]]; caps[i] = cap[idx[i]]; }
    int16_t* rows = nullptr;
    PcmArrival arr;
    if ((rc = upload_wav_rows(cfg, files, plan, idx, pcm_off, rows, arr))) return rc;
    WholeCall<int16_t> k = {.channels = g.first.first, .samplerate = g.first.second, .kbps = kbps, .flags = flags, .nstreams = n,
                            .d_pcm = rows, .pcm_off = pcm_off.data(), .nsamples = ns.data(), .tagged = tagged, .analyse = analyse,
                            .out = outs.data(), .cap = caps.data(), .out_bytes = nb.data(), .title_db = title.data()};
    if ((rc = whole_sync_run(k, cfg, &arr, analyse ? hist.data() : nullptr))) return rc;
    for (int i = 0; i < n; i++) {
      out_bytes[idx[i]] = nb[i];
      if (title_db) title_db[idx[i]] = analyse ? title[i] : RG_NOT_ENOUGH_SAMPLES;
    }
    for (int b = 0; analyse && b < RG_HIST; b++) album[b] += hist[b];
  }
  if (album_db) *album_db = analyse ? rg_analyze_result(album.data()) : RG_NOT_ENOUGH_SAMPLES;
  return MP3B200_OK;
}
}  // namespace

extern "C" {

int mp3b200_wav_plan(int kbps, int flags, int nfiles, const uint8_t* const* files, const int64_t* file_len,
                     mp3b200_wav_plan_entry* plan) {
  const int rc = wav_args(flags, MP3B200_RESAMPLE | MP3B200_WAV_TAG, nfiles, files, file_len, false, nullptr, nullptr, nullptr, nullptr);
  if (rc) return rc;
  if (nfiles > 0 && !plan) { g_err = "null array"; return MP3B200_ERR_HANDLE; }
  for (int s = 0; s < nfiles; s++) plan[s] = wav_plan_file(kbps, flags, (flags & MP3B200_WAV_TAG) != 0, files[s], file_len[s]);
  return MP3B200_OK;
}

int mp3b200_encode_wav(int kbps, int flags, int nfiles, const uint8_t* const* files, const int64_t* file_len, uint8_t* const* out,
                       const int64_t* cap, int64_t* out_bytes, int32_t* status) {
  return encode_wav(kbps, flags, false, nfiles, files, file_len, out, cap, out_bytes, status, nullptr, nullptr);
}

int mp3b200_encode_wav_tagged(int kbps, int flags, int nfiles, const uint8_t* const* files, const int64_t* file_len,
                              uint8_t* const* out, const int64_t* cap, int64_t* out_bytes, int32_t* status, double* title_db,
                              double* album_db) {
  return encode_wav(kbps, flags, true, nfiles, files, file_len, out, cap, out_bytes, status, title_db, album_db);
}

int mp3b200_debug_stage_wav(int kbps, int flags, int nfiles, const uint8_t* const* files, const int64_t* file_len, int16_t* rows,
                            int64_t cap, int32_t* slices) {
  int rc = wav_args(flags, MP3B200_RESAMPLE, nfiles, files, file_len, false, nullptr, nullptr, nullptr, nullptr);
  if (rc || nfiles == 0) return rc;
  std::vector<mp3b200_wav_plan_entry> plan((size_t)nfiles);
  std::vector<int> idx((size_t)nfiles);
  long long tot = 0;
  for (int s = 0; s < nfiles; s++) {
    plan[s] = wav_plan_file(kbps, flags, false, files[s], file_len[s]);
    idx[s] = s;
    if (plan[s].status != MP3B200_WAV_ENCODED || plan[s].channels != plan[0].channels || plan[s].sample_rate != plan[0].sample_rate) {
      g_err = "the tap takes encodable files of one configuration"; return MP3B200_ERR_CONFIG;
    }
    tot += plan[s].nsamples * plan[s].channels;
  }
  if (!rows || cap < tot) { g_err = "output buffer too small"; return MP3B200_ERR_BUFFER; }
  Config* cfg = nullptr;
  if ((rc = get_config(plan[0].channels, plan[0].sample_rate, kbps, flags, &cfg))) return rc;
  std::vector<int64_t> pcm_off;
  int16_t* d_rows = nullptr;
  PcmArrival arr;
  if ((rc = upload_wav_rows(cfg, files, plan, idx, pcm_off, d_rows, arr, true))) return rc;
  CK(cudaStreamSynchronize(t_ctx.up_st));
  long long at = 0;
  for (int s = 0; s < nfiles; s++) {
    const size_t n = (size_t)(plan[s].nsamples * plan[s].channels);
    CK(cudaMemcpy(rows + at, d_rows + pcm_off[s], sizeof(int16_t) * n, cudaMemcpyDeviceToHost));
    at += (long long)n;
  }
  if (slices) *slices = arr.chunks;
  return MP3B200_OK;
}

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
  if (rc || (rc = crc_tables_on(dev)) || (rc = wait_legacy(t_ctx))) return rc;
  std::vector<long long> at(off, off + nranges), l(len, len + nranges);
  for (long long& a : at) a += (long long)(uintptr_t)d_buf;
  for (int run = 0; run < (ms ? 2 : 1); run++) {          /* with ms, a second run is timed */
    if (run) CK(cudaEventRecord(t_ctx.ev[0], t_ctx.st));
    if ((rc = queue_music_crc(t_ctx, at, l))) return rc;
    if (nranges > 0) CK(cudaMemcpyAsync(crc, t_ctx.crc.p, sizeof(uint32_t) * (size_t)nranges, cudaMemcpyDeviceToHost, t_ctx.st));
    if (run) CK(cudaEventRecord(t_ctx.ev[1], t_ctx.st));
    CK(cudaStreamSynchronize(t_ctx.st));
    CK(cudaGetLastError());
  }
  if (ms) CK(cudaEventElapsedTime(ms, t_ctx.ev[0], t_ctx.ev[1]));
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
  return mp3b200_lametag_size_ex(channels, samplerate, kbps, 0);
}

int mp3b200_lametag_size_ex(int channels, int samplerate, int kbps, int flags) {
  const Config* c = host_config(channels, samplerate, kbps, flags);
  if (!c) return MP3B200_ERR_CONFIG;
  return c->tag.fits ? c->tag.frame_bytes : 0;
}

int mp3b200_lametag_build(int channels, int samplerate, int kbps, int64_t nframes, int64_t music_bytes, int music_crc, int encoder_padding,
                          uint8_t* buf, int cap) {
  return build_lametag(channels, samplerate, kbps, 0, nframes, music_bytes, music_crc, encoder_padding, 0, buf, cap);
}

int mp3b200_lametag_build_ex(int channels, int samplerate, int kbps, int flags, int64_t nframes, int64_t music_bytes, int music_crc,
                             int encoder_padding, int radio_gain, uint8_t* buf, int cap) {
  return build_lametag(channels, samplerate, kbps, flags, nframes, music_bytes, music_crc, encoder_padding,
                       mp3_radio_gain_field(radio_gain), buf, cap);
}

}  // extern "C"

#include "mp3_session.inc"
#include "mp3_handle.inc"
#include "mp3_session_handles.inc"

#ifdef Q_TASKSTAT
extern "C" int mp3b200_debug_taskstat(int* out, int rows) {
  if (rows > (1 << 16)) rows = 1 << 16;
  return cudaMemcpyFromSymbol(out, g_taskstat, sizeof(int) * 8 * (size_t)rows) == cudaSuccess ? 0 : -1;
}
#endif

#ifdef PSY_PHASESTAT
extern "C" int mp3b200_debug_psystat(long long* out, int rows) {
  if (rows > PSY_STAT_ROWS) rows = PSY_STAT_ROWS;
  return cudaMemcpyFromSymbol(out, g_psystat, sizeof(long long) * PSY_STAT_COLS * (size_t)rows) == cudaSuccess ? rows : -1;
}
#endif

#ifdef MP3_DOMAIN_CHECK
/* the out-of-domain counters of every DomainSite (mp3_device.cuh) on the current device, cleared after reading; returns the
 * number of sites (out needs that many slots) */
extern "C" int mp3b200_debug_domain_hits(unsigned long long* out, int cap) {
  if (cap < DOM_NSITES) return DOM_NSITES;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(out, g_domain_hits, sizeof(unsigned long long) * DOM_NSITES) != cudaSuccess) return -1;
  static const unsigned long long zero[DOM_NSITES] = {};
  return cudaMemcpyToSymbol(g_domain_hits, zero, sizeof zero) == cudaSuccess ? DOM_NSITES : -1;
}
#endif
