/* mp3b200.h -- C ABI of the H100-native batch MP3 encoder (libmp3b200.so).
 *
 * Drop-in boundary for the lamejs `Mp3Encoder` hot path.  Each entry point names the reference
 * interface it replaces (paths relative to zhuker/lamejs @ 582bbba).  Plain pointers and sizes only;
 * no torch / CUDA types cross this boundary.  All work runs on the CUDA device selected with
 * mp3b200_set_device() (default: device 0); there is NO CPU fallback -- every call fails with
 * MP3B200_ERR_CUDA when no usable sm_90 device is present.
 *
 * Error codes mirror lamejs/LAME where one exists (src/js/Lame.js:1045-1061,1494; BitStream.js:916-919).
 */
#ifndef MP3B200_H
#define MP3B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MP3B200_OK 0
#define MP3B200_ERR_CONFIG (-1)   /* unsupported channels/samplerate/bitrate: lame_init_params returns -1 */
#define MP3B200_ERR_BUFFER (-1)   /* output buffer too small: copy_buffer returns -1 (BitStream.js:916-919) */
#define MP3B200_ERR_HANDLE (-3)   /* bad handle: lame_encode_buffer returns -3 (Lame.js:1494) */
#define MP3B200_ERR_CUDA (-100)   /* CUDA failure or no device (no reference equivalent) */

typedef struct mp3b200_encoder mp3b200_encoder;

/* Select the CUDA device used by subsequently created encoders / batch calls (one process per GPU). */
int mp3b200_set_device(int device);

/* Replaces `new lamejs.Mp3Encoder(channels, samplerate, kbps)` (src/js/index.js:66-115).
 * channels 1|2; samplerate 8000|11025|12000|16000|22050|24000 (MPEG-2 / 2.5 LSF: one granule, 576-sample frames) or
 * 32000|44100|48000 (MPEG-1); kbps snapped to the nearest legal rate of that MPEG version like FindNearestBitrate
 * (src/js/Lame.js:408-423).  Configurations for which lamejs would RESAMPLE (lame_init_params picks out_samplerate !=
 * in_samplerate from the bitrate's low-pass, Lame.js:285-364 -- e.g. 44.1 kHz stereo below 112 kbps) return
 * MP3B200_ERR_CONFIG here; mp3b200_create_ex with MP3B200_RESAMPLE accepts those whose rate ratio is an integer.
 * This call is mp3b200_create_ex with flags = 0. */
int mp3b200_create(int channels, int samplerate, int kbps, mp3b200_encoder** out);

/* ---- resampling (lamejs fill_buffer_resample, Lame.js:1719-1843) -------------------------------------------------------
 * MP3B200_RESAMPLE also accepts a configuration for which lamejs resamples, when its output rate divides the input rate
 * (lamejs's own test, |in / out - round(in / out)| < 1e-4): 48000 -> 24000, 44100 -> 22050, 48000 / 32000 -> 16000 and
 * 48000 / 32000 / 24000 / 16000 -> 8000, e.g. `new Mp3Encoder(2, 48000, 64)`, which encodes at 24 kHz.  The caller feeds
 * samples at the input rate; the GPU resamples them (k_resample: one 33-tap filter, bit-exact with lamejs) and encodes at the
 * output rate, byte-identical to lamejs however the input is split into calls.  Non-integer ratios return MP3B200_ERR_CONFIG
 * with or without the flag: lamejs reads its input with fractional typed-array indices there, so NaN samples enter its
 * stream and its bytes depend on the call sizes.  Without the flag nothing changes; with it, configurations that encode at
 * their input rate behave exactly as without it.
 * On a resampled handle every handle call works as documented, with sample counts in input samples (state blobs carry their
 * own magic and both rates and are refused by a handle of another rate pair), except mp3b200_seek, which returns -2.
 * The _ex entry points below take the flags; the others are the same calls with flags = 0. */
#define MP3B200_RESAMPLE 1
int mp3b200_create_ex(int channels, int samplerate, int kbps, int flags, mp3b200_encoder** out);
/* the output rate lamejs encodes a configuration at (Lame.js:285-364; != samplerate: it resamples), 0 for a channel count
 * other than 1 or 2.  Pure host code. */
int mp3b200_out_samplerate(int channels, int samplerate, int kbps);

/* Replaces `encodeBuffer(left, right)` (src/js/index.js:117-130 -> Lame.js:1490-1667).  `right` may be NULL
 * for mono.  Writes the bytes of the frames completed by this call (possibly 0) into `out` and returns their
 * count; lamejs sizes its buffer as trunc(1.25*n + 7200).  Buffers are borrowed for the call only. */
int mp3b200_encode(mp3b200_encoder* h, const int16_t* left, const int16_t* right, int nsamples, uint8_t* out, int cap);

/* Replaces `flush()` (src/js/index.js:132-135 -> Lame.js:1381-1488): encodes the buffered tail padded with
 * zeros; a second flush returns 0; the encoder stays usable. */
int mp3b200_flush(mp3b200_encoder* h, uint8_t* out, int cap);

/* Replaces garbage collection of the Mp3Encoder object. */
void mp3b200_destroy(mp3b200_encoder* h);

/* Batched encodeBuffer / flush over N live encoders of one configuration (SURVEY.md 8(b) "Batch"): equivalent to
 * calling mp3b200_encode / mp3b200_flush on every handle in turn, but the frames all handles complete in this call
 * are encoded by ONE pipeline launch (handle i = stream i).  left[i]/right[i]: nsamples[i] Int16 (right or right[i]
 * NULL: mono / duplicate left); out[i] receives out_bytes[i] bytes (cap[i] >= trunc(1.25 * nsamples[i] + 7200) like
 * lamejs, 0 = unchecked); out_bytes[i] < 0 reports a per-handle error (NULL handle -3, buffer too small -1, a handle of
 * another configuration than the batch's first one with frames to encode -1).  A handle whose call failed keeps its
 * samples and its completed frames: its next call hands them out first.
 * A handle may be listed more than once: the call then runs as consecutive rounds, round k taking the k-th occurrence of
 * every handle, so each handle's entries run in list order (a repeated flush returns 0 bytes, like a second flush); a
 * call without repeats is one round.
 * A JS caller loops over its encoders instead (worker-example/worker.js, worker-realtime.js:46). */
int mp3b200_encode_batch(mp3b200_encoder* const* handles, const int16_t* const* left, const int16_t* const* right,
                         const int* nsamples, uint8_t* const* out, const int* cap, int nstreams, int* out_bytes);
int mp3b200_flush_batch(mp3b200_encoder* const* handles, uint8_t* const* out, const int* cap, int nstreams, int* out_bytes);

/* Streaming handles fed from device memory: mp3b200_encode / mp3b200_encode_f32 / mp3b200_encode_batch /
 * mp3b200_encode_batch_f32 with the sample rows in device memory (a model producing audio on the GPU in chunks feeds them
 * without a copy to the host).  Everything else means exactly what it means there: bytes, error codes, repeated handles,
 * failed handles keeping their samples, Float32 mode, tags, ReplayGain, resampling; a handle may take host and device calls
 * in any mix, and its state blob does not tell them apart.  The output stays in host memory.
 * Every row (right rows of mono handles aside) must be device or managed memory on the handle's device
 * (cudaPointerGetAttributes); anything else returns MP3B200_ERR_HANDLE before any handle changes.  Float32 rows are
 * checked on the device before any handle changes, and refused with MP3B200_ERR_CONFIG like the host calls refuse them.
 * The call first waits for work already queued on the legacy default stream (where torch / plain CUDA callers produce the
 * rows), and has finished reading the rows when it returns: the caller may then overwrite or free them.
 * Without a device these calls return MP3B200_ERR_CUDA. */
int mp3b200_encode_device(mp3b200_encoder* h, const int16_t* d_left, const int16_t* d_right, int nsamples, uint8_t* out, int cap);
int mp3b200_encode_device_f32(mp3b200_encoder* h, const float* d_left, const float* d_right, int nsamples, uint8_t* out, int cap);
int mp3b200_encode_batch_device(mp3b200_encoder* const* handles, const int16_t* const* d_left, const int16_t* const* d_right,
                                const int* nsamples, uint8_t* const* out, const int* cap, int nstreams, int* out_bytes);
int mp3b200_encode_batch_device_f32(mp3b200_encoder* const* handles, const float* const* d_left, const float* const* d_right,
                                    const int* nsamples, uint8_t* const* out, const int* cap, int nstreams, int* out_bytes);
/* the CUDA device a handle was created on (the device of mp3b200_set_device at mp3b200_create), or MP3B200_ERR_HANDLE */
int mp3b200_encoder_device(const mp3b200_encoder* h);

/* ---- encoder state: checkpoint / resume, and one stream cut into segments (SURVEY.md 8(e)(2)) ----------------------------
 * lamejs keeps an Mp3Encoder's state in JS objects (gfc.*: ATH adjust, block-type FSM, OldValue / CurrentStep, the previous
 * granule's masking, mfbuf); a JS caller checkpoints by keeping the object alive.  Here the state is a blob:
 *   export_state  writes everything the handle carries between calls (scalars, the previous unit's masking row from device
 *                 memory, the PCM tail later frames still read, FIFO accounting); buf == NULL returns the size.  Two handles
 *                 that encoded the same frames from the same samples export identical bytes.
 *   import_state  makes a handle of the same configuration continue exactly where the exporting one stood.  A blob whose
 *                 retained samples do not start at max(0, framesize*frames_done - 1104) is refused (-1), and the handle is
 *                 left as it was.
 *   seek          positions a FRESH handle at frame `frame` >= 1 with the sequential state of a stream start: the start of
 *                 a warm-up.  A segment encoder seeks W frames before its first frame, encodes them (discarding the bytes)
 *                 and compares its state with the predecessor segment's exported end state: equal blobs prove its frames are
 *                 the ones a single encoder would produce; otherwise it imports the predecessor's state and encodes again
 *                 (lamejs_b200/sharding.py encode_stream_segments).  `hist`: the stream samples
 *                 [max(0, frame*framesize - 1104), frame*framesize + 224), framesize = 576 * granules per frame; feeding
 *                 continues with sample frame*framesize + 224.  Not supported on a resampled handle (returns -2).
 * Return MP3B200_OK / bytes written, or a negative error (wrong configuration -2, buffer -1, handle -3). */
int mp3b200_export_state(mp3b200_encoder* h, void* buf, int cap);
int mp3b200_import_state(mp3b200_encoder* h, const void* buf, int len);
int mp3b200_seek(mp3b200_encoder* h, int64_t frame, const int16_t* left_hist, const int16_t* right_hist, int nhist);

/* ---- batch extension (same semantics, many independent streams per launch sequence) -------------------
 * Equivalent to, for each stream s: e = new Mp3Encoder(ch, sr, kbps); bytes = e.encodeBuffer(L_s, R_s) ++
 * e.flush().  This is the throughput path (a JS caller would loop over encoders, worker-example/worker.js). */

/* Number of bytes / frames that stream of `nsamples` per channel produces (closed form: CBR, no reservoir). */
int64_t mp3b200_stream_bytes(int channels, int samplerate, int kbps, int64_t nsamples);
/* the same with flags (MP3B200_RESAMPLE: nsamples are input samples) */
int64_t mp3b200_stream_bytes_ex(int channels, int samplerate, int kbps, int flags, int64_t nsamples);
int64_t mp3b200_stream_frames(int64_t nsamples);                 /* MPEG-1 configurations (1152-sample frames) */
/* any accepted configuration (MPEG-2 / 2.5 frames carry 576 samples); -1 if the configuration is rejected */
int64_t mp3b200_stream_frames_cfg(int channels, int samplerate, int kbps, int64_t nsamples);
/* granules per frame: 2 (MPEG-1: 32 / 44.1 / 48 kHz) or 1 (MPEG-2 / 2.5: 8 .. 24 kHz); -1 if rejected */
int mp3b200_granules_per_frame(int channels, int samplerate, int kbps);
/* the same two with flags (MP3B200_RESAMPLE: nsamples are input samples; the frames and granules are those of the output
 * rate the configuration encodes at) */
int64_t mp3b200_stream_frames_ex(int channels, int samplerate, int kbps, int flags, int64_t nsamples);
int mp3b200_granules_per_frame_ex(int channels, int samplerate, int kbps, int flags);

/* Whole-stream calls.  Every call below that encodes, analyses or tags whole streams (encodeBuffer(everything) + flush()
 * on fresh encoders: mp3b200_encode_streams*, mp3b200_replaygain_streams*, mp3b200_finish_tags_device and the session calls
 * mp3b200_encode_streams*_async*) checks its arguments by one set of rules before it looks up the configuration and before
 * it touches the device, so the answer is the same on a machine without a GPU:
 *   - nstreams < 0 returns MP3B200_ERR_HANDLE ("negative stream count");
 *   - a flag the call does not take returns MP3B200_ERR_CONFIG ("unknown flags"): every call takes MP3B200_RESAMPLE, and
 *     only the tagged encodes take MP3B200_REPLAYGAIN (the ReplayGain-only calls imply it);
 *   - with the ReplayGain analysis, more than 65535 streams return MP3B200_ERR_HANDLE;
 *   - with nstreams > 0, each of these returns MP3B200_ERR_HANDLE: a NULL nsamples, a NULL row array (left, or d_pcm / d_files
 *     and their offsets pcm_off / file_off), a NULL left[s], a negative nsamples[s], or a NULL output array the call
 *     writes: out, cap and out_bytes of the host encodes, out_off of the device encodes, out_bytes of the device tagged
 *     encodes, file_bytes of mp3b200_finish_tags_device;
 *   - a session call also returns MP3B200_ERR_HANDLE for a NULL d_status, for a NULL out_bytes of a tagged call, and for a
 *     NULL d_gain with MP3B200_REPLAYGAIN, whatever nstreams.
 * A call with several bad arguments is refused for one of them; which one is not specified.  right, d_out, title_db,
 * album_db and timings_ms may be NULL.
 * Host buffers.  left[s]/right[s]: nsamples[s] Int16 each; right ignored for mono; with stereo input, right == NULL or
 * right[s] == NULL encodes left[s] on both channels.  out[s] receives
 * out_bytes[s] = mp3b200_stream_bytes(...) bytes (cap[s] must be >= that).  Returns 0 or a negative error; arguments as
 * for every whole-stream call (above). */
int mp3b200_encode_streams(int channels, int samplerate, int kbps, int nstreams, const int16_t* const* left,
                           const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                           const int64_t* cap, int64_t* out_bytes);
/* the same with flags (MP3B200_RESAMPLE: input samples in, out_bytes[s] = mp3b200_stream_bytes_ex(...)) */
int mp3b200_encode_streams_ex(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* const* left,
                              const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                              const int64_t* cap, int64_t* out_bytes);

/* Device-resident variant for benchmarking kernel throughput: d_pcm is ONE device allocation holding, per
 * stream s, nsamples[s] Int16 of the left channel at sample offset pcm_off[s] and (stereo) the right channel at
 * pcm_off[s] + nsamples[s].  d_out is a device buffer; stream s is written at out_off[s].  `timings_ms`
 * (optional, 16 floats) receives per-kernel CUDA-event times in ms: [0] psy analysis + loudness, [1] attack pre-pass + per-stream
 * scan with the subband analysis (polyphase filterbank) running beside it, [2] masking, [3] MDCT, [4] quantizer first pass (all of its kernels), [5] re-validation passes, [6] total, [7] number of
 * quantizer passes; first pass by kernel: [8] k_q_prepare, [9] k_q_search (gr0 + gr1), [10] k_q_outer (gr0 + gr1),
 * [11] k_q_finish (gr0 + gr1), [12] k_q_pack, [13] the re-validation folded into the first pass (verify + repaired
 * searches / rate loops of the few frames whose speculated start did not stand); [14..15] reserved (0).
 * More than 65535 streams run as consecutive launches of at most 65535 streams: the times are summed over them, [7] is the
 * largest pass count of any of them.  The passes after the first run on the device, as a CUDA graph with a conditional
 * WHILE node (DESIGN.md 5, 14): [7] is read from the device with the times, and a new launch shape costs one capture.
 * The call runs on a stream of its own that first waits for work already queued on the legacy default stream (where torch /
 * plain CUDA callers produced d_pcm) and returns after that stream has drained.  Arguments as for every whole-stream call
 * (above). */
int mp3b200_encode_streams_device(int channels, int samplerate, int kbps, int nstreams, const int16_t* d_pcm,
                                  const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                  const int64_t* out_off, float* timings_ms);
/* the same with flags.  With MP3B200_RESAMPLE, d_pcm / nsamples hold input samples, and timings_ms[14] receives the
 * resampler's time (k_resample; 0 for a configuration that encodes at its input rate).  [6] does not include it. */
int mp3b200_encode_streams_device_ex(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* d_pcm,
                                     const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                     const int64_t* out_off, float* timings_ms);

/* ---- container / metadata step after the path (SURVEY.md 8(f3)) ------------------------------------------------------
 * lamejs carries LAME's Xing / Info / LAME tag writer (src/js/VBRTag.js) and keeps its two inputs up to date on every
 * Mp3Encoder call -- gfc.nMusicCRC and VBR_seek_table.nBytesWritten (BitStream.js:924-935) -- but switches the writer off
 * (index.js:107: gfp.bWriteVbrTag = false).  Here the writer can be switched on.  Semantics are LAME's (VBRTag.java, which
 * VBRTag.js transliterates): with the tag on, the first bytes an encoder hands out are an all-zero frame of the stream's own
 * bitrate (InitVbrTag); after flush() mp3b200_get_lametag_frame returns the finished frame, which the caller writes over
 * that placeholder (lame_get_lametag_frame / putVbrTag).  The CRC-16 over all audio bytes is computed on the GPU
 * (k_music_crc, lamejs_b200/csrc/k_tag.cuh) from the bytes where the packer left them.
 *   set_write_vbr_tag   gfp.bWriteVbrTag, before the first sample.  Returns 1 (on), 0 (off: asked to, or InitVbrTag refused
 *                       because the frame cannot hold side info + 156 bytes, VBRTag.js:508-513), negative on error.
 *   get_lametag_frame   VBRTag.getLameTagFrame (VBRTag.js:829-923): 0 when the tag is off or no frame has been encoded;
 *                       the size needed when `cap` is too small (or buf NULL); else writes that many bytes and returns it.
 *   music_crc / bytes_written   gfc.nMusicCRC / nBytesWritten so far (-1 with the tag off: the accumulators are idle then).
 *   lametag_size        the tag frame's size for a configuration (0: does not fit; negative: rejected configuration).
 *   lametag_build       the same frame from numbers instead of a handle (pure host arithmetic, no device needed): for callers
 *                       that encode one stream in segments and combine counts and CRCs themselves.
 *   encode_streams_tagged   mp3b200_encode_streams with the tag on (same input rules and PCM upload): out[s] = finished
 *                       tag frame ++ audio frames (cap[s] >= mp3b200_stream_bytes + mp3b200_lametag_size); one k_music_crc
 *                       launch for the batch. */
int mp3b200_set_write_vbr_tag(mp3b200_encoder* h, int on);
int mp3b200_get_lametag_frame(mp3b200_encoder* h, uint8_t* buf, int cap);
int mp3b200_music_crc(mp3b200_encoder* h);
int64_t mp3b200_bytes_written(mp3b200_encoder* h);
int mp3b200_lametag_size(int channels, int samplerate, int kbps);
int mp3b200_lametag_size_ex(int channels, int samplerate, int kbps, int flags);   /* with flags: MP3B200_RESAMPLE handles */
int mp3b200_lametag_build(int channels, int samplerate, int kbps, int64_t nframes, int64_t music_bytes, int music_crc,
                          int encoder_padding, uint8_t* buf, int cap);
int mp3b200_encode_streams_tagged(int channels, int samplerate, int kbps, int nstreams, const int16_t* const* left,
                                  const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                                  const int64_t* cap, int64_t* out_bytes);

/* ---- ReplayGain (lamejs gfp.findReplayGain, GainAnalysis.js; LAME writes it by default) --------------------------------
 * With MP3B200_REPLAYGAIN, mp3b200_encode_streams_tagged_ex also runs lamejs's ReplayGain analysis on every stream, on the
 * GPU beside the encoder (lamejs_b200/csrc/k_replaygain.cuh), and fills the tag's Radio Replay Gain field as lamejs does
 * with findReplayGain on and decode_on_the_fly off: the analysis sees what lamejs puts into mfbuf (the scaled input, or the
 * resampler's output), in the pieces lamejs analyses it in, flush zeros included, and every sum and histogram bin equals
 * lamejs's.  title_db[s] (optional) receives GetTitleGain of stream s in dB, album_db (optional) GetAlbumGain over the batch
 * (analyzeResult of the summed histograms); -24601 (GAIN_NOT_ENOUGH_SAMPLES) when a stream holds less than one RMS window
 * (the tag then carries -51.0 dB, the clamp) or when the tag does not fit the frame (lamejs analyses only with the tag on;
 * the streams are then written without either).  The peak amplitude field stays 0: lamejs finds it only by decoding.
 * Flags MP3B200_RESAMPLE and MP3B200_REPLAYGAIN may be combined; flags = 0 is mp3b200_encode_streams_tagged.  A batch with
 * MP3B200_REPLAYGAIN holds at most 65535 streams.  Arguments as for every whole-stream call (above).
 * Streaming handles:
 *   set_find_replay_gain  gfp.findReplayGain, before the first sample and after mp3b200_set_write_vbr_tag (which switches it
 *                         off again).  Returns 1 (on), 0 (off: asked to, or the tag is off: lamejs analyses only with the tag
 *                         on, Lame.js:911-916), negative on error.  Every sample a call feeds, flush zeros included, is analysed
 *                         in the pieces lamejs analyses it in; each flush ends a title (GetTitleGain in flush_bitstream) and a
 *                         handle that goes on after a flush starts a new one.  The tag frame carries the last title's gain.
 *   get_replay_gain       after a flush: 1 and the last title's gain in dB (-24601: less than one RMS window) and gfc.RadioGain;
 *                         0 before the first flush or with the analysis off.
 *   album_gain            GetAlbumGain over the titles the handles ended (analyzeResult of their summed B histograms).
 * mp3b200_export_state, mp3b200_import_state and mp3b200_seek return -2 on a handle that analyses ReplayGain: a state blob
 * does not carry the analysis. */
#define MP3B200_REPLAYGAIN 2
int mp3b200_encode_streams_tagged_ex(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* const* left,
                                     const int16_t* const* right, const int64_t* nsamples, uint8_t* const* out,
                                     const int64_t* cap, int64_t* out_bytes, double* title_db, double* album_db);
/* Tagged whole streams on device buffers: mp3b200_encode_streams_tagged_ex for PCM that is already on the GPU, written as
 * finished files into a device buffer.  The output is byte-identical to what mp3b200_encode_streams_tagged_ex (or _f32)
 * returns for the same samples, and title_db / album_db (optional) receive the same gains.
 *   d_pcm, pcm_off, nsamples   as for mp3b200_encode_streams_device_ex: one device allocation, per stream s nsamples[s]
 *                              samples of the left channel at pcm_off[s] and (stereo) the right channel behind them.
 *   flags                      MP3B200_RESAMPLE | MP3B200_REPLAYGAIN, meaning what they mean for _tagged_ex; any other bit
 *                              returns MP3B200_ERR_CONFIG.
 *   d_out, out_off             stream s is written as one file at d_out + out_off[s]: its tag frame, then its audio frames.
 *                              A stream gets a tag frame where _tagged_ex writes one: the tag fits the configuration
 *                              (mp3b200_lametag_size_ex > 0) and the stream has at least one frame (every stream has: flush()
 *                              always encodes one).  The room stream s needs is mp3b200_stream_bytes_ex + mp3b200_lametag_size_ex
 *                              for such a stream, mp3b200_stream_bytes_ex otherwise.  Nothing outside
 *                              [out_off[s], out_off[s] + out_bytes[s]) is written.
 *   out_bytes                  host array: out_bytes[s] receives the length of stream s's file.
 *   title_db, album_db         as for _tagged_ex, including -24601 when a stream holds less than one RMS window, or when the
 *                              tag does not fit and nothing is analysed.
 * A batch with MP3B200_REPLAYGAIN holds at most 65535 streams (MP3B200_ERR_HANDLE, as for _tagged_ex); without it larger
 * batches run as consecutive launches, as mp3b200_encode_streams_device does.  The call runs on a stream of its own that
 * first waits for work already queued on the legacy default stream (where torch / plain CUDA callers produced d_pcm and
 * d_out) and returns after that stream has drained.  The packer writes each stream's audio straight behind the room of its
 * tag frame; the frames are finished on the device (music CRC, Radio Replay Gain field, the tag's own CRC) by one kernel
 * (k_tag_finish), as the session's tagged calls finish them.
 * _device_f32 takes Float32 samples, laid out the same way, as mp3b200_encode_streams_device_f32 does; a sample that is not
 * finite, or beyond 2^40 once scaled, returns MP3B200_ERR_CONFIG, and no tag frame is placed (the audio bytes in d_out are
 * then unspecified). */
int mp3b200_encode_streams_tagged_device(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* d_pcm,
                                         const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out, const int64_t* out_off,
                                         int64_t* out_bytes, double* title_db, double* album_db);
int mp3b200_encode_streams_tagged_device_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* d_pcm,
                                             const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out, const int64_t* out_off,
                                             int64_t* out_bytes, double* title_db, double* album_db);
/* mp3b200_lametag_build with flags (MP3B200_RESAMPLE) and the Radio Replay Gain field of an analysed stream: radio_gain is
 * gfc.RadioGain = floor(title_db * 10 + 0.5), clamped to +-51.0 dB like lamejs; for segment callers that analyse the whole
 * stream themselves (ReplayGain is not combined across segments).  mp3b200_replaygain_streams below is that analysis, and
 * mp3b200_finish_tags_device the whole tag step on the joined audio in device memory. */
int mp3b200_set_find_replay_gain(mp3b200_encoder* h, int on);
int mp3b200_get_replay_gain(mp3b200_encoder* h, double* title_db, int* radio_gain);
int mp3b200_album_gain(mp3b200_encoder* const* handles, int n, double* album_db);
int mp3b200_lametag_build_ex(int channels, int samplerate, int kbps, int flags, int64_t nframes, int64_t music_bytes, int music_crc,
                             int encoder_padding, int radio_gain, uint8_t* buf, int cap);
/* ReplayGain of whole streams without the encoder: the analysis lamejs runs for a fresh Mp3Encoder with findReplayGain fed
 * encodeBuffer(whole stream) and then flush() -- the same pieces, the flush zeros, and under MP3B200_RESAMPLE the
 * resampler's output -- and nothing else: no encoder kernel runs.  For segment callers, which encode one stream in pieces
 * (lamejs_b200/sharding.py) and analyse it once beside them.
 *   left, right, nsamples      as for mp3b200_encode_streams_ex / _f32 (Int16 rows, or Float32 rows rounded and scaled as
 *                              lamejs's Float32Array store does; a sample that is not finite, or beyond 2^40 once scaled,
 *                              returns MP3B200_ERR_CONFIG).  Stereo with right == NULL or right[s] == NULL takes left[s].
 *   _device / _device_f32      rows laid out as mp3b200_encode_streams_device_ex reads them: stream s at d_pcm + pcm_off[s],
 *                              the right channel behind the left.  The call waits for work queued on the legacy default
 *                              stream and returns after its own stream has drained, as mp3b200_encode_streams_tagged_device.
 *   flags                      0 or MP3B200_RESAMPLE; any other bit returns MP3B200_ERR_CONFIG.
 *   title_db, album_db         (optional) GetTitleGain of each stream in dB and GetAlbumGain of the batch, -24601 for less
 *                              than one RMS window.  Bit-identical to what mp3b200_encode_streams_tagged_ex with
 *                              MP3B200_REPLAYGAIN returns for the same rows wherever the tag fits the configuration.  Where it
 *                              does not (mp3b200_lametag_size_ex == 0) that call analyses nothing and returns -24601; these
 *                              calls still analyse.
 * Arguments as for every whole-stream call (above): at most 65535 streams per call. */
int mp3b200_replaygain_streams(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* const* left,
                               const int16_t* const* right, const int64_t* nsamples, double* title_db, double* album_db);
int mp3b200_replaygain_streams_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* const* left,
                                   const float* const* right, const int64_t* nsamples, double* title_db, double* album_db);
int mp3b200_replaygain_streams_device(int channels, int samplerate, int kbps, int flags, int nstreams, const int16_t* d_pcm,
                                      const int64_t* pcm_off, const int64_t* nsamples, double* title_db, double* album_db);
int mp3b200_replaygain_streams_device_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* d_pcm,
                                          const int64_t* pcm_off, const int64_t* nsamples, double* title_db, double* album_db);
/* The tag step of mp3b200_encode_streams_tagged_device on audio already in device memory: turns the untagged audio of whole
 * streams (one stream encoded in segments and joined, say) into finished files.
 *   d_files, file_off, nsamples   file s lies at d_files + file_off[s]: mp3b200_lametag_size_ex bytes of room, then the
 *                              mp3b200_stream_bytes_ex(..., nsamples[s]) audio bytes of encodeBuffer(nsamples[s] samples) +
 *                              flush() on a fresh encoder.  The tag frame is written into the room: music CRC of the audio
 *                              (k_music_crc), frame / byte counts, seek table and encoder padding from nsamples[s].
 *   title_db                   host array (may be NULL): the Radio Replay Gain field of file s from title_db[s], rounded and
 *                              clamped to +-51.0 dB as lamejs does; NULL writes the field as 0 (nothing analysed).
 *   file_bytes                 host array: file_bytes[s] receives the file's length.
 *   flags                      0 or MP3B200_RESAMPLE.
 * Where the tag does not fit the configuration there is no room and nothing is written; nothing outside
 * [file_off[s], file_off[s] + file_bytes[s]) is ever written.  The files are byte-identical to what
 * mp3b200_encode_streams_tagged_device writes for the same samples: with MP3B200_REPLAYGAIN when title_db comes from
 * mp3b200_replaygain_streams, without it when title_db is NULL.  Ordering as mp3b200_replaygain_streams_device; arguments
 * as for every whole-stream call (above). */
int mp3b200_finish_tags_device(int channels, int samplerate, int kbps, int flags, int nstreams, uint8_t* d_files,
                               const int64_t* file_off, const int64_t* nsamples, const double* title_db, int64_t* file_bytes);
/* Test tap: one whole stream through mp3b200_encode_streams_tagged_ex with MP3B200_REPLAYGAIN (flags: MP3B200_RESAMPLE).
 * win_sums [w][2] = lsum, rsum of RMS window w (bit-exact), win_idx[w] its histogram index, for w < nwin_cap; hist (12000
 * bins), title_db; stats[0] windows, [1] repair passes, [2] chunks run again, [3] the analysis time in ms (a float's bits).
 * Any output pointer may be NULL. */
int mp3b200_debug_replaygain(int channels, int samplerate, int kbps, int flags, const int16_t* left, const int16_t* right,
                             int64_t nsamples, double* win_sums, int32_t* win_idx, int64_t nwin_cap, int32_t* hist,
                             double* title_db, int32_t* stats);

/* The rest of VBRTag.js's surface:
 *   put_vbr_tag     putVbrTag (VBRTag.js:937-965) on a stream held in memory: writes the finished frame over the placeholder,
 *                   behind an ID3v2 tag if the stream starts with one (skipId3v2; the port's inverted test is not reproduced).
 *                   0 ok / nothing to write, -1 like the reference (no frame counted yet, empty or too short stream).
 *   get_vbr_tag     getVbrTag (VBRTag.js:375-470): the reader side -- frame / byte counts, seek table, quality, encoder delay
 *                   and padding from the first frame of any Xing / Info tagged stream.  1 ok, 0 no tag (reference: null), -2
 *                   buffer too short.  Pure host code.
 *   crc16_combine   CRC-16 of A || B from crc(A), crc(B) and |B| (the rule k_music_crc and the handles use): lets callers that
 *                   encode one stream as segments on several GPUs (INTEGRATION.md) put one tag on the joined stream. */
typedef struct mp3b200_vbr_tag_data {
  int32_t h_id, samprate, flags, frames, bytes, vbr_scale, headersize, enc_delay, enc_padding;
  uint8_t toc[100];
} mp3b200_vbr_tag_data;
int mp3b200_put_vbr_tag(mp3b200_encoder* h, uint8_t* stream, int64_t len);
int mp3b200_get_vbr_tag(const uint8_t* frame, int64_t len, mp3b200_vbr_tag_data* out);
int mp3b200_crc16_combine(int crc_a, int crc_b, int64_t len_b);

/* ID3 tags (SURVEY.md 8(f3)).  lamejs carries only a stub (index.js:56-64) and switches the automatic tags off (index.js:109);
 * the writer is the Java original's, src/main/java/mp3/ID3Tag.java: lame_get_id3v2_tag :961-1102 (ID3v2.3, ISO-8859-1 text
 * frames TSSE TIT2 TPE1 TALB TYER COMM TRCK TCON TLEN, optional padding), lame_get_id3v1_tag :1141-1189 (128 bytes, v1.1 when a
 * track is set).  Fields are Latin-1 strings, NULL or "" = not set (the id3tag_set_* calls, applied in the order of the struct);
 * `genre` is a number 0..147 or a name of ID3Tag.java:56-89.  Both return the tag size written, the size needed when `cap` is
 * smaller, 0 when the reference writes no such tag (v2: nothing asks for it and every field fits version 1; v1: nothing set, or
 * V2_ONLY), negative for a malformed year / track / genre.  The version 2 tag goes in front of the stream (and of the Info / LAME
 * tag frame), the version 1 tag behind it.  Pure host code. */
#define MP3B200_ID3_ADD_V2 2     /* id3tag_add_v2 */
#define MP3B200_ID3_V1_ONLY 4    /* id3tag_v1_only */
#define MP3B200_ID3_V2_ONLY 8    /* id3tag_v2_only */
#define MP3B200_ID3_SPACE_V1 16  /* id3tag_space_v1: pad version 1 fields with spaces */
#define MP3B200_ID3_PAD_V2 32    /* id3tag_set_pad(padding), 128 bytes if padding <= 0 */
typedef struct mp3b200_id3tag {
  const char *title, *artist, *album, *year, *comment, *track, *genre;
  int flags, padding;
  int64_t num_samples;           /* gfp.num_samples for the TLEN frame; -1 = unknown (no TLEN) */
  int samplerate;
} mp3b200_id3tag;
int mp3b200_id3v2_tag(const mp3b200_id3tag* t, uint8_t* buf, int cap);
int mp3b200_id3v1_tag(const mp3b200_id3tag* t, uint8_t* buf, int cap);
const char* mp3b200_id3_genre_name(int index);

/* Test / bench tap of k_music_crc: CRC-16 (VBRTag.js:547-556, start 0) of the ranges [off[i], off[i] + len[i]) of a DEVICE
 * buffer; `ms` (optional) receives the CUDA-event time of one launch sequence incl. its 4-byte-per-range read-back. */
int mp3b200_debug_music_crc(const uint8_t* d_buf, const int64_t* off, const int64_t* len, int nranges, uint32_t* crc, float* ms);

/* Replaces `lamejs.WavHeader.readHeader(dataView)` (src/js/index.js:154-193): the RIFF/WAVE front-end lamejs ships for its
 * examples.  Returns 1 and fills `out`; 0 where the reference returns undefined (not RIFF / not WAVE / "fmt " not first);
 * -1 where it throws 'extended fmt chunk not implemented' (fmt length other than 16 or 18); -2 where its DataView read runs
 * past the buffer (RangeError).  Pure host code, no device needed.  PCM starts at data + data_offset. */
typedef struct mp3b200_wav_header { int64_t data_offset, data_len; int32_t channels; uint32_t sample_rate; } mp3b200_wav_header;
int mp3b200_wav_read_header(const uint8_t* data, int64_t len, mp3b200_wav_header* out);

/* ---- WAV files in, MP3 files out (DESIGN.md 18) ---------------------------------------------------------------------------
 * A batch of whole WAV files encoded as lamejs's worker-example/worker.js encodes one, but with the whole file in one call:
 *   w = WavHeader.readHeader(f); v = new Int16Array(f.buffer, w.dataOffset, w.dataLen / 2);
 *   stereo: left[i] = v[2 i], right[i] = v[2 i + 1] for i < dataLen / 4 (new Int16Array(dataLen / (2 channels)));
 *   e = new Mp3Encoder(w.channels, w.sampleRate, kbps); file = e.encodeBuffer(left, right) ++ e.flush().
 * (worker.js feeds 1152-sample calls and drops the last n mod 1152 samples: that is its loop, not the encoder's; every
 * sample is encoded here.)  Typed-array lengths truncate: the view holds floor(dataLen / 2) samples, a channel
 * floor(dataLen / 2) (mono) or floor(dataLen / 4) (stereo).  Each file gets a status; the first that applies:
 *   MP3B200_WAV_NOT_WAV         readHeader returns undefined (not RIFF / not WAVE / "fmt " not first)
 *   MP3B200_WAV_EXTENDED_FMT    readHeader throws 'extended fmt chunk not implemented' (fmt length other than 16 or 18)
 *   MP3B200_WAV_RANGE_ERROR     a RangeError: the header runs past the end of the file, or the view does (odd dataOffset, or
 *                               dataOffset + 2 floor(dataLen / 2) > length: truncated files, streaming WAVs whose dataLen is
 *                               0xFFFFFFFF), or new Int16Array(dataLen / 0) of a file with 0 channels and data
 *   MP3B200_WAV_NOT_PCM16       the fmt chunk's format tag is not 1 (PCM) or its bits per sample not 16.  A deliberate
 *                               deviation: lamejs never reads these fields and encodes such data as Int16 noise
 *   MP3B200_WAV_UNSUPPORTED     a configuration mp3b200_create_ex(channels, sampleRate, kbps, flags & MP3B200_RESAMPLE)
 *                               refuses (channels other than 1 or 2, a rate lamejs resamples without MP3B200_RESAMPLE, a
 *                               non-integer ratio)
 *   MP3B200_WAV_ENCODED         encoded.
 * A file that is not encoded changes nothing about the bytes, status or gains of the others. */
#define MP3B200_WAV_ENCODED 0
#define MP3B200_WAV_NOT_WAV 1
#define MP3B200_WAV_EXTENDED_FMT 2
#define MP3B200_WAV_RANGE_ERROR 3
#define MP3B200_WAV_NOT_PCM16 4
#define MP3B200_WAV_UNSUPPORTED 5
/* mp3b200_wav_plan only: size the files as mp3b200_encode_wav_tagged writes them (its tag frame included) */
#define MP3B200_WAV_TAG 4
typedef struct mp3b200_wav_plan_entry {
  int32_t status;               /* MP3B200_WAV_* */
  int32_t channels;             /* from the header (0 where readHeader gave none) */
  int32_t sample_rate;          /* the header's rate (values above 2^31 - 1 read as -1) */
  int32_t out_samplerate;       /* the rate the file is encoded at (!= sample_rate: resampled); 0 unless encoded */
  int64_t data_offset;          /* where the PCM starts in the file (0 where readHeader gave none) */
  int64_t nsamples;             /* samples per channel once the view and the split have succeeded, else 0 */
  int64_t out_bytes;            /* the exact size of the MP3 file: mp3b200_stream_bytes_ex, + mp3b200_lametag_size_ex with
                                   MP3B200_WAV_TAG; 0 unless encoded */
} mp3b200_wav_plan_entry;
/* files[s]: file_len[s] bytes of file s.  flags within MP3B200_RESAMPLE | MP3B200_WAV_TAG.  Fills plan[s] for every file
 * and returns 0.  Pure host arithmetic: the same answer without a device. */
int mp3b200_wav_plan(int kbps, int flags, int nfiles, const uint8_t* const* files, const int64_t* file_len,
                     mp3b200_wav_plan_entry* plan);
/* Encodes the files whose status is MP3B200_WAV_ENCODED: out[s] receives out_bytes[s] bytes (cap[s] >= plan out_bytes;
 * a smaller cap for a file that is encoded returns MP3B200_ERR_BUFFER before anything runs), status[s] the file's status
 * (out_bytes[s] = 0 for a file that is not encoded).  flags within MP3B200_RESAMPLE.  The bytes of every file are those
 * mp3b200_encode_streams_ex returns for its channels.  The data regions are copied to the GPU as they are, one copy per file
 * (per upload slice of large batches), and de-interleaved there (k_stage_wav); the files of each (channels, sampleRate)
 * run as one whole-stream encode, one configuration after another.
 * Arguments as for every whole-stream call (above), checked before any CUDA call: nfiles < 0, a NULL files / file_len /
 * out / cap / out_bytes / status array (nfiles > 0), a NULL files[s] or a negative file_len[s] return MP3B200_ERR_HANDLE; an
 * unknown flag MP3B200_ERR_CONFIG; with MP3B200_REPLAYGAIN, more than 65535 files MP3B200_ERR_HANDLE.  A bad file is
 * reported in status[s], never by failing the call. */
int mp3b200_encode_wav(int kbps, int flags, int nfiles, const uint8_t* const* files, const int64_t* file_len, uint8_t* const* out,
                       const int64_t* cap, int64_t* out_bytes, int32_t* status);
/* The same with the Info / LAME tag: every encoded file is what mp3b200_encode_streams_tagged_ex returns for it.  flags within
 * MP3B200_RESAMPLE | MP3B200_REPLAYGAIN.  title_db[s] (optional) is that call's title gain of file s (-24601 for a file not
 * encoded); album_db (optional) GetAlbumGain over the summed histograms of every file analysed in the call, whatever their
 * configurations (the rule of mp3b200_album_gain). */
int mp3b200_encode_wav_tagged(int kbps, int flags, int nfiles, const uint8_t* const* files, const int64_t* file_len,
                              uint8_t* const* out, const int64_t* cap, int64_t* out_bytes, int32_t* status, double* title_db,
                              double* album_db);
/* Test tap of k_stage_wav: stages the files (encodable, all of one configuration; flags within MP3B200_RESAMPLE) as
 * mp3b200_encode_wav does, on rows filled with 0x7f bytes first, and copies the staged rows back: file after file, its left
 * row, then (stereo) its right row.  slices (optional) receives the number of upload slices used. */
int mp3b200_debug_stage_wav(int kbps, int flags, int nfiles, const uint8_t* const* files, const int64_t* file_len, int16_t* rows,
                            int64_t cap, int32_t* slices);

/* ---- stage taps for parity tests (one stream, whole-stream semantics) -----------------------------------
 * Run the pipeline for one stream given host PCM and copy intermediate results back.  Any output pointer may be
 * NULL.  Shapes ([F] = mp3b200_stream_frames(n)):
 *   xr          float [F][2 gr][nch][576]   MDCT spectrum (NewMDCT.js mdct_sub48 output)
 *   blocktype   int32 [F][2][nch]           final block type per granule (PsyModel.js block_type_set)
 *   en_l/thm_l  float [F][2][nch][22], en_s/thm_s float [F][2][nch][13][3]   masking handed to the quantizer
 *   ath_adjust  double[F]                   ATH.adjust after adjust_ATH (Encoder.js:166-243)
 *   l3_enc      int32 [F][2][nch][576], ginfo int32 [F][2][nch][16] (global_gain, part2_3_length, part2_length,
 *               big_values, count1, scalefac_compress, table_select[3], region0, region1, preflag, scalefac_scale,
 *               count1table, block_type, reserved)
 * If `force_blocktype` is non-NULL (int32 [F][2][nch]) it overrides the psy model's block decision for the
 * filterbank stage (used to test the MDCT in isolation). */
int mp3b200_debug_stages(int channels, int samplerate, int kbps, const int16_t* left, const int16_t* right,
                         int64_t nsamples, const int32_t* force_blocktype, float* xr, int32_t* blocktype,
                         float* en_l, float* thm_l, float* en_s, float* thm_s, double* ath_adjust,
                         int32_t* l3_enc, int32_t* ginfo, uint8_t* bytes_out, int64_t bytes_cap);

/* The same taps, and the quantizer's state, through one struct (mp3b200_debug_stages is a thin wrapper of it).  `size` must
 * be sizeof(mp3b200_debug_taps): a caller built against an older, shorter struct (before `flags`) is refused with
 * MP3B200_ERR_HANDLE.  Inputs and the first outputs are those of mp3b200_debug_stages; in addition ([G] granules per frame):
 *   scalefac       int32 [F][G][nch][39]  final scalefactors; gr1 bands that scfsi shares with gr0 hold -1 (as in lamejs)
 *   subblock_gain  int32 [F][G][nch][3]
 *   xmin           float [F][G][nch][39]  calc_xmin's output as the rate loop receives it: the psymax bands (21 long, 36 short),
 *                                         0 above them and for granules without energy (where lamejs skips the rate loop)
 *   max_nonzero_coeff int32 [F][G][nch], xrpow_max double [F][G][nch]   after init_xrpow / calc_xmin, before the rate loop
 *   scfsi          int32 [F][nch][4]
 *   old_value, cur_step  int32 [F][3][nch]: gfc.OldValue / CurrentStep at the frame's start [0], after gr0 [1] (MPEG-1; 0 for
 *                  LSF) and after the frame [2], read from the speculation bookkeeping once the fixed-point loop has ended.
 *                  These are the states the final bytes were encoded from: the last verification found every frame's start
 *                  state equal to its predecessor's end state, and a search result kept from an earlier, speculated start
 *                  was kept only because the search from this start landed on the same gain and granule info.
 * `flags` selects the configuration like the _ex entry points (mp3b200_debug_stages: 0).  With MP3B200_RESAMPLE a
 * configuration lamejs resamples is tapped after k_resample: left / right / nsamples are input samples, and every shape above
 * is that of the output rate ([F] = mp3b200_stream_frames_ex(..., flags, nsamples), [G] = mp3b200_granules_per_frame_ex).
 * Any output pointer may be NULL.
 * The encoder computes the short-block half of the psy model (en_s / thm_s) only for the units whose masking a short
 * granule reads, and for each stream's last unit (DESIGN.md 2); the taps compute it for every unit. */
typedef struct mp3b200_debug_taps {
  int32_t size, channels, samplerate, kbps;
  const int16_t *left, *right;
  int64_t nsamples;
  const int32_t* force_blocktype;
  float* xr; int32_t* blocktype; float *en_l, *thm_l, *en_s, *thm_s; double* ath_adjust;
  int32_t *l3_enc, *ginfo; uint8_t* bytes_out; int64_t bytes_cap;
  int32_t *scalefac, *subblock_gain; float* xmin; int32_t* max_nonzero_coeff; double* xrpow_max;
  int32_t *scfsi, *old_value, *cur_step;
  int32_t flags;
} mp3b200_debug_taps;
int mp3b200_debug_stages_ex(const mp3b200_debug_taps* t);
/* Debug psy-row capture, off by default.  on != 0 clears the records and turns capture on for every thread and session;
 * 0 turns it off (the records stay until taken).  While it is on, each pipeline launch fills its front-end rows with a
 * poison pattern before the long-block analysis (float and double fields a quiet NaN, mask_idx 8, attack 0, both block-type
 * rows 1 = START), synchronises its stream after the attack pre-pass, after the short-block analysis and after the MDCT, and
 * records the rows there; a launch inside CUDA stream capture fails with MP3B200_ERR_CUDA.  Launches are numbered from 0 in
 * the order they start.  Each record is an int32[8] header and its payload:
 *   {1, launch, stream, frame0, nframes, nch, G, row_bytes}: the stream's long rows u = -1 .. G nframes - 1, nch per unit
 *     (eb_l float[64], peaks float[9], loudness float, mask_idx uint8[64], attack uint8[4], one pad byte; row_bytes each)
 *   {2, launch, count, nch, G, k_psy_analysis launches, 0, row_bytes}: the short list, count int32 pairs (stream,
 *     ((u + 1) << 1) | channel) in list order, then each entry's short row (ecb_s double[3][64], eb_s float[3][64])
 *   {3, launch, stream, frame0, nframes, nch, G, row_bytes}: the stream's rows after the MDCT, with n = G nframes:
 *     ATH.adjust seen by the psy calls of each frame (double[nframes]), the adjustment the quantizer uses (double[nframes]),
 *     the masking rows u = -1 .. n - 1, nch per unit (en_l float[22], thm_l float[22], en_s float[13][3],
 *     thm_s float[13][3]; row_bytes each; row u is what granule u + 1 uses), xr float[n][nch][576], the final block type
 *     int8[n][2] and the block type the psy call of the unit saw before it (int8[n][2]; both hold 2 per unit whatever nch),
 *     then zero bytes up to a multiple of 8 */
int mp3b200_debug_psy_capture(int on);
/* Copies the records held (bytes) to buf and clears them when cap is large enough; returns their size either way. */
int64_t mp3b200_debug_psy_take(void* buf, int64_t cap);

/* Test tap of k_resample: y[c * ny + m], m < ny, = output m of channel c (nch rows) of the resampler of a configuration that
 * MP3B200_RESAMPLE accepts with resampling, for the input left / right (nsamples each; right NULL: left) extended with zeros
 * on both sides.  MP3B200_ERR_CONFIG for a configuration that does not resample. */
int mp3b200_debug_resample(int channels, int samplerate, int kbps, const int16_t* left, const int16_t* right, int64_t nsamples,
                           float* y, int64_t ny);

/* ---- Float32 input (lamejs encodeBuffer with a Float32Array or a plain Array, Lame.js:1500-1510,1554-1560) -------------
 * lamejs stores every value the caller passes into a Float32Array, x = Float32(v), and scales it in place,
 * x = Float32((double)x * scale), when the preset's scale is not 1; the encoder works on those values.  The _f32 twins below
 * take such Float32 samples (a caller with doubles rounds them to Float32 once, as that store does) and encode them exactly
 * as lamejs does; an integer-valued sample in Int16 range encodes exactly like that Int16 sample through the Int16 calls.
 * Samples that are not finite (before or after the scale) are refused with MP3B200_ERR_CONFIG: the host calls refuse them
 * before anything runs and leave a handle untouched; mp3b200_encode_streams_device_f32 finds them on the device, and its
 * output buffer is then unspecified.  lamejs would carry NaN through its psy model and rate loop.
 * Samples beyond 2^40 (2^25 x full scale) once scaled are refused the same way: the library is compared with lamejs up to
 * there (DESIGN.md 12).  Below that, a frame whose bits do not fit its slot even at
 * global_gain 255 (from about 2e5 x full scale, depending on signal and bitrate) is refused with MP3B200_ERR_CONFIG by the
 * call that encodes it, the call in which lamejs throws; it is never packed.  Every handle of a refused call is left exactly
 * as it was before the call (samples, pending frames, ReplayGain analysis), so quieter input continues.
 * Streaming handles: a handle switches to Float32 mode at its first Float32 call (encode_f32, encode_batch_f32, seek_f32)
 * and stays there; its retained samples are converted exactly, and the samples of later Int16 calls are converted too, so
 * any mix of Int16 and Float32 calls encodes as the same mix of Int16Array / Float32Array calls does in lamejs.  A batch may
 * mix handles of both modes.  A Float32-mode handle exports a blob with its own magic ('M3F1', resampled 'M3G1') that carries
 * Float32 samples; importing a blob sets the handle's mode.  flush, the tag and the ReplayGain calls are unchanged.
 * The whole-stream calls take the flags of their Int16 twins: encode_streams_f32 those of _ex, encode_streams_tagged_f32
 * those of _tagged_ex, encode_streams_device_f32 those of _device_ex (d_pcm: one device allocation of Float32 samples laid
 * out like d_pcm there; timings included). */
int mp3b200_encode_f32(mp3b200_encoder* h, const float* left, const float* right, int nsamples, uint8_t* out, int cap);
int mp3b200_encode_batch_f32(mp3b200_encoder* const* handles, const float* const* left, const float* const* right,
                             const int* nsamples, uint8_t* const* out, const int* cap, int nstreams, int* out_bytes);
int mp3b200_seek_f32(mp3b200_encoder* h, int64_t frame, const float* left_hist, const float* right_hist, int nhist);
int mp3b200_encode_streams_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* const* left,
                               const float* const* right, const int64_t* nsamples, uint8_t* const* out,
                               const int64_t* cap, int64_t* out_bytes);
int mp3b200_encode_streams_tagged_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* const* left,
                                      const float* const* right, const int64_t* nsamples, uint8_t* const* out,
                                      const int64_t* cap, int64_t* out_bytes, double* title_db, double* album_db);
int mp3b200_encode_streams_device_f32(int channels, int samplerate, int kbps, int flags, int nstreams, const float* d_pcm,
                                      const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                      const int64_t* out_off, float* timings_ms);
/* Test taps: mp3b200_debug_stages_ex with the input `left` / `right` (right NULL: left) instead of t->left / t->right, and
 * mp3b200_debug_resample / mp3b200_debug_replaygain with Float32 input. */
int mp3b200_debug_stages_f32(const mp3b200_debug_taps* t, const float* left, const float* right);
int mp3b200_debug_resample_f32(int channels, int samplerate, int kbps, const float* left, const float* right, int64_t nsamples,
                               float* y, int64_t ny);
int mp3b200_debug_replaygain_f32(int channels, int samplerate, int kbps, int flags, const float* left, const float* right,
                                 int64_t nsamples, double* win_sums, int32_t* win_idx, int64_t nwin_cap, int32_t* hist,
                                 double* title_db, int32_t* stats);

/* ---- Encode sessions: whole device-resident streams, queued on the caller's CUDA stream (DESIGN.md 14) ----------------
 * A session is bound to one CUDA stream of the device that is current when it is created (NULL: the legacy default
 * stream).  mp3b200_encode_streams_async / _async_f32 encode what mp3b200_encode_streams_device_ex / _device_f32 encode, with
 * the same layout of d_pcm and d_out and the same bytes, but they only queue the work on the session's stream and return:
 * it runs after everything queued there before the call, and work queued there afterwards sees the bytes and d_status.
 * Nothing else orders the call: it does not wait for the legacy default stream.
 *   flags       MP3B200_RESAMPLE or 0 (MP3B200_REPLAYGAIN is refused: mp3b200_encode_streams_tagged_async below takes it).
 *   d_status    int32[4] of device memory, written by the call's last queued operation: [0] a Float32 sample was refused
 *               (not finite, or beyond 2^40 once scaled), [1] a frame did not fit its bit budget (where lamejs throws),
 *               [2] the number of quantizer passes (timings_ms[7] of the synchronous call), [3] an internal fault.  When [0],
 *               [1] or [3] is non-zero the output must not be used; mp3b200_check_status turns the words, copied to the host
 *               once the stream has reached them, into the error code and mp3b200_last_error text of the synchronous call.
 * What the host can see is refused before anything is queued, with the codes and texts of the synchronous call: the
 * arguments by the rules of every whole-stream call (above), a bad configuration; a stream that is capturing a graph returns
 * MP3B200_ERR_HANDLE.
 * The call does not wait for the device, except: on the first use of a configuration on the device (its tables are
 * uploaded), when the session's workspace or pinned staging grows (which may synchronise the device), and when
 * MP3B200_SESSION_SLOTS calls of the session are still in flight (it waits for the oldest).  A session that has seen a
 * launch shape before never waits.  The quantizer's re-validation loop runs on the device, as in every call (a CUDA graph
 * with a conditional WHILE node, captured once per launch shape and kept by the session, at most 32 of them).
 * One call runs at a time per session; sessions share no buffer, so several may be used from one thread or from many.
 * The buffers must stay alive until the stream has reached the call's end.  mp3b200_session_destroy waits for the session's
 * queued work, then frees it. */
#define MP3B200_SESSION_SLOTS 4
typedef struct mp3b200_session mp3b200_session;
int mp3b200_session_create(void* cuda_stream, mp3b200_session** out);
int mp3b200_session_destroy(mp3b200_session* s);
int mp3b200_encode_streams_async(mp3b200_session* s, int channels, int samplerate, int kbps, int flags, int nstreams,
                                 const int16_t* d_pcm, const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                 const int64_t* out_off, int32_t* d_status);
int mp3b200_encode_streams_async_f32(mp3b200_session* s, int channels, int samplerate, int kbps, int flags, int nstreams,
                                     const float* d_pcm, const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                     const int64_t* out_off, int32_t* d_status);
/* status: the first 4 words of d_status in host memory.  0, or the error the synchronous call returns (last_error set). */
int mp3b200_check_status(const int32_t* status);

/* Finished files from a session (DESIGN.md 15): mp3b200_encode_streams_tagged_device / _f32 queued on the session's stream.
 * The same layout and bytes: stream s becomes one file at d_out + out_off[s], its Info / LAME tag frame and then its audio,
 * for flags within MP3B200_RESAMPLE | MP3B200_REPLAYGAIN.  The tag frame is finished on the device (music CRC, Radio Replay
 * Gain field, the tag's own CRC), and the ReplayGain repair loop runs there as a second conditional-WHILE graph, so the
 * call never waits for a result.
 *   out_bytes   host, [nstreams]: each file's length (audio + tag frame), known in closed form and filled when the call
 *               returns.
 *   d_gain      device, [nstreams + 1], written on the session's stream: GetTitleGain of each stream and, last, the album
 *               gain in dB; -24601 wherever the synchronous call hands that out (less than one RMS window, no
 *               MP3B200_REPLAYGAIN, a configuration whose tag does not fit).  May be NULL without MP3B200_REPLAYGAIN.
 *   d_status    device, int32[8]: [0 .. 3] as above (mp3b200_check_status reads them; a ReplayGain loop that hits its bound
 *               raises [3] and reads as the synchronous call's "ReplayGain repair did not converge"), [4] the analysis's
 *               pass count, [5] the chunks it ran again, [6] and [7] zero.
 * Refused before anything is queued, with the synchronous call's codes and texts: the arguments by the rules of every
 * whole-stream call (above), a bad configuration; a capturing stream returns MP3B200_ERR_HANDLE.  The call waits for the device only where
 * mp3b200_encode_streams_async does: everything it uploads is staged in the call's pinned slot. */
int mp3b200_encode_streams_tagged_async(mp3b200_session* s, int channels, int samplerate, int kbps, int flags, int nstreams,
                                        const int16_t* d_pcm, const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                        const int64_t* out_off, int64_t* out_bytes, double* d_gain, int32_t* d_status);
int mp3b200_encode_streams_tagged_async_f32(mp3b200_session* s, int channels, int samplerate, int kbps, int flags, int nstreams,
                                            const float* d_pcm, const int64_t* pcm_off, const int64_t* nsamples, uint8_t* d_out,
                                            const int64_t* out_off, int64_t* out_bytes, double* d_gain, int32_t* d_status);

/* Streaming handles in a session (DESIGN.md 16): encodeBuffer / flush() on n live handles of one configuration, queued on the
 * session's stream.  Entry i's bytes go to d_out + out_off[i]; out_bytes[i] (host) is filled when the call returns and equals
 * what mp3b200_encode_batch_device / _f32 / mp3b200_flush_batch return for the same handles and calls.  d_status is the
 * int32[4] of mp3b200_encode_streams_async (mp3b200_check_status reads it).  Rows are device (or managed) memory on the
 * session's device and may be freed once the stream has passed the call.
 * A handle's first session call binds it to the session (nothing is uploaded, nothing blocks; a handle's tail and carried
 * state live on its device from mp3b200_create on): until mp3b200_session_release gives it back, every host-side call on it
 * (encode, flush, the batch calls, export / import, seek, the tag and ReplayGain setters and getters) and any other
 * session's call returns MP3B200_ERR_HANDLE.  mp3b200_destroy and mp3b200_session_destroy release first.
 * A call refused on the device (a non-finite Float32 sample or one beyond 2^40 once scaled, a frame over its bit budget)
 * commits nothing: each handle it names is marked refused, every later call that names one reports the same refusal in its
 * status, and at release each such handle is exactly where it stood before the refused call.
 * Refused before anything is queued: NULL or repeated handles, a handle with the tag or ReplayGain on, a handle bound to
 * another session, rows that are not device memory on the session's device, a capturing stream, more than 65535 handles
 * (MP3B200_ERR_HANDLE); handles of different configurations or of another device (MP3B200_ERR_CONFIG).  The call waits for
 * the device only where mp3b200_encode_streams_async does. */
int mp3b200_session_encode_batch(mp3b200_session* s, mp3b200_encoder* const* handles, const int16_t* const* d_left,
                                 const int16_t* const* d_right, const int* nsamples, int n, uint8_t* d_out, const int64_t* out_off,
                                 int* out_bytes, int32_t* d_status);
int mp3b200_session_encode_batch_f32(mp3b200_session* s, mp3b200_encoder* const* handles, const float* const* d_left,
                                     const float* const* d_right, const int* nsamples, int n, uint8_t* d_out, const int64_t* out_off,
                                     int* out_bytes, int32_t* d_status);
int mp3b200_session_flush_batch(mp3b200_session* s, mp3b200_encoder* const* handles, int n, uint8_t* d_out, const int64_t* out_off,
                                int* out_bytes, int32_t* d_status);
/* the exact bytes the handle's next call of nsamples samples (-1: flush) hands out; host arithmetic only, bound or not */
int mp3b200_encode_bytes(const mp3b200_encoder* h, int nsamples);
/* the same for every call of a schedule on a fresh handle of the configuration (flags: MP3B200_RESAMPLE), with the tag
 * switched on when write_vbr_tag is non-zero and the tag fits: out_bytes[i] for the call of nsamples[i] samples (-1: flush),
 * the placeholder included.  Host arithmetic only: needs no device. */
int mp3b200_encode_bytes_schedule(int channels, int samplerate, int kbps, int flags, int write_vbr_tag, const int* nsamples, int n,
                                  int* out_bytes);
/* waits for the session's work, settles refusals and gives the handles back to the host calls (unbound handles: no-op),
 * a tagged handle with its music CRC and a ReplayGain handle with its title gain, RadioGain and title count */
int mp3b200_session_release(mp3b200_session* s, mp3b200_encoder* const* handles, int n);
/* the samples per channel a handle's tail buffer holds: the most any handle of the configuration retains after a call that
 * encodes its pending frames (host calls grow a handle's tails when refused calls leave it more) */
int64_t mp3b200_session_tail_capacity(int channels, int samplerate, int kbps, int flags);

/* Tagged and ReplayGain handles in a session (DESIGN.md 17).  mp3b200_session_encode_batch_tagged / _f32 and
 * mp3b200_session_flush_batch_tagged take the arguments of the three calls above and live handles of one configuration in
 * any mix: plain, with the tag (mp3b200_set_write_vbr_tag), and with the tag and ReplayGain (mp3b200_set_find_replay_gain).
 * out_bytes[i] is what mp3b200_encode_bytes says, and the bytes are those of mp3b200_encode_batch_device / _f32 /
 * mp3b200_flush_batch, the all-zero placeholder a tagged handle's first feeding call (or flush) hands out included.  The
 * music CRC, the analysis and the title gains stay on the device and commit only when the call stands.
 *   d_status    int32[8]: [0 .. 3] as for mp3b200_encode_streams_async (mp3b200_check_status reads them; a ReplayGain repair
 *               loop that hits its bound raises [3]: "ReplayGain repair did not converge"), [4] the analysis's pass count,
 *               [5] the chunks it ran again, [6] and [7] zero.
 * Refused before anything is queued: what the calls above refuse, less the rule on the tag and ReplayGain. */
int mp3b200_session_encode_batch_tagged(mp3b200_session* s, mp3b200_encoder* const* handles, const int16_t* const* d_left,
                                        const int16_t* const* d_right, const int* nsamples, int n, uint8_t* d_out, const int64_t* out_off,
                                        int* out_bytes, int32_t* d_status);
int mp3b200_session_encode_batch_tagged_f32(mp3b200_session* s, mp3b200_encoder* const* handles, const float* const* d_left,
                                            const float* const* d_right, const int* nsamples, int n, uint8_t* d_out,
                                            const int64_t* out_off, int* out_bytes, int32_t* d_status);
int mp3b200_session_flush_batch_tagged(mp3b200_session* s, mp3b200_encoder* const* handles, int n, uint8_t* d_out,
                                       const int64_t* out_off, int* out_bytes, int32_t* d_status);
/* Queues, for each handle (one configuration), the frame mp3b200_get_lametag_frame would return at this point of the
 * stream to d_out + out_off[i]; out_bytes[i] (host, known at return) is its size, 0 with the tag off or before the first
 * frame.  The music CRC and the Radio Replay Gain field come from the device.  d_status: int32[4] as for
 * mp3b200_encode_streams_async, non-zero where a handle named was refused by an earlier call.  Binds unbound handles. */
int mp3b200_session_lametag_frames(mp3b200_session* s, mp3b200_encoder* const* handles, int n, uint8_t* d_out, const int64_t* out_off,
                                   int* out_bytes, int32_t* d_status);
/* mp3b200_album_gain queued on the session's stream: GetAlbumGain over the B histograms of the handles that analyse, one double
 * written to device memory d_album (-24601: nothing analysed).  d_status as for mp3b200_session_lametag_frames. */
int mp3b200_session_album_gain(mp3b200_session* s, mp3b200_encoder* const* handles, int n, double* d_album, int32_t* d_status);
/* the loop graphs (quantizer and ReplayGain repair) the session has instantiated so far: flat once its shapes are warm */
int64_t mp3b200_session_graph_instantiations(mp3b200_session* s);

const char* mp3b200_last_error(void);
/* total number of kernel launches issued by this library since load (bench.py "gpu_launches") */
int64_t mp3b200_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
