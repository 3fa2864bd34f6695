'use strict';
/**
 * lamejs-compatible facade over libmp3b200.so (H100-native MP3 encoder).
 *
 *   const lamejs = require('mp3b200');            // instead of require('lamejs')
 *   const enc = new lamejs.Mp3Encoder(2, 44100, 128);
 *   const mp3 = enc.encodeBuffer(left, right);    // Int16Array (or, as in lamejs, Float32Array / Array of numbers) in,
 *                                                 // Int8Array out (frames completed by this call)
 *   const tail = enc.flush();
 *
 * Same constructor / encodeBuffer / flush surface and return types as zhuker/lamejs src/js/index.js:66-136.
 * Binding: ffi-napi over the C ABI declared in include/mp3b200.h.  No node in the build image: the file is exercised there under
 * Qt's JavaScript engine with a stubbed ffi (tests/test_js_shim.py: syntax, exports, call order and arity), not against the GPU.
 */
const ffi = require('ffi-napi');
const ref = require('ref-napi');

const voidPtr = ref.refType(ref.types.void);
const voidPtrPtr = ref.refType(voidPtr);
const lib = ffi.Library(process.env.MP3B200_LIB || 'libmp3b200', {
  mp3b200_create: ['int', ['int', 'int', 'int', voidPtrPtr]],
  mp3b200_encode: ['int', [voidPtr, 'pointer', 'pointer', 'int', 'pointer', 'int']],
  mp3b200_flush: ['int', [voidPtr, 'pointer', 'int']],
  mp3b200_destroy: ['void', [voidPtr]],
  mp3b200_export_state: ['int', [voidPtr, 'pointer', 'int']],
  mp3b200_import_state: ['int', [voidPtr, 'pointer', 'int']],
  mp3b200_seek: ['int', [voidPtr, 'int64', 'pointer', 'pointer', 'int']],
  mp3b200_encode_f32: ['int', [voidPtr, 'pointer', 'pointer', 'int', 'pointer', 'int']],
  mp3b200_seek_f32: ['int', [voidPtr, 'int64', 'pointer', 'pointer', 'int']],
  mp3b200_set_write_vbr_tag: ['int', [voidPtr, 'int']],
  mp3b200_get_lametag_frame: ['int', [voidPtr, 'pointer', 'int']],
  mp3b200_set_find_replay_gain: ['int', [voidPtr, 'int']],
  mp3b200_get_replay_gain: ['int', [voidPtr, 'pointer', 'pointer']],
  mp3b200_album_gain: ['int', ['pointer', 'int', 'pointer']],
  mp3b200_lametag_size: ['int', ['int', 'int', 'int']],
  mp3b200_wav_read_header: ['int', ['pointer', 'int64', 'pointer']],
  mp3b200_last_error: ['string', []],
});

/**
 * `options.writeVbrTag` (beyond lamejs, which hard-codes gfp.bWriteVbrTag = false at index.js:107): LAME's Info / LAME tag.
 * The first bytes handed out are then an all-zero placeholder frame; after flush(), getLameTagFrame() returns the finished
 * frame (frame / byte counts, seek table, encoder delay and padding, CRC-16 of the audio computed on the GPU) to be written
 * over the first `length` bytes of the file -- what LAME's frontend does with lame_get_lametag_frame (VBRTag.js:829-965).
 */
function Mp3Encoder(channels, samplerate, kbps, options) {
  if (arguments.length < 3) {                // index.js:67-72
    console.error('WARN: Mp3Encoder(channels, samplerate, kbps) not specified');
    channels = 1; samplerate = 44100; kbps = 128;
  }
  const hp = ref.alloc(voidPtr);
  const rc = lib.mp3b200_create(channels, samplerate, kbps, hp);
  if (rc !== 0) throw new Error('mp3b200_create failed (' + rc + '): ' + lib.mp3b200_last_error());
  const h = hp.deref();
  let tagRoom = 0;
  if (options && options.writeVbrTag) {
    const on = lib.mp3b200_set_write_vbr_tag(h, 1);          // 0: the frame is too small for the tag (InitVbrTag refuses)
    if (on < 0) throw new Error('mp3b200_set_write_vbr_tag failed (' + on + '): ' + lib.mp3b200_last_error());
    if (on === 1) tagRoom = lib.mp3b200_lametag_size(channels, samplerate, kbps);
    // options.findReplayGain: gfp.findReplayGain (needs the tag): each flush() ends a title; replayGain() reads it
    if (options.findReplayGain) {
      const rg = lib.mp3b200_set_find_replay_gain(h, 1);
      if (rg < 0) throw new Error('mp3b200_set_find_replay_gain failed (' + rg + '): ' + lib.mp3b200_last_error());
    }
  }
  this._handle = h;
  let maxSamples = 1152;
  let buf = Buffer.alloc((0 | (1.25 * maxSamples + 7200)) + tagRoom);   // index.js:113-114

  const asBuf = (a) => Buffer.from(a.buffer, a.byteOffset, a.byteLength);
  // lamejs copies whatever it is given into Float32Arrays (Lame.js:1500-1510): an Int16Array pair keeps the Int16 entry
  // point, anything else (Float32Array, Float64Array, a plain Array of numbers) is stored into a Float32Array the same way
  const isInt16 = (a) => a instanceof Int16Array;
  const asF32 = (a) => (a instanceof Float32Array ? a : Float32Array.from(a));

  this.encodeBuffer = function (left, right) {
    if (channels === 1) right = left;
    if (left.length > maxSamples) {                          // index.js:122-126
      maxSamples = left.length;
      buf = Buffer.alloc((0 | (1.25 * maxSamples + 7200)) + tagRoom);
    }
    const n = isInt16(left) && isInt16(right)
      ? lib.mp3b200_encode(h, asBuf(left), asBuf(right), left.length, buf, buf.length)
      : lib.mp3b200_encode_f32(h, asBuf(asF32(left)), asBuf(asF32(right)), left.length, buf, buf.length);
    if (n < 0) throw new Error('mp3b200_encode failed (' + n + '): ' + lib.mp3b200_last_error());
    return new Int8Array(buf.subarray(0, n));                // a fresh copy, like index.js:129
  };

  this.flush = function () {
    const n = lib.mp3b200_flush(h, buf, buf.length);
    if (n < 0) throw new Error('mp3b200_flush failed (' + n + '): ' + lib.mp3b200_last_error());
    return new Int8Array(buf.subarray(0, n));
  };

  // ---- beyond lamejs: the Info / LAME tag frame (empty Int8Array when the tag is off or nothing was encoded yet) ----
  this.getLameTagFrame = function () {
    const t = Buffer.alloc(2880);                            // VBRTag.MAXFRAMESIZE
    const n = lib.mp3b200_get_lametag_frame(h, t, t.length);
    if (n < 0) throw new Error('mp3b200_get_lametag_frame failed (' + n + '): ' + lib.mp3b200_last_error());
    return new Int8Array(t.subarray(0, n));
  };

  // ---- beyond lamejs: the encoder state as a blob (checkpoint / resume; segment workers, see INTEGRATION.md) ----
  this.exportState = function () {
    const n = lib.mp3b200_export_state(h, ref.NULL, 0);
    if (n < 0) throw new Error('mp3b200_export_state failed (' + n + '): ' + lib.mp3b200_last_error());
    const blob = Buffer.alloc(n);
    const m = lib.mp3b200_export_state(h, blob, n);
    if (m < 0) throw new Error('mp3b200_export_state failed (' + m + '): ' + lib.mp3b200_last_error());
    return blob.subarray(0, m);
  };
  this.importState = function (blob) {
    const rc = lib.mp3b200_import_state(h, blob, blob.length);
    if (rc !== 0) throw new Error('mp3b200_import_state failed (' + rc + '): ' + lib.mp3b200_last_error());
  };
  this.seek = function (frame, leftHist, rightHist) {
    if (channels === 1 || !rightHist) rightHist = leftHist;
    const rc = isInt16(leftHist) && isInt16(rightHist)
      ? lib.mp3b200_seek(h, frame, asBuf(leftHist), asBuf(rightHist), leftHist.length)
      : lib.mp3b200_seek_f32(h, frame, asBuf(asF32(leftHist)), asBuf(asF32(rightHist)), leftHist.length);
    if (rc !== 0) throw new Error('mp3b200_seek failed (' + rc + '): ' + lib.mp3b200_last_error());
  };

  /** {titleDb, radioGain} of the title the last flush() ended, or null (before it, or without options.findReplayGain) */
  this.replayGain = function () {
    const db = ref.alloc('double'), radio = ref.alloc('int');
    const rc = lib.mp3b200_get_replay_gain(h, db, radio);
    if (rc < 0) throw new Error('mp3b200_get_replay_gain failed (' + rc + '): ' + lib.mp3b200_last_error());
    return rc === 1 ? { titleDb: db.deref(), radioGain: radio.deref() } : null;
  };
  this.close = function () { lib.mp3b200_destroy(h); };
}

/** lamejs.WavHeader (src/js/index.js:138-193), parsed by the library: same fields, same outcomes -- undefined for a
 * non-RIFF / non-WAVE / fmt-not-first buffer, throws 'extended fmt chunk not implemented' for fmt lengths other than 16 / 18,
 * RangeError where the reference's DataView reads leave the buffer. */
function WavHeader() { this.dataOffset = 0; this.dataLen = 0; this.channels = 0; this.sampleRate = 0; }
WavHeader.readHeader = function (dataView) {
  const bytes = Buffer.from(dataView.buffer, dataView.byteOffset, dataView.byteLength);
  const out = Buffer.alloc(24);                              // struct mp3b200_wav_header {i64, i64, i32, u32}
  const rc = lib.mp3b200_wav_read_header(bytes, bytes.length, out);
  if (rc === 0) return undefined;
  if (rc === -1) throw 'extended fmt chunk not implemented';
  if (rc !== 1) throw new RangeError('Offset is outside the bounds of the DataView');
  const w = new WavHeader();
  w.dataOffset = Number(out.readBigInt64LE(0)); w.dataLen = Number(out.readBigInt64LE(8));
  w.channels = out.readInt32LE(16); w.sampleRate = out.readUInt32LE(20);
  return w;
};

/** GetAlbumGain over the titles the encoders (options.findReplayGain) have ended with flush() */
Mp3Encoder.albumGain = function (encoders) {
  const hs = Buffer.alloc(8 * Math.max(encoders.length, 1));
  encoders.forEach((e, i) => ref.writePointer(hs, i * 8, e._handle));
  const out = ref.alloc('double');
  const rc = lib.mp3b200_album_gain(hs, encoders.length, out);
  if (rc < 0) throw new Error('mp3b200_album_gain failed (' + rc + '): ' + lib.mp3b200_last_error());
  return out.deref();
};

module.exports = { Mp3Encoder, WavHeader };
