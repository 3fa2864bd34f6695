"""Static sharding of independent streams over ranks + the final byte gather (SURVEY.md 8(e)).

Streams (lamejs Mp3Encoder instances) never exchange data while encoding, so the multi-GPU plan is: stream j goes to
rank j % world (round-robin, like config C4), every rank encodes its shard with no collective on the data path, and the
encoded bytes are gathered to rank 0 at the end.  CBR without reservoir makes every stream's byte count a closed form of
its sample count (mp3b200_stream_bytes), so each rank knows all sizes up front and the gather needs no size exchange.
Backend-agnostic: NCCL on GPUs (bench.py), gloo in the CPU tests."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
import torch.distributed as dist


def shard_streams(nstreams, world, rank):
    """Indices of the streams rank `rank` encodes (round-robin)."""
    return list(range(rank, nstreams, world))


def shard_layout(stream_bytes, world):
    """Per rank: (stream indices, byte offset of each of its streams inside the rank's packed buffer, total)."""
    out = []
    for r in range(world):
        idx = shard_streams(len(stream_bytes), world, r)
        offs = np.concatenate([[0], np.cumsum([stream_bytes[i] for i in idx])]).astype(np.int64)
        out.append((idx, offs[:-1], int(offs[-1])))
    return out


def gather_encoded(packed, stream_bytes, group=None, dst=0):
    """`packed`: this rank's encoded streams back to back (uint8 tensor on the backend's device).  Returns on `dst` the
    list of per-stream byte tensors in global stream order, None elsewhere.  One collective: a padded gather."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    layout = shard_layout(stream_bytes, world)
    cap = max(l[2] for l in layout)
    buf = torch.zeros(cap, dtype=torch.uint8, device=packed.device)
    buf[: packed.numel()] = packed
    bufs = [torch.empty_like(buf) for _ in range(world)] if rank == dst else None
    dist.gather(buf, bufs, dst=dst, group=group)
    if rank != dst:
        return None
    result = [None] * len(stream_bytes)
    for r, (idx, offs, _) in enumerate(layout):
        for i, o in zip(idx, offs):
            result[i] = bufs[r][int(o): int(o) + int(stream_bytes[i])]
    return result


# ---- one long stream cut into contiguous frame ranges (SURVEY.md 8(e)(2)) -------------------------------------------------
# An MP3 frame depends on its predecessors only through a small sequential state (ATH adjust, block-type FSM, bin-search start
# gain, the previous granule's masking); after a few frames that state no longer depends on where the encoder started.  Rank r
# therefore starts `warmup` frames early from a stream-START state (Mp3Encoder.seek), throws those frames away, and keeps going
# through its own range; afterwards the ranks pass their END states down the line (one ~4 KB blob each): a rank whose state
# after the warm-up equals its predecessor's end state has produced exactly the single-encoder bytes; a rank that does not
# (e.g. a long quiet passage, where ATH adjust decays over many frames) imports the true state and encodes its range again.
# The result is always the single-encoder stream; speculation only decides how parallel the work was.

def segment_bounds(nsamples, framesize, world):
    """Frame ranges [lo, hi) per rank: boundaries lie among the frames encodeBuffer alone completes (the flush tail belongs to
    the last rank); returns (bounds, frames_without_flush)."""
    body = max(0, (nsamples - 224) // framesize)          # frames complete after n samples: f * framesize + 224 <= n
    cuts = [body * r // world for r in range(world)] + [None]
    return [(cuts[r], cuts[r + 1]) for r in range(world)], body


def encode_segment(make_encoder, left, right, framesize, lo, hi, warmup, state_in=None):
    """Encodes frames [lo, hi) of the stream (hi None: to the end, with flush).  state_in: the exact state at frame lo (blob) or
    None = warm up from `warmup` frames earlier.  Returns (bytes, state assumed at lo, end state or None for the last range)."""
    n = len(left)
    first = lambda f: f * framesize + 224                  # samples that complete exactly f frames
    enc = make_encoder()
    if state_in is not None:
        enc.import_state(state_in)
        at_lo = state_in
    elif lo == 0:
        at_lo = None                                       # stream start: exact by construction
    else:
        start = lo - warmup
        if start >= 1:
            h0 = max(0, start * framesize - 1104)
            enc.seek(start, left[h0:first(start)], None if right is None else right[h0:first(start)])
            pos = first(start)
        else:                                              # the warm-up reaches the stream start: no guess involved
            pos = 0
        warm = enc.encodeBuffer(left[pos:first(lo)], None if right is None else right[pos:first(lo)])
        del warm
        at_lo = enc.export_state() if start >= 1 else None
    pos = first(lo) if lo > 0 else 0
    end = n if hi is None else first(hi)
    out = enc.encodeBuffer(left[pos:end], None if right is None else right[pos:end])
    if hi is None:
        out += enc.flush()
        end_state = None
    else:
        end_state = enc.export_state()
    enc.close()
    return out, at_lo, end_state


def encode_stream_segments_local(make_encoder, left, right, framesize, nseg, warmup=8):
    """All ranks' work in one process, in rank order (tests, and what a single GPU would do): returns (stream bytes, number of
    ranges that had to be re-encoded from the true state)."""
    bounds, _ = segment_bounds(len(left), framesize, nseg)
    spec = [encode_segment(make_encoder, left, right, framesize, lo, hi, warmup) for lo, hi in bounds]
    out, redone, prev_end = [], 0, None
    for r, (lo, hi) in enumerate(bounds):
        b, at_lo, end_state = spec[r]
        if r > 0 and at_lo is not None and at_lo != prev_end:
            b, _, end_state = encode_segment(make_encoder, left, right, framesize, lo, hi, warmup, state_in=prev_end)
            redone += 1
        out.append(b)
        prev_end = end_state
    return b"".join(out), redone


def encode_stream_segments(make_encoder, left, right, framesize, warmup=8, group=None, device="cpu"):
    """One stream over the ranks of `group`: every rank passes the same PCM (or at least the part its range and warm-up read).
    Speculative encode in parallel, then one pass of end states down the line (send / recv of a fixed-size blob + a flag).
    Returns on rank 0 the whole stream's bytes and the number of re-encoded ranges; (None, n) elsewhere."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    bounds, _ = segment_bounds(len(left), framesize, world)
    lo, hi = bounds[rank]
    b, at_lo, end_state = encode_segment(make_encoder, left, right, framesize, lo, hi, warmup)
    redone = 0
    if rank > 0:
        size = torch.zeros(1, dtype=torch.int64, device=device)
        dist.recv(size, src=rank - 1, group=group)
        blob = torch.empty(int(size.item()), dtype=torch.uint8, device=device)
        dist.recv(blob, src=rank - 1, group=group)
        prev_end = blob.cpu().numpy().tobytes()
        if at_lo is not None and at_lo != prev_end:
            b, _, end_state = encode_segment(make_encoder, left, right, framesize, lo, hi, warmup, state_in=prev_end)
            redone = 1
    if rank < world - 1:
        blob = torch.from_numpy(np.frombuffer(end_state, dtype=np.uint8).copy()).to(device)
        dist.send(torch.tensor([blob.numel()], dtype=torch.int64, device=device), dst=rank + 1, group=group)
        dist.send(blob, dst=rank + 1, group=group)
    sizes = torch.zeros(world, dtype=torch.int64, device=device)
    sizes[rank] = len(b)
    dist.all_reduce(sizes, group=group)
    cnt = torch.tensor([redone], dtype=torch.int64, device=device)
    dist.all_reduce(cnt, group=group)
    cap = int(sizes.max().item())
    buf = torch.zeros(cap, dtype=torch.uint8, device=device)
    buf[: len(b)] = torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).to(device)
    bufs = [torch.empty_like(buf) for _ in range(world)] if rank == 0 else None
    dist.gather(buf, bufs, dst=0, group=group)
    if rank != 0:
        return None, int(cnt.item())
    return b"".join(bufs[r][: int(sizes[r].item())].cpu().numpy().tobytes() for r in range(world)), int(cnt.item())


# ---- finished files from segments ----------------------------------------------------------------------------------------
# The segments are encoded untagged, exactly as above; the file is finished afterwards on rank 0.  Every field of the tag
# frame is a closed form of the sample count (frames, bytes, seek table, encoder padding) or a function of the joined audio
# (music CRC), and lamejs's ReplayGain depends only on the PCM and on the pieces one encodeBuffer(whole) + flush() feeds it,
# not on the encoded bytes.  So rank 0 analyses the whole stream once on a second host thread (its own CUDA stream) while
# its range encodes, joins the ranges' audio behind the tag frame's room in one buffer and finishes the frame there
# (mp3b200_finish_tags_device).  The result is the file encode_streams_replaygain makes of the whole stream.

def _finished(encode_audio, room, analyse, finish, file_device):
    """encode_audio() -> (joined audio bytes, or None off rank 0; ranges re-encoded).  analyse() (None: no analysis) runs on
    a second thread beside it and returns the title gain.  finish(buf, title_db) writes the tag frame into buf[:room] of the
    buffer holding the audio behind it and returns the file's length.  Returns (file bytes, ranges re-encoded, title_db),
    with title_db None when nothing was analysed, or (None, redone, None) where encode_audio gave no audio."""
    with ThreadPoolExecutor(max_workers=1) as pool:
        gain = pool.submit(analyse) if analyse is not None else None
        try:
            audio, redone = encode_audio()
        finally:
            title_db = gain.result() if gain is not None else None     # joins the thread; re-raises its error
    if audio is None:
        return None, redone, None
    buf = torch.zeros(room + len(audio), dtype=torch.uint8, device=file_device)
    if audio:
        buf[room:] = torch.frombuffer(bytearray(audio), dtype=torch.uint8).to(file_device)
    n = finish(buf, title_db)
    return buf[:n].cpu().numpy().tobytes(), redone, title_db


def encode_segments_tagged_local(make_encoder, left, right, framesize, nseg, warmup, room, analyse, finish, file_device="cpu"):
    """encode_stream_segments_local made into a finished file by _finished (its arguments: room, analyse, finish)"""
    return _finished(lambda: encode_stream_segments_local(make_encoder, left, right, framesize, nseg, warmup), room, analyse,
                     finish, file_device)


def encode_segments_tagged(make_encoder, left, right, framesize, room, analyse, finish, warmup=8, group=None, device="cpu",
                           file_device="cpu"):
    """encode_stream_segments made into a finished file on rank 0 by _finished; only rank 0 runs `analyse`"""
    rank = dist.get_rank(group)
    return _finished(lambda: encode_stream_segments(make_encoder, left, right, framesize, warmup, group, device), room,
                     analyse if rank == 0 else None, finish, file_device)


def _library_parts(channels, samplerate, kbps, left, right, find_replay_gain):
    """the libmp3b200 pieces of a segmented finished file: (make_encoder, framesize, room, analyse, finish, file_device)"""
    from . import encoder as E
    if E.out_samplerate(channels, samplerate, kbps) != samplerate:
        raise ValueError("(%d, %d, %d) is resampled by lamejs: a resampled stream cannot be cut into segments (seek does not "
                         "take resampling encoders)" % (channels, samplerate, kbps))
    gr = E.granules_per_frame(channels, samplerate, kbps)
    if gr < 0:
        raise E.Mp3B200Error("unsupported configuration: channels=%d samplerate=%d kbps=%d" % (channels, samplerate, kbps))
    right = None if channels == 1 else right
    probe = E.Mp3Encoder(channels, samplerate, kbps)
    device = probe.device                                   # the library's device: where the encoders and the file live
    probe.close()
    room = E.lametag_size(channels, samplerate, kbps)
    n = len(left)

    def analyse():
        if E._on_cuda(left) or E._on_cuda(right):
            (l,), (r,), f32 = E._device_rows([left], [right], device)
            pcm = l if channels == 1 else torch.cat([l, r])
            return E.replay_gain_streams_device(channels, samplerate, kbps, pcm.data_ptr(), [0], [n], float32=f32)[0][0]
        return E.replay_gain_streams(channels, samplerate, kbps, [left], None if right is None else [right])[0][0]

    def finish(buf, title_db):
        return E.finish_tags_device(channels, samplerate, kbps, buf.data_ptr(), [0], [n],
                                    None if title_db is None else [title_db])[0]

    # lamejs analyses only when the tag is written (Lame.js:911-916)
    return (lambda: E.Mp3Encoder(channels, samplerate, kbps), 576 * gr, room, analyse if find_replay_gain and room > 0 else None,
            finish, "cuda:%d" % device)


def _title(title_db):
    from .encoder import GAIN_NOT_ENOUGH_SAMPLES
    return float(GAIN_NOT_ENOUGH_SAMPLES) if title_db is None else title_db


def encode_stream_segments_tagged_local(channels, samplerate, kbps, left, right, nseg, warmup=8, find_replay_gain=False):
    """One stream cut into `nseg` frame ranges, encoded one after another in this process, as one finished file: returns (file
    bytes, ranges re-encoded, title_db), the file byte-identical to encode_streams_replaygain([left], [right],
    find_replay_gain=...)[0][0] and title_db to its title gain (-24601 when nothing was analysed).  Int16 or floating-point
    rows, in host memory or CUDA tensors on the library's device; configurations lamejs resamples raise ValueError."""
    make, fs, room, analyse, finish, file_device = _library_parts(channels, samplerate, kbps, left, right, find_replay_gain)
    out, redone, title_db = encode_segments_tagged_local(make, left, None if channels == 1 else right, fs, nseg, warmup, room,
                                                         analyse, finish, file_device)
    return out, redone, _title(title_db)


def encode_stream_segments_tagged(channels, samplerate, kbps, left, right, warmup=8, find_replay_gain=False, group=None,
                                  device="cpu"):
    """encode_stream_segments_tagged_local over the ranks of `group` (one range each; `device` is the collectives' device, as
    for encode_stream_segments): returns the same on rank 0, (None, ranges re-encoded, None) elsewhere.  Rank 0 analyses
    the whole stream beside its own range and finishes the file on the library's device."""
    make, fs, room, analyse, finish, file_device = _library_parts(channels, samplerate, kbps, left, right, find_replay_gain)
    out, redone, title_db = encode_segments_tagged(make, left, None if channels == 1 else right, fs, room, analyse, finish,
                                                   warmup, group, device, file_device)
    return (None, redone, None) if out is None else (out, redone, _title(title_db))
