"""The psy rows of k_psy_analysis / k_attack_prepass / k_psy_short against the oracle's psy trace, row for row and bit for bit
(tests/test_gpu_front_end_rows.py), and the launch shapes every front-end row is checked in.  Every call runs under
lamejs_b200.debug_psy_capture(): the launch poisons the rows before the analysis, so a row it forgets to write shows as NaN
(or as mask_idx 8), and the bytes of the call must still equal the oracle's, which shows that no kernel read a row the
launch did not write."""
import numpy as np

import oracle_f32
import oracle_inputs
import oracle_lib
from synth import make_signal

BT_SHORT = 2
PCM_SLICES = 8              # MP3_MAX_PCM_CHUNKS: host calls of <= 8 streams and >= 2^20 samples upload in 8 time slices


class Ref:
    """the oracle encoder of one stream, fed the same calls as the GPU: psy rows, block types and bytes across all calls, and
    `states`: the state after each call (oracle_lib.STATE_DTYPE) by the number of frames encoded so far"""

    def __init__(self, ch, sr, kb, f32=False, trace_frames=4096):
        self.ch = ch
        mod = oracle_f32 if f32 else None
        self.enc = (oracle_f32.Encoder(ch, sr, kb, trace_frames=trace_frames, psy_trace=True) if mod else
                    oracle_lib.OracleEncoder(ch, sr, kb, trace_frames=trace_frames, psy_trace=True))
        self.out = []
        self.states = {}

    def _after_call(self, b):
        st = self.enc.state()
        self.states[int(st["frames_done"])] = st
        self.out.append(b)
        return b

    def call(self, l, r=None):
        return self._after_call(self.enc.encode_buffer(l, r))

    def flush(self):
        return self._after_call(self.enc.flush())

    def stream(self, l, r=None):
        """one whole stream (encodeBuffer once, flush): its bytes"""
        return self.call(l, r) + self.flush() if len(l) else self.flush()

    def done(self):
        """psy rows, blocktype_old per psy call (`bt_old`), frame trace (`tr`), block types [unit][ch] and partition counts of
        everything encoded so far"""
        self.psy = self.enc.psy_traces()
        self.bt_old = self.enc.psy_block_traces()
        G = self.G = 2 if self.sr_out >= 32000 else 1
        tr = self.tr = self.enc.traces()
        self.bt = tr["blocktype"][:, :G, :self.ch].reshape(-1, self.ch)
        self.npl, self.nps = self.enc.npart()
        return self


def make_ref(ch, sr, kb, f32=False):
    r = Ref(ch, sr, kb, f32)
    r.sr_out = oracle_lib.out_samplerate(ch, sr, kb)
    return r


def bits(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a.view(np.uint32)


def unit_want(ref, c, ch):
    """the oracle's long row of absolute unit c (c = -1: psymodel_init's values)"""
    if c < 0:
        return np.zeros(64, np.float32), np.zeros(64, np.int64), np.full(9, 10.0, np.float32), np.float32(0), np.zeros(4, np.int64)
    f, gr = divmod(c, ref.G)
    p = ref.psy[f]
    return p["eb_l"][gr, ch], p["mask_idx_l"][gr, ch], p["peaks"][gr, ch], p["loudness"][gr, ch], p["attack"][gr, ch]


def short_want(ref, c, ch):
    if c < 0:
        return np.ones((3, 64), np.float32), np.zeros((3, 64), np.float32)
    f, gr = divmod(c, ref.G)
    p = ref.psy[f]
    return p["ecb_s"][gr, ch], p["eb_s"][gr, ch]


def read_rule(ref, frame0, n):
    """S(u) for u = -1 .. n - 1 of a launch's stream: R(u) = u is its last unit, or granule u + 1 is short in either channel;
    S(u) = R(u) or R(u + 1)"""
    G = ref.G

    def R(u):
        if u < 0 or u >= n:
            return False
        return u == n - 1 or bool((ref.bt[G * frame0 + u + 1] == BT_SHORT).any())
    return [u for u in range(-1, n) if R(u) or R(u + 1)]


def check_launch(rec, refs, label, fail):
    """rec: one launch of a PsyCapture; refs[z]: the Ref (done()) of the launch's stream z"""
    short_want_set = []
    for s in rec["streams"]:
        z, frame0, nframes, G = s["z"], s["frame0"], s["nframes"], s["G"]
        ref = refs[z]
        assert ref.G == G, (label, ref.G, G)
        rows = s["rows"]
        n = G * nframes
        for u in range(-1, n):
            c = G * frame0 + u
            for ch in range(rows.shape[1]):
                got = rows[u + 1, ch]
                eb, mi, pk, ld, at = unit_want(ref, c, ch)
                npl = ref.npl
                bad = []
                if not np.array_equal(bits(got["eb_l"][:npl]), bits(eb[:npl])):
                    bad.append("eb_l")
                if not np.array_equal(got["mask_idx"][:npl].astype(np.int64), np.asarray(mi[:npl], np.int64)):
                    bad.append("mask_idx")
                if not np.array_equal(bits(got["peaks"]), bits(pk)):
                    bad.append("peaks")
                if bits(got["loudness"]) != bits(ld):
                    bad.append("loudness")
                # the halo row's attack is written only where it is unit -1 of the stream (psymodel_init's 0): after the
                # first call the scan starts from the carried lastAttacks and nothing reads it
                if (u >= 0 or c < 0) and not np.array_equal(got["attack"].astype(np.int64), np.asarray(at, np.int64)):
                    bad.append("attack")
                if bad:
                    fail.append("%s: stream %d unit %d (c %d) ch %d: %s" % (label, z, u, c, ch, ",".join(bad)))
        short_want_set += [(z, u, ch) for u in read_rule(ref, frame0, n) for ch in range(rows.shape[1])]
    got_list = [tuple(int(v) for v in e) for e in rec["short"]]
    if sorted(got_list) != sorted(short_want_set):
        extra = sorted(set(got_list) - set(short_want_set))[:5]
        missing = sorted(set(short_want_set) - set(got_list))[:5]
        fail.append("%s: short list: %d listed, %d by the rule; extra %s missing %s" % (label, len(got_list), len(short_want_set),
                                                                                   extra, missing))
    frame0s = {s["z"]: s["frame0"] for s in rec["streams"]}
    for (z, u, ch), row in zip(got_list, rec["short_rows"]):
        ref = refs[z]
        c = ref.G * frame0s[z] + u
        ecb, eb = short_want(ref, c, ch)
        nps = ref.nps
        if not (np.array_equal(bits(row["ecb_s"][:, :nps].astype(np.float32)), bits(ecb[:, :nps])) and
                np.array_equal(bits(row["eb_s"][:, :nps]), bits(eb[:, :nps]))):
            fail.append("%s: short row of stream %d unit %d (c %d) ch %d" % (label, z, u, c, ch))


# ---- signals aimed at K2's edges ------------------------------------------------------------------------------------------

def impulses(n, seed=0, amp=20000):
    """single impulses at the 64-sample sub-block boundaries of the units (unit c's high-pass output q is centred on sample
    576 c + 183 + q), inside the 448-sample overlap of consecutive units [576 c + 352, 576 c + 800), and at its two ends;
    one or two impulses per unit, on either side of the boundary"""
    x = np.zeros(n, np.int16)
    rng = np.random.default_rng(seed)
    for c in range(0, n // 576 + 1):
        k = c % 13
        if k < 10:
            p = 576 * c + 183 + 64 * k - (c // 13) % 2
        elif k == 10:
            p = 576 * c + 352 + int(rng.integers(0, 448))
        elif k == 11:
            p = 576 * c + 352 - (c // 13) % 2
        else:
            p = 576 * c + 799 + (c // 13) % 2
        if 0 <= p < n and c % 2 == 0:
            x[p] = amp if c % 4 == 0 else -amp
    return x


def quiet(n, lsb, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(-lsb, lsb + 1, n).astype(np.int16)


def k2_signal(kind, n, seed):
    """(left, right) of one of the K2 edge signals"""
    if kind == "silence":
        z = np.zeros(n, np.int16)
        return z, z.copy()
    if kind.startswith("quiet"):
        lsb = int(kind[5:])
        return quiet(n, lsb, seed), quiet(n, max(1, lsb // 2), seed + 1)
    if kind == "dc_pos":
        return np.full(n, 32767, np.int16), np.full(n, -32768, np.int16)
    if kind == "dc_neg":
        return np.full(n, -32768, np.int16), np.full(n, 32767, np.int16)
    if kind == "nyquist":
        x = np.where(np.arange(n) % 2 == 0, 32767, -32768).astype(np.int16)
        return x, (-x.astype(np.int32)).clip(-32768, 32767).astype(np.int16)
    if kind == "impulses":
        return impulses(n, seed), impulses(n, seed + 1, amp=-12000)
    if kind == "mixed":
        # impulses over noise, a silent stretch, quiet noise: attacks, short blocks and the loudness rule in one stream
        l, r = make_signal("burst", n, 44100, seed)
        l = (l.astype(np.int32) // 4 + impulses(n, seed)).clip(-32768, 32767).astype(np.int16)
        a, b = n // 3, n // 2
        l[a:b] = 0
        r[a:b] = quiet(b - a, 3, seed)
        return l, r
    raise ValueError(kind)


K2_KINDS = ["silence", "quiet1", "quiet8", "quiet64", "dc_pos", "dc_neg", "nyquist", "impulses", "mixed"]


# ---- shapes ---------------------------------------------------------------------------------------------------------------

def native_configs():
    """every rate of CONFIG_MATRIX_RATES, mono and stereo, at a bitrate it encodes without resampling (npart_l and npart_s
    differ by rate)"""
    out = []
    for sr in oracle_inputs.CONFIG_MATRIX_RATES:
        kb = 128 if sr >= 32000 else 64 if sr >= 16000 else 32
        for ch in (1, 2):
            assert oracle_lib.out_samplerate(ch, sr, kb) == sr, (ch, sr, kb)
            out.append((ch, sr, kb))
    return out


def capture_call(M, fn):
    with M.debug_psy_capture() as cap:
        res = fn()
    return res, cap.launches


def whole_streams(M, ch, sr, kb, sigs, label, fail, check, f32=False, resample=False):
    """one host call over `sigs` (a batch when several); rows (`check`) and bytes against one oracle per stream"""
    refs = [make_ref(ch, sr, kb, f32) for _ in sigs]
    want = [rf.stream(l, r if ch == 2 else None) for rf, (l, r) in zip(refs, sigs)]
    for rf in refs:
        rf.done()
    got, launches = capture_call(M, lambda: M.encode_streams(ch, sr, kb, [l for l, _ in sigs], [r for _, r in sigs] if ch == 2 else None,
                                                             resample=resample))
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            fail.append("%s: bytes of stream %d" % (label, i))
    base = 0
    for rec in launches:
        k = len(rec["streams"])
        check(rec, refs[base:base + k], label, fail)
        base += k
    if base != len(sigs):
        fail.append("%s: %d streams recorded, %d encoded" % (label, base, len(sigs)))
    return launches


def stream_lengths(M, ch, sr, kb):
    """0, 1, 575, 576, 1376, 1377 samples (only the halo, or the halo and one unit) and two longer streams whose frame
    counts differ in parity"""
    fs = 576 * M.granules_per_frame(ch, sr, kb)
    return [0, 1, 575, 576, 1376, 1377, 12 * fs + 300, 13 * fs + 300]


def shape_whole(M, fail, check):
    for j, (ch, sr, kb) in enumerate(native_configs()):
        lens = stream_lengths(M, ch, sr, kb)
        for i, n in enumerate(lens):
            kind = K2_KINDS[(i + j) % len(K2_KINDS)]
            whole_streams(M, ch, sr, kb, [k2_signal(kind, n, 100 * j + i)], "whole %d/%d/%d n=%d %s" % (ch, sr, kb, n, kind), fail,
                          check)


BATCHES = [
    ((2, 44100, 128), [0, 1, 700, 1376, 1377, 5000, 1152 * 7, 1152 * 31 + 5, 1152 * 64]),
    ((1, 44100, 128), [0, 1, 700, 1376, 1377, 5000, 1152 * 7, 1152 * 31 + 5, 1152 * 64]),
    ((2, 22050, 64), [0, 1, 575, 576, 800, 1329, 5000, 576 * 40 + 3]),
    ((1, 16000, 24), [0, 1, 575, 576, 800, 1329, 5000, 576 * 40 + 3]),
]


def shape_batches(M, fail, check):
    for (ch, sr, kb), lens in BATCHES:
        sigs = [k2_signal(K2_KINDS[i % len(K2_KINDS)], n, 300 + i) if i % 2 else make_signal("burst", n, sr, 300 + i)
                for i, n in enumerate(lens)]
        whole_streams(M, ch, sr, kb, sigs, "batch %d/%d/%d" % (ch, sr, kb), fail, check)


def slice_of(c, pcm_base, n, nchunks=PCM_SLICES):
    """psy_unit_in_slice: the upload slice holding the last sample of unit c's 1024-sample window"""
    last = min(576 * c - 224 + 1023 - pcm_base, n - 1)
    mine = 0
    while mine < nchunks - 1 and last >= n * (mine + 1) // nchunks:
        mine += 1
    return mine


def slice_pairs(G, lens):
    """(u_lo[j], whether a block of slice j's launch holds a unit of slice j + 1) for slices j = 0 .. 6, over streams of lens"""
    u_lo = [None] * PCM_SLICES
    mine = {}
    for s, n in enumerate(lens):
        F = (n + 576 * G - 1) // (576 * G) + 2      # more units than the stream has only widens the search below
        for u in range(-1, G * F):
            j = slice_of(u, 0, n)
            mine[s, u] = j
            u_lo[j] = u if u_lo[j] is None else min(u_lo[j], u)
    out = []
    for j in range(PCM_SLICES - 1):
        if u_lo[j] is None:
            continue
        cross = any(mine.get((s, u)) == j and mine.get((s, u + 1)) == j + 1 and (u - u_lo[j]) % 2 == 0
                    for (s, u) in mine)
        out.append((u_lo[j], cross))
    return out


def slice_lengths(M, ch, sr, kb, nstreams, seed):
    """stream lengths of >= 2^20 samples in all (both channels): the first stream's slice boundary n / 2 is exactly the last
    sample of unit c's window (576 c + 799, where >= and > in the slice rule part) and c lies beyond slice 3's launch (which
    would compute it from slice 4's samples); and slice boundaries fall inside a block's pair of units for both an even and
    an odd u_lo[j]"""
    G = M.granules_per_frame(ch, sr, kb)
    rng = np.random.default_rng(seed)
    tot = (1 << 20) // ch + 1
    for _ in range(400):
        c = int(rng.integers(tot // nstreams // 1152 + 1, tot // nstreams // 1152 + 40))
        lens = [2 * (576 * c + 799) + int(rng.integers(0, 2))]
        lens += [int(v) for v in rng.integers(tot // nstreams, tot // nstreams + 20000, nstreams - 1)]
        if sum(lens) * ch < (1 << 20):
            continue
        pairs = slice_pairs(G, lens)
        if ((c - pairs[3][0]) % 2 == 0 and any(x and lo % 2 == 0 for lo, x in pairs) and
                any(x and lo % 2 for lo, x in pairs)):
            return lens
    raise AssertionError("no slicing found")


def shape_slices(M, fail, check):
    for (ch, sr, kb), nstreams in (((2, 44100, 128), 1), ((1, 22050, 64), 3)):
        lens = slice_lengths(M, ch, sr, kb, nstreams, 7 + nstreams)
        sigs = [k2_signal("mixed", n, 500 + i) for i, n in enumerate(lens)]
        launches = whole_streams(M, ch, sr, kb, sigs, "slices %d/%d/%d" % (ch, sr, kb), fail, check)
        G = M.granules_per_frame(ch, sr, kb)
        want = len({slice_of(u, 0, n) for n in lens for u in range(-1, G * M.stream_frames(n, ch, sr, kb))})
        for rec in launches:
            if rec["k2_launches"] != want:
                fail.append("slices %d/%d/%d: %d k_psy_analysis launches, %d slices hold units" % (ch, sr, kb, rec["k2_launches"], want))
