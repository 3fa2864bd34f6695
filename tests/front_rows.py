"""The front end's remaining rows against the oracle, row for row and bit for bit (tests/test_gpu_front_end_rows.py): the
block types and ATH adjustments of k_stream_scan, the masking rows of k_psy_masking and the xr rows of k_mdct, as the debug
capture records them after k_mdct.  The launch poisons them (and the subband slabs k_mdct reads) before the psy analysis, so
a row it forgets to write shows as NaN, or as block type START where the scan never stores one.  The shapes, the oracle and
the whole-stream driver are tests/psy_rows.py's.

What is compared, for stream unit u (absolute granule c = G frame0 + u) of a launch:
  bt[u]          the oracle's block type of granule c
  bt_prev[u]     blocktype_old as the oracle's psy call of granule c found it
  ath_q[f]       the frame trace's ath_adjust of frame frame0 + f; ath_psy[f] the one before it (0.01 at stream start)
  ratio row u-1  the masking granule c uses: en_l / thm_l always, en_s / thm_s where granule c is short in either channel
                 (elsewhere the short half is not written and stays poisoned); the halo row (u = 0) in all 122 floats
  last row       (u = G nframes - 1) in all 122 floats: the oracle's gfc.en / gfc.thm after the call, the masking handed on
  xr[u]          the frame trace's xr of granule c, all 576 lines

Run as a script (MP3B200_LIB set to a variant build) it checks every row (check_rows) in the whole-stream, ragged-batch and
upload-slice shapes and prints one JSON line {"fail": [first differences], "nfail": n}."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import psy_rows as P  # noqa: E402

BT_START, BT_SHORT = 1, 2
ATH_START = 0.01            # ATH.adjust before the first adjust_ATH (lamejs's start value)
MASK_FIELDS = ("en_l", "thm_l", "en_s", "thm_s")


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize == 8 else np.uint32)


def _floats(rows):
    """ratio rows (PSY_RATIO_DTYPE [..., nch]) as float32 [..., nch, 122] in the record's order"""
    return np.ascontiguousarray(rows).view(np.float32).reshape(rows.shape + (122,))


def _granules(ref, key, c0, n, nch):
    """the frame trace's field `key` of granules c0 .. c0 + n - 1, [n][nch][...]"""
    a = ref.tr[key][:, :ref.G, :nch]
    return a.reshape((-1, nch) + a.shape[3:])[c0:c0 + n]


def _state_floats(st, nch):
    """gfc.en / gfc.thm of an oracle state as [nch][122], the ratio row's order"""
    return np.concatenate([np.asarray(st[k][:nch], np.float32).reshape(nch, -1) for k in MASK_FIELDS], axis=1)


def check_front(rec, refs, label, fail):
    """rec: one launch of a PsyCapture; refs[z]: the psy_rows.Ref (done()) of the launch's stream z.  Appends one entry per
    (stream, unit, channel) that differs, naming the fields, in unit order."""
    for s in rec["streams"]:
        z, frame0, nframes, G = s["z"], s["frame0"], s["nframes"], s["G"]
        if "ratio" not in s:
            fail.append("%s: stream %d: no rows recorded after the MDCT" % (label, z))
            continue
        ref = refs[z]
        assert ref.G == G, (label, ref.G, G)
        nch = s["ratio"].shape[1]
        n, c0 = G * nframes, G * frame0
        if not n:
            continue
        if len(ref.tr) < frame0 + nframes:
            fail.append("%s: stream %d: the oracle traced %d frames, the launch ends at %d" % (label, z, len(ref.tr), frame0 + nframes))
            continue
        bad = {}

        def mark(mask, field):
            for u, ch in np.argwhere(np.asarray(mask).reshape(n, nch)):
                bad.setdefault((int(u), int(ch)), []).append(field)

        mark(s["bt"].astype(np.int64) != _granules(ref, "blocktype", c0, n, nch), "bt")
        prev = ref.bt_old[:, :G, :nch].reshape(-1, nch)[c0:c0 + n]
        mark(s["bt_prev"].astype(np.int64) != prev, "bt_prev")
        # masking: ratio row u - 1 is what granule c uses
        got = s["ratio"][:n]
        short = (ref.bt[c0:c0 + n] == BT_SHORT).any(axis=1)
        for k in MASK_FIELDS:
            want = _granules(ref, k, c0, n, nch)
            d = (bits(got[k]) != bits(want)).reshape(n, nch, -1).any(axis=2)
            if k in ("en_s", "thm_s"):
                d &= (short | (np.arange(n) == 0))[:, None]        # the halo row is compared in full
            mark(d, k)
        mark((bits(s["xr"]) != bits(_granules(ref, "xr", c0, n, nch))).any(axis=2), "xr")
        # the last unit's row in full: the masking the oracle hands the granule after the call
        st = ref.states.get(frame0 + nframes)
        if st is None:
            fail.append("%s: stream %d: no oracle state after frame %d" % (label, z, frame0 + nframes))
        else:
            d = (bits(_floats(s["ratio"][n])) != bits(_state_floats(st, nch))).any(axis=1)
            for ch in np.nonzero(d)[0]:
                bad.setdefault((n - 1, int(ch)), []).append("masking handed on")
        for (u, ch) in sorted(bad):
            fail.append("%s: stream %d unit %d (c %d) ch %d: %s" % (label, z, u, c0 + u, ch, ",".join(bad[u, ch])))
        # ATH: the adjustment each frame's psy calls saw, and the one after adjust_ATH
        ath = ref.tr["ath_adjust"]
        want_q = ath[frame0:frame0 + nframes]
        want_psy = np.concatenate([[ath[frame0 - 1] if frame0 else ATH_START], want_q[:-1]])
        for f in np.nonzero((bits(s["ath_psy"]) != bits(want_psy)) | (bits(s["ath_q"]) != bits(want_q)))[0]:
            fail.append("%s: stream %d frame %d (absolute %d): ath_psy %r / %r, ath_q %r / %r" % (
                label, z, f, frame0 + f, s["ath_psy"][f], want_psy[f], s["ath_q"][f], want_q[f]))


def check_rows(rec, refs, label, fail):
    """every front-end row of one launch: the psy rows and the short list (psy_rows.check_launch), then the rows after k_mdct"""
    P.check_launch(rec, refs, label, fail)
    check_front(rec, refs, label, fail)


def read_rows(bt):
    """R(u) of a launch's stream from its own block types bt [n][nch]: u is the last unit or granule u + 1 is short"""
    n = len(bt)
    return np.array([u == n - 1 or bool((bt[u + 1] == BT_SHORT).any()) for u in range(n)], bool)


def check_unpoisoned(rec, label, fail, halo_start=False):
    """Without an oracle (a seeked handle): every row the launch writes holds no NaN and no block type the scan never stores
    there; with halo_start, the halo row is the stream-start masking (1e20) and the first frame's psy calls saw ATH.adjust
    0.01."""
    for s in rec["streams"]:
        z, n = s["z"], s["G"] * s["nframes"]
        if not n:
            continue
        R = read_rows(s["bt"])
        r = _floats(s["ratio"])
        checks = [("ath_psy", np.isnan(s["ath_psy"]).any()), ("ath_q", np.isnan(s["ath_q"]).any()),
                  ("xr", np.isnan(s["xr"]).any()), ("halo row", np.isnan(r[0]).any()),
                  ("en_l/thm_l", np.isnan(r[1:, :, :44]).any()), ("en_s/thm_s where read", np.isnan(r[1:][R][..., 44:]).any()),
                  ("bt", not np.isin(s["bt"], (0, 1, 2, 3)).all()), ("bt_prev", np.isin(s["bt_prev"], (BT_START,)).any())]
        if halo_start:
            checks += [("halo row != 1e20", (bits(r[0]) != bits(np.float32(1e20))).any()),
                       ("ath_psy of the first frame", s["ath_psy"][0] != ATH_START)]
        for what, bad in checks:
            if bad:
                fail.append("%s: stream %d: %s" % (label, z, what))


def main():
    import lamejs_b200 as M

    assert os.path.samefile(M.lib()._name, os.environ["MP3B200_LIB"])
    fail = []
    P.shape_whole(M, fail, check_rows)
    P.shape_batches(M, fail, check_rows)
    P.shape_slices(M, fail, check_rows)
    print(json.dumps({"fail": fail[:50], "nfail": len(fail)}))


if __name__ == "__main__":
    main()
