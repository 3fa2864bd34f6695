"""The quantizer's rows against the oracle, row for row and bit for bit (tests/test_gpu_front_end_rows.py,
tests/test_gpu_quant_rows.py), as the debug capture records them after the quantizer's fixed point: what k_q_prepare hands
the searches and rate loops, the quantised lines and side info k_q_search / k_q_outer / k_q_finish leave, and the frame
states of the speculation bookkeeping.  The launch poisons them before it starts (mp3_encoder.cu, q_poison), so a row that
no kernel of the launch wrote shows as the poison instead of as a row an earlier launch of the same input left behind.

What is compared, for frame f of a launch's stream (absolute frame frame0 + f), granule gr and channel ch:
  xrq, xrpow     the quant row trace's xrq / xrpow (cod_info.xr as outer_loop receives it, init_xrpow's rows), all 576 lines
  neg            the sign bits of the quant row trace's xrq (bit b of word w: line 32 w + b is negative)
  have, mnz, xrpow_max
                 init_xrpow's result, max_nonzero_coeff after calc_xmin, xrpow_max after init_xrpow
  xmin           calc_xmin's bands 0 .. psymax - 1 where the granule has energy.  A granule without energy (have 0) never
                 reaches calc_xmin in lamejs, whose l3_xmin keeps whatever the previous granule left; k_q_prepare copies its
                 warp's xmin row there as it stands, and nothing reads it.  There only `have` is compared.
  prep block type, and the geometry of the side info (sfbmax, sfbdivide, sfb_lmax, psymax, psy_lmax, sfb_smin): the
                 oracle's block type and the constants of that block type (init_outer_loop)
  l3enc          the frame trace's l3_enc
  side info      the 15 columns of stage_taps.GINFO_FIELDS (table 14 named 16, as the oracle's writer names it), scalefac
                 and subblock_gain
  frame state    in_old / in_step, out_old / out_step with OldValue / CurrentStep at the frame's start and end; MPEG-1:
                 bs_gain0 / bs_step0 with the state after gr0; used0 with gr0's part2_3_length + part2_length; scfsi;
                 stream == z, rel_frame == f and valid == 1 for every frame

A granule without energy holds, by the same rule as lamejs: have 0, mnz 575, xrq and xrpow the oracle's rows, all lines 0,
global_gain 210 and part2_3_length 0; everything but xmin is compared there like anywhere else."""
import numpy as np

from stage_taps import GINFO_FIELDS

BT_SHORT = 2
# device side-info field of each GINFO_FIELDS trace name
DEV_FIELD = {"region0": "region0_count", "region1": "region1_count", "count1table": "count1table_select", "blocktype": "block_type"}
# (sfbmax, sfbdivide, sfb_lmax, psymax, psy_lmax, sfb_smin) of long and short blocks (init_outer_loop)
GEOMETRY = ("sfbmax", "sfbdivide", "sfb_lmax", "psymax", "psy_lmax", "sfb_smin")
GEO_LONG, GEO_SHORT = (21, 11, 21, 21, 21, 12), (36, 18, 0, 36, 0, 0)
# q_poison's values
POISON_NEG = 0xAAAAAAAA
POISON_GAIN = 1


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize == 8 else np.uint32)


def sign_words(xr):
    """the packer's sign masks of rows xr [..., 576]: uint32 [..., 18], bit b of word w set where line 32 w + b is < 0"""
    neg = (np.asarray(xr) < 0).reshape(xr.shape[:-1] + (18, 32)).astype(np.uint64)
    return (neg << np.arange(32, dtype=np.uint64)).sum(axis=-1).astype(np.uint32)


def poisoned_rows(s):
    """per quantizer row of a recorded stream, whether it still holds q_poison's pattern: {name: bool [n][nch]}"""
    p, g = s["prep"], s["ginfo"]
    return {"xrq": (bits(s["xrq"]) == bits(np.float32(1.0))).all(axis=-1),
            "xrpow": (bits(s["xrpow"]) == bits(np.float32(1.0))).all(axis=-1),
            "l3enc": (s["l3enc"] == 1).all(axis=-1),
            "neg": (s["neg"] == POISON_NEG).all(axis=-1),
            "prep": (p["have"] == 1) & (p["mnz"] == 575) & (p["xrpow_max"] == 1.0) & (p["xmin"] == 1.0).all(axis=-1),
            "ginfo": (g["global_gain"] == POISON_GAIN) & (g["part2_3_length"] == 0)}


def check_quant(rec, refs, label, fail):
    """rec: one launch of a PsyCapture; refs[z]: the psy_rows.Ref (done()) of the launch's stream z.  Appends one entry per
    (stream, frame, granule, channel) that differs, naming the fields, in frame order; frame-state fields come first in
    their frame (gr -1)."""
    for s in rec["streams"]:
        z, frame0, nframes, G = s["z"], s["frame0"], s["nframes"], s["G"]
        if "qstate" not in s:
            fail.append("%s: stream %d: no quantizer rows recorded" % (label, z))
            continue
        if not nframes:
            continue
        ref = refs[z]
        assert ref.G == G, (label, ref.G, G)
        nch = s["prep"].shape[1]
        if len(ref.tr) < frame0 + nframes:
            fail.append("%s: stream %d: the oracle traced %d frames, the launch ends at %d" % (label, z, len(ref.tr), frame0 + nframes))
            continue
        tr = ref.tr[frame0:frame0 + nframes]
        n = G * nframes
        bad = {}

        def want(key):
            a = tr[key][:, :G, :nch]
            return a.reshape((n, nch) + a.shape[3:])

        def mark(mask, field):
            for u, ch in np.argwhere(np.asarray(mask).reshape(n, nch)):
                f, gr = divmod(int(u), G)
                bad.setdefault((f, gr, int(ch)), []).append(field)

        def rows_differ(got, exp):
            d = bits(got) != bits(np.asarray(exp, got.dtype)) if got.dtype.kind == "f" else got != exp
            return d.reshape(n, nch, -1).any(axis=2)

        p, g = s["prep"], s["ginfo"]
        have = want("have") != 0
        mark(rows_differ(s["xrq"], want("xrq")), "xrq")
        mark(rows_differ(s["xrpow"], want("xrpow")), "xrpow")
        mark(rows_differ(s["neg"], sign_words(want("xrq"))), "neg")
        mark((p["have"] != 0) != have, "have")
        mark(p["mnz"] != want("max_nonzero_coeff"), "mnz")
        mark(bits(p["xrpow_max"]) != bits(want("xrpow_max")), "xrpow_max")
        bt = want("blocktype")
        psymax = np.where(bt == BT_SHORT, 36, 21)
        in_band = np.arange(39) < psymax[..., None]
        mark(((bits(p["xmin"]) != bits(want("xmin"))) & in_band).any(axis=-1) & have, "xmin")
        mark(p["block_type"] != bt, "prep block_type")
        mark(rows_differ(s["l3enc"].astype(np.int32), want("l3_enc")), "l3enc")
        for k, i in GINFO_FIELDS:
            dev = DEV_FIELD.get(k, k)
            got = g[dev] if i is None else g[dev][..., i]
            if k == "table_select":
                got = np.where(got == 14, 16, got)          # stage_taps.compare: the writer's name of table 14
            mark(got != (want(k) if i is None else want(k)[..., i]), "%s%s" % (k, "" if i is None else "[%d]" % i))
        mark(rows_differ(g["scalefac"], want("scalefac")), "scalefac")
        mark(rows_differ(g["subblock_gain"][..., :3], want("subblock_gain")), "subblock_gain")
        geo = np.where((bt == BT_SHORT)[..., None], np.array(GEO_SHORT), np.array(GEO_LONG))
        for j, k in enumerate(GEOMETRY):
            mark(g[k] != geo[..., j], k)
        # the frame states
        q = s["qstate"]
        pairs = [("in_old", "old_value_in"), ("in_step", "cur_step_in"), ("out_old", "old_value_out"), ("out_step", "cur_step_out")]
        if G == 2:
            pairs += [("bs_gain0", "old_value_mid"), ("bs_step0", "cur_step_mid")]
        for dev, key in pairs:
            for f, ch in np.argwhere(q[dev][:, :nch] != tr[key][:, :nch]):
                bad.setdefault((int(f), -1, int(ch)), []).append(dev)
        used0 = tr["part2_3_length"][:, 0, :nch] + tr["part2_length"][:, 0, :nch]
        for f, ch in np.argwhere(q["used0"][:, :nch] != used0):
            bad.setdefault((int(f), -1, int(ch)), []).append("used0")
        for f, ch in np.argwhere((q["scfsi"][:, :nch] != tr["scfsi"][:, :nch]).any(axis=-1)):
            bad.setdefault((int(f), -1, int(ch)), []).append("scfsi")
        for k, v in (("stream", np.full(nframes, z)), ("rel_frame", np.arange(nframes)), ("valid", np.ones(nframes))):
            for f in np.nonzero(q[k] != v)[0]:
                bad.setdefault((int(f), -1, -1), []).append(k)
        for (f, gr, ch) in sorted(bad):
            where = ("state" + ("" if ch < 0 else " ch %d" % ch)) if gr < 0 else "gr %d ch %d" % (gr, ch)
            fail.append("%s: stream %d frame %d (absolute %d) %s: %s" % (label, z, f, frame0 + f, where, ",".join(bad[f, gr, ch])))


def check_unpoisoned(rec, label, fail):
    """Without an oracle (a seeked handle): no quantizer row of the launch still holds the poison, every frame was packed
    (valid 1) with its own stream and frame number, and each frame starts from the state its predecessor in the launch ended
    with"""
    for s in rec["streams"]:
        z, nframes = s["z"], s["nframes"]
        if "qstate" not in s:
            fail.append("%s: stream %d: no quantizer rows recorded" % (label, z))
            continue
        if not nframes:
            continue
        for what, m in poisoned_rows(s).items():
            if m.any():
                u, ch = np.argwhere(m)[0]
                fail.append("%s: stream %d unit %d ch %d: %s poisoned" % (label, z, u, ch, what))
        q = s["qstate"]
        nch = s["prep"].shape[1]
        checks = [("valid", (q["valid"] != 1).any()), ("stream", (q["stream"] != z).any()),
                  ("rel_frame", (q["rel_frame"] != np.arange(nframes)).any()),
                  ("in_old[k + 1] != out_old[k]", (q["in_old"][1:, :nch] != q["out_old"][:-1, :nch]).any()),
                  ("in_step[k + 1] != out_step[k]", (q["in_step"][1:, :nch] != q["out_step"][:-1, :nch]).any())]
        for what, b in checks:
            if b:
                fail.append("%s: stream %d: %s" % (label, z, what))
