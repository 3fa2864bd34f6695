"""Comparison of the CUDA stage taps (lamejs_b200.debug_stages) with the oracle's per-frame traces, shared by the parity
tests: block types, ATH adjustment, the float32 intermediates bit for bit, the quantized lines, every side-info
column of the granule info, and the quantizer's inputs and carried state (scalefactors, xmin, the bin search's
OldValue / CurrentStep chain)."""
import numpy as np

# debug_stages "ginfo" column j holds the trace field GINFO_FIELDS[j] (a (name, index) pair for the per-region arrays)
GINFO_FIELDS = [("global_gain", None), ("part2_3_length", None), ("part2_length", None), ("big_values", None), ("count1", None),
                ("scalefac_compress", None), ("table_select", 0), ("table_select", 1), ("table_select", 2), ("region0", None),
                ("region1", None), ("preflag", None), ("scalefac_scale", None), ("count1table", None), ("blocktype", None)]

ALL_TAPS = ("xr", "blocktype", "en_l", "thm_l", "en_s", "thm_s", "ath_adjust", "l3_enc", "ginfo", "bytes",
            "scalefac", "subblock_gain", "xmin", "max_nonzero_coeff", "xrpow_max", "scfsi", "old_value", "cur_step")

# quantizer state taps: debug_stages "old_value" / "cur_step" [F][3][nch] are the frame start, the state after gr0 (MPEG-1;
# 0 for LSF) and the frame end; the oracle traces them as these fields
STATE_FIELDS = {"old_value": ("old_value_in", "old_value_mid", "old_value_out"),
                "cur_step": ("cur_step_in", "cur_step_mid", "cur_step_out")}


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    u = np.uint64 if a.dtype.itemsize == 8 else np.uint32
    return a.shape == b.shape and a.dtype.itemsize == b.dtype.itemsize and np.array_equal(a.view(u), b.view(u))


def _first_diff(got, want):
    """index of the first element whose bit pattern differs (None if all equal)"""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.shape == want.shape, (got.shape, want.shape)
    u = np.uint64 if got.dtype.itemsize == 8 else np.uint32
    bad = np.argwhere(got.view(u) != want.view(u)) if got.dtype.kind == "f" else np.argwhere(got != want)
    return bad[0].tolist() if len(bad) else None


def compare_quant_state(g, tr, G, ch, label=""):
    """The quantizer's inputs and carried state: scalefactors and subblock gains, calc_xmin's output, max_nonzero_coeff and
    xrpow_max before the rate loop, scfsi, and OldValue / CurrentStep at frame start, after gr0 and at frame end.

    scfsi-shared bands: where gr1 of an MPEG-1 channel reuses gr0's scalefactors (scfsi[ch][band group] = 1), lamejs's
    scfsi_calc sets the gr1 scalefactors of those bands to -1 before the bitstream is written; k_q_finish does the same in
    the device's granule info, so both hold -1 there and the columns are compared as they are.

    On the device side alone, each frame must start from the state its predecessor ended with (in[k+1] == out[k]) and the
    stream's first frame from lamejs's start values (OldValue 180, CurrentStep 4)."""
    sl = (slice(None), slice(0, G), slice(0, ch))
    for k in ("scalefac", "subblock_gain", "max_nonzero_coeff"):
        d = _first_diff(g[k], tr[k][sl])
        assert d is None, (label, k, "first (frame, granule, channel, ...) differing: %s" % d)
    for k in ("xmin", "xrpow_max"):                                   # floats: bit patterns, relative tolerance 0
        d = _first_diff(g[k], tr[k][sl])
        assert d is None, (label, k, "first (frame, granule, channel, ...) differing: %s" % d)
    d = _first_diff(g["scfsi"], tr["scfsi"][:, :ch])
    assert d is None, (label, "scfsi", d)
    for k, fields in STATE_FIELDS.items():
        for j, f in enumerate(fields):
            d = _first_diff(g[k][:, j], tr[f][:, :ch])
            assert d is None, (label, f, "first (frame, channel) differing: %s" % d)
        v = g[k]
        if len(v):
            assert (v[0, 0] == (180 if k == "old_value" else 4)).all(), (label, k, "stream start", v[0, 0].tolist())
            d = _first_diff(v[1:, 0], v[:-1, 2])
            assert d is None, (label, k, "device chain: frame start != predecessor's end at (frame - 1, channel) %s" % d)


def compare(g, tr, ref, G, ch, label=""):
    """Asserts every tap of `g` (debug_stages with want=ALL_TAPS) equals the oracle trace `tr` / bytes `ref`."""
    assert np.array_equal(g["blocktype"], tr["blocktype"][:, :G, :ch]), label
    assert np.array_equal(g["ath_adjust"], tr["ath_adjust"]), label
    for k in ("xr", "en_l", "thm_l", "en_s", "thm_s"):
        assert bits_equal(g[k], tr[k][:, :G, :ch]), (label, k)          # relative tolerance: 0
    assert np.array_equal(g["l3_enc"], tr["l3_enc"][:, :G, :ch]), label
    for j, (k, i) in enumerate(GINFO_FIELDS):
        want = tr[k][:, :G, :ch] if i is None else tr[k][:, :G, :ch, i]
        got = g["ginfo"][..., j]
        if k == "table_select":
            # Huffman table 14 does not exist; the side info names it 16 (BitStream.js).  The oracle's writer renames it in
            # place, so its traces hold 16; the CUDA packer renames it as it writes and its granule info keeps 14.
            got = np.where(got == 14, 16, got)
        bad = np.argwhere(got != want)
        assert len(bad) == 0, (label, k, i, "first (frame, granule, channel) differing: %s" % (bad[0].tolist() if len(bad) else None))
    compare_quant_state(g, tr, G, ch, label)
    assert g["bytes"].tobytes() == ref, label
