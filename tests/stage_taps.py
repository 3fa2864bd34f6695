"""Comparison of the CUDA stage taps (lamejs_b200.debug_stages) with the oracle's per-frame traces, shared by the parity
tests: block types, ATH adjustment, the float32 intermediates bit for bit, the quantized lines and every side-info
column of the granule info."""
import numpy as np

# debug_stages "ginfo" column j holds the trace field GINFO_FIELDS[j] (a (name, index) pair for the per-region arrays)
GINFO_FIELDS = [("global_gain", None), ("part2_3_length", None), ("part2_length", None), ("big_values", None), ("count1", None),
                ("scalefac_compress", None), ("table_select", 0), ("table_select", 1), ("table_select", 2), ("region0", None),
                ("region1", None), ("preflag", None), ("scalefac_scale", None), ("count1table", None), ("blocktype", None)]

ALL_TAPS = ("xr", "blocktype", "en_l", "thm_l", "en_s", "thm_s", "ath_adjust", "l3_enc", "ginfo", "bytes")


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


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
    assert g["bytes"].tobytes() == ref, label
