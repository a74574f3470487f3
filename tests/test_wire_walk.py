"""The pair walk (lfr_wire_walk_matches, include/lfr_wire.h) against the full host decode
(lfr_wire_decode_matches): the same pair-level arrays on every encoding, the same refusals, and match
offsets that point at each match's length prefix.  CPU only; the device decode of the matches the walk
locates is tests/test_gpu_wire_decode.py."""
import struct

import numpy as np
import pytest

from lfr_b200 import synth, wire
from proto_runtime import MatchingFile, matchset_to_proto

PAIR_LEVEL = ("pair_ptr", "fact1", "fact2", "name1_off", "name1_len", "name2_off", "name2_len")


def _f32(tag, v):
    return bytes([tag]) + struct.pack("<f", v)


def _varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    return bytes(out + bytes([v]))


def _lenpref(tag, payload):
    return bytes([tag]) + _varint(len(payload)) + payload


def one_match_file(match: bytes) -> bytes:
    """A MatchingFile of one pair ("x", "y") holding the given Match payload."""
    pair = _lenpref(0x0A, b"x") + _f32(0x15, 2.0) + _lenpref(0x1A, b"y") + _f32(0x25, 4.0) + _lenpref(0x2A, match)
    return _lenpref(0x0A, pair)


def small_matchset():
    """tests/test_wire.py's small_ms: proto3 corner cases, zero scalars omitted on the wire."""
    ms = synth.generate("cfg1", scale=0.25)
    ms.feat1[0] = 0
    ms.sim[1] = 0.0
    ms.disp1[2, :] = 0.0
    ms.disp2[3, 4] = -0.0
    ms.pair_fact2[0] = 0.0
    ms.feat1[5] = 2 ** 32 - 1
    return ms


def encodings():
    """{name: MatchingFile bytes}: every well-formed encoding tests/test_wire.py decodes, and the other
    legal forms a Match may take."""
    ms = small_matchset()
    out = {"protobuf": matchset_to_proto(ms).SerializeToString(),
           "unknown_top_level": wire.encode_matching_file(ms) + bytes([0x78, 0x05, 0x82, 0x01, 0x03, 1, 2, 3])}
    mf = MatchingFile()
    ip = mf.image_pairs.add()
    ip.image_name1, ip.image_name2, ip.fact1, ip.fact2 = "a", "b", 1.0, 2.0
    m = ip.matches.add()
    m.feature_idx1, m.feature_idx2, m.similarity = 7, 9, 0.5
    for g in range(3):
        d = m.disp1.add()
        d.di, d.dj = g + 1.0, -(g + 1.0)
    for g in range(11):
        d = m.disp2.add()
        d.di, d.dj = 0.25 * g, 0.5 * g
    out["short_and_long_displacement_lists"] = mf.SerializeToString()
    disps = [_f32(0x0D, 1.5) + _f32(0x15, -2.5),                       # canonical
             _f32(0x15, 4.0) + _f32(0x0D, 3.0),                        # dj first
             _f32(0x0D, 5.0), _f32(0x15, 6.0), b"",                    # zeros omitted
             _f32(0x0D, 7.0) + bytes([0x18, 0x2A]) + _f32(0x15, 8.0),  # unknown varint inside
             _f32(0x0D, 9.0) + _f32(0x0D, 10.0) + _f32(0x15, 11.0),    # repeated: the last one counts
             _f32(0x0D, 1.0) + bytes([0x19]) + b"\1" * 8 + _f32(0x15, 2.0),   # unknown fixed64
             _f32(0x0D, 1.0) + bytes([0x22, 2, 9, 9]) + _f32(0x15, 2.0),      # unknown bytes
             _f32(0x0D, 1.0) + bytes([0x2D]) + b"\1" * 4,                     # unknown fixed32
             bytes([0x0D]) + b"\0" * 4 + bytes([0x15]) + b"\0" * 4]          # explicit zeros, 10 bytes
    out["non_canonical_displacements"] = one_match_file(
        bytes([0x08, 3, 0x10, 4]) + _f32(0x1D, 0.75) + b"".join(_lenpref(0x22, d) for d in disps)
        + _lenpref(0x2A, _f32(0x0D, -1.0) + _f32(0x15, -3.0)))
    # repeated scalars (the last one counts), 10-byte varints (feature_idx truncated to 32 bits), unknown
    # fields of wire types 0, 1, 2 and 5 at the Match level
    out["repeated_scalars_long_varints_unknown_fields"] = one_match_file(
        bytes([0x08, 3, 0x08, 5, 0x10] + [0xFF] * 9 + [0x01]) + _f32(0x1D, 0.5) + _f32(0x1D, 0.25)
        + bytes([0x30, 7, 0x39]) + b"\2" * 8 + bytes([0x42, 1, 0, 0x4D]) + b"\3" * 4
        + bytes([0x08] + [0x80] * 9 + [0x00]))
    out["zero_omitted_scalars"] = one_match_file(b"")
    return out


def malformed_match_files():
    """Buffers whose pair level walks but whose matches the host decode rejects."""
    bad = {"varint_11_bytes": bytes([0x08] + [0x80] * 10 + [0x01]),
           "fixed32_cut": bytes([0x1D, 1, 2]),
           "displacement_past_the_match": bytes([0x22, 0x7F, 0x0D]),
           "unknown_bytes_past_the_match": bytes([0x42, 0x09, 1])}
    for wt in (3, 4, 6, 7):
        bad["wire_type_%d" % wt] = bytes([0x30 | wt, 0])
        bad["wire_type_%d_in_displacement" % wt] = _lenpref(0x22, bytes([0x18 | wt, 0]))
    return {k: one_match_file(v) for k, v in bad.items()}


def _decode_arrays(data):
    try:
        return wire._pair_level(data, with_matches=True)
    except wire.ParseError:
        return None


def _walk_arrays(data):
    try:
        return wire.walk_matching_file(data)
    except wire.ParseError:
        return None


@pytest.mark.parametrize("name", sorted(encodings()))
def test_walk_gives_the_decodes_pair_level(name):
    data = encodings()[name]
    want, got = _decode_arrays(data), _walk_arrays(data)
    assert want is not None and got is not None
    for k in PAIR_LEVEL:
        assert got[k].tobytes() == want[k].tobytes(), k
    off = got["match_off"]
    assert off.shape == want["feat1"].shape and np.all(np.diff(off.astype(np.int64)) > 0)
    buf = np.frombuffer(data, np.uint8)
    assert np.all(buf[off.astype(np.int64) - 1] == 0x2A)   # each offset follows a Match tag (field 5, bytes)
    assert np.all(off < len(data))


def test_walk_on_a_file_of_several_megabytes():
    """The size at which the decode deals pairs to worker threads; the walk stays serial."""
    blob = wire.encode_matching_file(synth.generate("cfg2", scale=0.5))
    assert len(blob) > (4 << 20)
    want, got = _decode_arrays(blob), _walk_arrays(blob)
    for k in PAIR_LEVEL:
        assert got[k].tobytes() == want[k].tobytes(), k
    assert got["match_off"].shape == want["sim"].shape


def test_walk_refuses_what_the_scan_refuses():
    """Truncations at every byte, garbage and length prefixes past the end: the walk fails exactly where
    lfr_wire_scan_matches does; where it passes, only the contents of matches can still be wrong."""
    small = one_match_file(bytes([0x08, 3, 0x10, 4]) + _f32(0x1D, 0.75) + _lenpref(0x22, _f32(0x0D, 1.0) + _f32(0x15, 2.0)))
    data = wire.encode_matching_file(synth.generate("cfg1", scale=0.1))
    cases = [small[:k] for k in range(len(small))] + [data[:k] for k in range(0, len(data), 13)]
    cases += [b"\x0a\xff\xff\xff\xff\x0f", data[:-3], b"\x0a\x05\x2a\x09", b"\x0b"]
    L = wire._lib()
    import ctypes as C
    n_walk_ok = 0
    for b in cases:
        buf = np.frombuffer(b, np.uint8)
        scan_ok = L.lfr_wire_scan_matches(buf.ctypes.data if buf.size else None, buf.size, C.byref(C.c_uint64()),
                                          C.byref(C.c_uint64())) == 0
        walk_ok = _walk_arrays(b) is not None
        assert walk_ok == scan_ok
        n_walk_ok += walk_ok
        if _decode_arrays(b) is not None:
            assert walk_ok
    assert 0 < n_walk_ok < len(cases)
    for name, b in malformed_match_files().items():
        assert _walk_arrays(b) is not None and _decode_arrays(b) is None, name


def test_walk_refuses_wrong_capacities():
    import ctypes as C
    data = encodings()["protobuf"]
    a = wire.walk_matching_file(data)
    P, M = a["pair_ptr"].shape[0] - 1, a["match_off"].shape[0]
    L = wire._lib()
    buf = np.frombuffer(data, np.uint8)
    for p, m in ((P - 1, M), (P, M - 1), (P, M + 1)):
        arrs = {k: np.zeros(max(p + (k == "pair_ptr"), 1), a[k].dtype) for k in PAIR_LEVEL}
        off = np.zeros(max(m, 1), np.uint64)
        w = wire.WireMatches(n_pairs=p, n_matches=m, **{k: v.ctypes.data for k, v in arrs.items()})
        assert L.lfr_wire_walk_matches(buf.ctypes.data, buf.size, C.byref(w), off.ctypes.data) != 0
    arrs = {k: np.zeros_like(a[k]) for k in PAIR_LEVEL}
    w = wire.WireMatches(n_pairs=P, n_matches=M, **{k: v.ctypes.data for k, v in arrs.items()})
    assert L.lfr_wire_walk_matches(buf.ctypes.data, buf.size, C.byref(w), None) != 0   # match_off required


def test_decode_rule_is_a_match_count_threshold():
    """lfr_wire_decode_on_device (include/lfr_graph.h): the drop-in's choice between the decoder on the GPU
    and the host decode on its device route, from the match count alone; needs no device."""
    import os
    from lfr_b200.capi import B200_LIB_PATH, GRAPH_SYMBOLS, Library
    if not os.path.exists(B200_LIB_PATH):
        pytest.skip("product library not built")
    lib = Library(B200_LIB_PATH)
    assert "lfr_wire_decode_on_device" in GRAPH_SYMBOLS
    f = lib.lib.lfr_wire_decode_on_device
    assert f(0) == 0 and f(25195) == 0 and f(100572) == 0 and f(634185) == 1 and f(5483733) == 1   # cfg2 x 0.25 ... cfg5
    flips = [n for n in range(1, 700001, 97) if f(n) != f(n - 97 if n > 97 else 0)]
    assert len(flips) == 1                       # one threshold
