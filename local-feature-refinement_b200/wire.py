"""types.proto I/O: MatchingFile in, SolutionFile out (solve.cc:412-481, 643-679).

The bytes are decoded / encoded by the native codec in csrc/lfr_wire.cc (csrc/liblfr_host.so) through
the C ABI of include/lfr_wire.h (no libprotobuf, no per-match Python loop).  A
matches file may be split into `<path>.part.0, .part.1, ...`
(compute_match_graph.py:189-205); like solve.cc:416-424 the parts are read only
when `<path>` itself does not exist.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional

import numpy as np

from .capi import load_host
from .matchset import MatchSet


class WireMatches(C.Structure):
    _fields_ = [("n_pairs", C.c_uint64), ("n_matches", C.c_uint64), ("pair_ptr", C.c_void_p),
                ("fact1", C.c_void_p), ("fact2", C.c_void_p), ("name1_off", C.c_void_p),
                ("name1_len", C.c_void_p), ("name2_off", C.c_void_p), ("name2_len", C.c_void_p),
                ("feat1", C.c_void_p), ("feat2", C.c_void_p), ("sim", C.c_void_p),
                ("disp1", C.c_void_p), ("disp2", C.c_void_p)]


WIRE_SYMBOLS = ["lfr_wire_scan_matches", "lfr_wire_decode_matches", "lfr_wire_walk_matches", "lfr_wire_encode_matches",
                "lfr_wire_encode_solution", "lfr_wire_decode_solution"]

_bound = False


def _lib():
    global _bound
    L = load_host()
    if not _bound:
        L.lfr_wire_scan_matches.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.lfr_wire_scan_matches.restype = C.c_int
        L.lfr_wire_decode_matches.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(WireMatches)]
        L.lfr_wire_decode_matches.restype = C.c_int
        L.lfr_wire_walk_matches.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(WireMatches), C.c_void_p]
        L.lfr_wire_walk_matches.restype = C.c_int
        L.lfr_wire_encode_matches.argtypes = [C.c_uint64] + [C.c_void_p] * 12 + [C.c_void_p, C.c_uint64]
        L.lfr_wire_encode_matches.restype = C.c_int64
        L.lfr_wire_encode_solution.argtypes = [C.c_uint64] + [C.c_void_p] * 7 + [C.c_void_p, C.c_uint64]
        L.lfr_wire_encode_solution.restype = C.c_int64
        L.lfr_wire_decode_solution.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                               C.POINTER(C.c_uint64)] + [C.c_void_p] * 7
        L.lfr_wire_decode_solution.restype = C.c_int
        _bound = True
    return L


class ParseError(RuntimeError):
    """"Failed to parse proto object." (solve.cc:433-436)"""


def matches_files(path: str) -> List[str]:
    """solve.cc:416-424"""
    if os.path.exists(path):
        return [path]
    out = []
    k = 0
    while os.path.exists("%s.part.%d" % (path, k)):
        out.append("%s.part.%d" % (path, k))
        k += 1
    return out


def _pair_level(data: bytes, with_matches: bool) -> dict:
    """lfr_wire_decode_matches (with_matches) or lfr_wire_walk_matches on `data`: the arrays of
    lfr_wire_matches by field name, plus `match_off` from the walk.  Raises ParseError."""
    L = _lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    np_, nm = C.c_uint64(), C.c_uint64()
    ptr = buf.ctypes.data if buf.size else None
    if L.lfr_wire_scan_matches(ptr, buf.size, C.byref(np_), C.byref(nm)) != 0:
        raise ParseError("Failed to parse proto object.")
    P, M = int(np_.value), int(nm.value)
    a = dict(
        pair_ptr=np.zeros(P + 1, np.uint64), fact1=np.zeros(P, np.float32), fact2=np.zeros(P, np.float32),
        name1_off=np.zeros(P, np.uint64), name1_len=np.zeros(P, np.uint32),
        name2_off=np.zeros(P, np.uint64), name2_len=np.zeros(P, np.uint32),
    )
    if with_matches:
        a.update(feat1=np.zeros(M, np.uint32), feat2=np.zeros(M, np.uint32), sim=np.zeros(M, np.float32),
                 disp1=np.zeros((M, 18), np.float32), disp2=np.zeros((M, 18), np.float32))
    w = WireMatches(n_pairs=P, n_matches=M, **{k: v.ctypes.data for k, v in a.items()})
    if with_matches:
        rc = L.lfr_wire_decode_matches(ptr, buf.size, C.byref(w))
    else:
        a["match_off"] = np.zeros(M, np.uint64)
        rc = L.lfr_wire_walk_matches(ptr, buf.size, C.byref(w), a["match_off"].ctypes.data)
    if rc != 0:
        raise ParseError("Failed to parse proto object.")
    return a


def intern_names(data: bytes, a: dict, names: List[str], index: dict):
    """Image ids of both sides of every pair of `a` (_pair_level), names numbered in order of first
    appearance; `names` / `index` carry the numbering across the parts of one file."""
    P = a["pair_ptr"].shape[0] - 1
    img1 = np.zeros(P, np.int64)
    img2 = np.zeros(P, np.int64)
    for p in range(P):
        for (off, ln, dst) in ((a["name1_off"], a["name1_len"], img1), (a["name2_off"], a["name2_len"], img2)):
            nm_ = data[int(off[p]): int(off[p]) + int(ln[p])].decode("utf-8", errors="surrogateescape")
            if nm_ not in index:
                index[nm_] = len(names)
                names.append(nm_)
            dst[p] = index[nm_]
    return img1, img2


def walk_matching_file(data: bytes) -> dict:
    """The pair level of one MatchingFile and the byte offset of every match (lfr_wire_walk_matches):
    pair_ptr, fact1, fact2, name1_off, name1_len, name2_off, name2_len, match_off.  No match is decoded;
    raises ParseError on what lfr_wire_scan_matches rejects."""
    return _pair_level(data, with_matches=False)


def decode_matching_file(data: bytes) -> MatchSet:
    a = _pair_level(data, with_matches=True)
    names: List[str] = []
    img1, img2 = intern_names(data, a, names, {})
    return MatchSet(image_names=names, pair_img1=img1, pair_img2=img2, pair_fact1=a["fact1"],
                    pair_fact2=a["fact2"], pair_ptr=a["pair_ptr"].astype(np.int64), feat1=a["feat1"],
                    feat2=a["feat2"], sim=a["sim"], disp1=a["disp1"], disp2=a["disp2"])


def read_matching_file(path: str) -> MatchSet:
    files = matches_files(path)
    parts = []
    for f in files:
        with open(f, "rb") as fh:
            parts.append(decode_matching_file(fh.read()))
    if len(parts) == 1:
        return parts[0]
    return MatchSet.concatenate(parts)


def _names_blob(names: List[str]):
    enc = [n.encode("utf-8", errors="surrogateescape") for n in names]
    off = np.zeros(len(enc) + 1, np.uint64)
    if enc:
        off[1:] = np.cumsum([len(e) for e in enc])
    blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
    return blob, off


def encode_matching_file(ms: MatchSet, pair_lo: int = 0, pair_hi: Optional[int] = None) -> bytes:
    L = _lib()
    pair_hi = ms.n_pairs if pair_hi is None else pair_hi
    blob, off = _names_blob(ms.image_names)
    n = pair_hi - pair_lo
    pair_ptr = np.ascontiguousarray(ms.pair_ptr[pair_lo:pair_hi + 1], dtype=np.uint64)
    n1 = np.ascontiguousarray(ms.pair_img1[pair_lo:pair_hi], dtype=np.uint32)
    n2 = np.ascontiguousarray(ms.pair_img2[pair_lo:pair_hi], dtype=np.uint32)
    f1 = np.ascontiguousarray(ms.pair_fact1[pair_lo:pair_hi], dtype=np.float32)
    f2 = np.ascontiguousarray(ms.pair_fact2[pair_lo:pair_hi], dtype=np.float32)
    arrs = [pair_ptr, n1, n2, f1, f2, blob, off,
            np.ascontiguousarray(ms.feat1, np.uint32), np.ascontiguousarray(ms.feat2, np.uint32),
            np.ascontiguousarray(ms.sim, np.float32), np.ascontiguousarray(ms.disp1, np.float32),
            np.ascontiguousarray(ms.disp2, np.float32)]
    ptrs = [x.ctypes.data for x in arrs]
    # one call into a buffer of the largest possible size (a match is at most 18 x 12 displacement bytes +
    # 17 of scalars + 3 of framing; a pair two names, two facts and framing) instead of a sizing call first
    n_m = int(pair_ptr[-1] - pair_ptr[0]) if n else 0
    longest = int(np.max(off[1:] - off[:-1])) if len(ms.image_names) else 0
    cap = 240 * n_m + (2 * longest + 64) * n + 16
    out = np.empty(cap, np.uint8)
    need = int(L.lfr_wire_encode_matches(n, *ptrs, out.ctypes.data, cap))
    assert 0 <= need <= cap
    return out[:need].tobytes()


def write_matching_file(ms: MatchSet, path: str, pairs_per_part: Optional[int] = None) -> List[str]:
    """Write `path`, or `path.part.N` every `pairs_per_part` pairs like
    compute_match_graph.py:78,189-205 (dump_interval = 5000)."""
    if pairs_per_part is None or ms.n_pairs <= pairs_per_part:
        with open(path, "wb") as fh:
            fh.write(encode_matching_file(ms))
        return [path]
    files = []
    k = 0
    for lo in range(0, ms.n_pairs, pairs_per_part):
        f = "%s.part.%d" % (path, k)
        with open(f, "wb") as fh:
            fh.write(encode_matching_file(ms, lo, min(ms.n_pairs, lo + pairs_per_part)))
        files.append(f)
        k += 1
    return files


def encode_solution(image_names: List[str], fact: np.ndarray, img_ptr: np.ndarray,
                    feature_idx: np.ndarray, di: np.ndarray, dj: np.ndarray) -> bytes:
    L = _lib()
    blob, off = _names_blob(image_names)
    arrs = [np.ascontiguousarray(img_ptr, np.uint64), blob, off, np.ascontiguousarray(fact, np.float32),
            np.ascontiguousarray(feature_idx, np.uint32), np.ascontiguousarray(di, np.float32),
            np.ascontiguousarray(dj, np.float32)]
    ptrs = [x.ctypes.data for x in arrs]
    need = L.lfr_wire_encode_solution(len(image_names), *ptrs, None, 0)
    out = np.zeros(max(int(need), 1), np.uint8)
    got = L.lfr_wire_encode_solution(len(image_names), *ptrs, out.ctypes.data, int(need))
    assert got == need
    return out[:need].tobytes()


def decode_solution(data: bytes):
    """-> list of (image_name, fact, feature_idx[], di[], dj[])"""
    L = _lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    ptr = buf.ctypes.data if buf.size else None
    ni, nd = C.c_uint64(), C.c_uint64()
    if L.lfr_wire_decode_solution(ptr, buf.size, C.byref(ni), C.byref(nd), *([None] * 7)) != 0:
        raise ParseError("Failed to parse proto object.")
    I, D = int(ni.value), int(nd.value)
    img_ptr = np.zeros(I + 1, np.uint64); noff = np.zeros(I, np.uint64); nlen = np.zeros(I, np.uint32)
    fact = np.zeros(I, np.float32); fi = np.zeros(D, np.uint32)
    di = np.zeros(D, np.float32); dj = np.zeros(D, np.float32)
    rc = L.lfr_wire_decode_solution(ptr, buf.size, C.byref(ni), C.byref(nd), img_ptr.ctypes.data,
                                    noff.ctypes.data, nlen.ctypes.data, fact.ctypes.data, fi.ctypes.data,
                                    di.ctypes.data, dj.ctypes.data)
    if rc != 0:
        raise ParseError("Failed to parse proto object.")
    out = []
    for i in range(I):
        a, b = int(img_ptr[i]), int(img_ptr[i + 1])
        nm = data[int(noff[i]): int(noff[i]) + int(nlen[i])].decode("utf-8", errors="surrogateescape")
        out.append((nm, float(fact[i]), fi[a:b], di[a:b], dj[a:b]))
    return out
