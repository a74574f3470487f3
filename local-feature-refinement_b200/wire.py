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
                "lfr_wire_encode_solution", "lfr_wire_decode_solution", "lfr_wire_join_solution",
                "lfr_wire_join_solution_entries", "lfr_wire_encode_solution_carried", "lfr_wire_update_solution",
                "lfr_wire_update_solution_since", "lfr_host_problem_record", "lfr_wire_update_solution_since_record",
                "lfr_wire_update_solution_groups", "lfr_host_problem_record_groups"]

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
        L.lfr_wire_join_solution.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        L.lfr_wire_join_solution.restype = C.c_int
        L.lfr_wire_join_solution_entries.argtypes = L.lfr_wire_join_solution.argtypes + [C.c_void_p]
        L.lfr_wire_join_solution_entries.restype = C.c_int
        L.lfr_wire_encode_solution_carried.argtypes = ([C.c_uint64] + [C.c_void_p] * 7 + [C.c_void_p, C.c_uint64, C.c_void_p,
                                                        C.c_uint64, C.POINTER(C.c_uint64)])
        L.lfr_wire_encode_solution_carried.restype = C.c_int64
        L.lfr_wire_update_solution.argtypes = ([C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32]
                                               + [C.c_void_p] * 3 + [C.c_uint32, C.c_void_p, C.c_void_p,
                                                                     C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)])
        L.lfr_wire_update_solution.restype = C.c_int
        L.lfr_wire_update_solution_since.argtypes = ([C.c_void_p, C.c_uint64, C.c_uint32] + [C.c_void_p] * 10 +
                                                     [C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)])
        L.lfr_wire_update_solution_since.restype = C.c_int
        L.lfr_host_problem_record.argtypes = [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 3 + [C.c_uint64]
        L.lfr_host_problem_record.restype = C.c_int64
        L.lfr_wire_update_solution_since_record.argtypes = ([C.c_void_p, C.c_uint64, C.c_uint32] + [C.c_void_p] * 6 +
                                                            [C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64),
                                                             C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)])
        L.lfr_wire_update_solution_since_record.restype = C.c_int
        L.lfr_wire_update_solution_groups.argtypes = ([C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] +
                                                      [C.c_void_p] * 9 + [C.POINTER(C.c_uint64), C.POINTER(C.c_uint32),
                                                                            C.POINTER(C.c_uint32)])
        L.lfr_wire_update_solution_groups.restype = C.c_int
        L.lfr_host_problem_record_groups.argtypes = ([C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 3 + [C.c_uint32] +
                                                     [C.c_void_p, C.c_uint64, C.c_void_p])
        L.lfr_host_problem_record_groups.restype = C.c_int64
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


def encode_solution_carried(image_names: List[str], fact: np.ndarray, img_ptr: np.ndarray, feature_idx: np.ndarray,
                            di: np.ndarray, dj: np.ndarray, carry: bytes):
    """encode_solution() of a scene's output merged with the earlier SolutionFile `carry`
    (lfr_wire_encode_solution_carried, include/lfr_wire.h): each scene image gets, after its displacements,
    the entries `carry` has for it and the scene does not (ascending feature); then come the winning Image
    messages of `carry` whose names are not scene images, in file order.  Returns (bytes, number of carried
    entries).  Raises ParseError on bytes the decoder rejects and ValueError on repeated image names."""
    L = _lib()
    blob, off = _names_blob(image_names)
    arrs = [np.ascontiguousarray(img_ptr, np.uint64), blob, off, np.ascontiguousarray(fact, np.float32),
            np.ascontiguousarray(feature_idx, np.uint32), np.ascontiguousarray(di, np.float32),
            np.ascontiguousarray(dj, np.float32)]
    ptrs = [x.ctypes.data for x in arrs]
    buf = np.frombuffer(carry, dtype=np.uint8)
    fptr = buf.ctypes.data if buf.size else None
    n = C.c_uint64()
    need = int(L.lfr_wire_encode_solution_carried(len(image_names), *ptrs, fptr, buf.size, None, 0, C.byref(n)))
    if need < 0:
        if len(set(image_names)) != len(image_names):
            raise ValueError("repeated image names")
        raise ParseError("Failed to parse proto object.")
    out = np.zeros(max(need, 1), np.uint8)
    got = L.lfr_wire_encode_solution_carried(len(image_names), *ptrs, fptr, buf.size, out.ctypes.data, need, C.byref(n))
    assert got == need
    return out[:need].tobytes(), int(n.value)


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


def join_solution(data: bytes, image_names: List[str], node_image: np.ndarray, node_feat: np.ndarray,
                  entries: bool = False):
    """Start positions of a scene's nodes from the SolutionFile `data` (lfr_wire_join_solution,
    include/lfr_wire.h): images matched by name bytes (`image_names` by image id), displacements by
    feature; the last Image message with a name wins, and within it the last displacement of a feature.
    Returns (positions [N, 2] float64, 0 where a node has no entry; number of nodes started), and with
    `entries` also has_entry [N] bool, which nodes have an entry (lfr_wire_join_solution_entries).  Raises
    ParseError on bytes the decoder rejects."""
    L = _lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    blob, off = _names_blob(list(image_names))
    img = np.ascontiguousarray(node_image, dtype=np.uint32).reshape(-1)
    feat = np.ascontiguousarray(node_feat, dtype=np.uint32).reshape(-1)
    N = int(img.shape[0])
    pos = np.zeros((N, 2), np.float64)
    n = C.c_uint64()
    args = [buf.ctypes.data if buf.size else None, buf.size, len(image_names), blob.ctypes.data, off.ctypes.data, N,
            img.ctypes.data if N else None, feat.ctypes.data if N else None, pos.ctypes.data if N else None, C.byref(n)]
    if entries:
        has = np.zeros(N, np.uint8)
        rc = L.lfr_wire_join_solution_entries(*args, has.ctypes.data if N else None)
    else:
        rc = L.lfr_wire_join_solution(*args)
    if rc != 0:
        raise ParseError("Failed to parse proto object.")
    return (pos, int(n.value), has.astype(bool)) if entries else (pos, int(n.value))


def update_solution(data: bytes, image_names: List[str], node_image: np.ndarray, node_feat: np.ndarray,
                    node_comp: np.ndarray, n_components: int):
    """The host form of Plan.update_solution (lfr_wire_update_solution, include/lfr_wire.h): a component
    (node_comp, lfr_problem.comp) is touched when one of its nodes has no entry in `data` under the rule of
    join_solution.  Returns (positions [N, 2] float64: the entry of a held node, else 0; held [N] bool: entry
    AND component not touched; number of held nodes; number of touched components).  Raises ParseError on
    bytes the decoder rejects, ValueError on a component id out of range."""
    L = _lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    blob, off = _names_blob(list(image_names))
    img = np.ascontiguousarray(node_image, dtype=np.uint32).reshape(-1)
    feat = np.ascontiguousarray(node_feat, dtype=np.uint32).reshape(-1)
    comp = np.ascontiguousarray(node_comp, dtype=np.uint32).reshape(-1)
    N = int(img.shape[0])
    if N and int(comp.max()) >= n_components:
        raise ValueError("a component id is out of range")
    pos = np.zeros((N, 2), np.float64)
    held = np.zeros(N, np.uint8)
    n = C.c_uint64()
    t = C.c_uint32()
    rc = L.lfr_wire_update_solution(buf.ctypes.data if buf.size else None, buf.size, len(image_names), blob.ctypes.data,
                                    off.ctypes.data, N, img.ctypes.data if N else None, feat.ctypes.data if N else None,
                                    comp.ctypes.data if N else None, int(n_components), pos.ctypes.data if N else None,
                                    held.ctypes.data if N else None, C.byref(n), C.byref(t))
    if rc != 0:
        raise ParseError("Failed to parse proto object.")
    return pos, held.astype(bool), int(n.value), int(t.value)


def update_solution_since(data: bytes, p, previous: MatchSet):
    """The host form of Plan.update_solution(previous=...) (lfr_wire_update_solution_since, include/lfr_host.h):
    update_solution() on Problem `p` (its reference is_root), where a component is also touched when it is not
    unchanged since the graph stage over every pair of `previous` (the MatchingFile that produced `data`; the
    rule is in include/lfr_graph.h).  Returns (positions [N, 2], held [N] bool, held nodes, touched components,
    changed components).  Raises ParseError on bytes the decoder rejects, RuntimeError when the arrays or the
    earlier stage are rejected."""
    from .capi import Library
    from .graph import HostInput, host_input_arrays
    L = _lib()
    g = p.graph
    s, keep = Library.marshal(p)
    buf = np.frombuffer(data, dtype=np.uint8)
    blob, off = _names_blob(list(g.image_names))
    pblob, poff = _names_blob(list(previous.image_names))
    _, arrs = host_input_arrays(previous)
    inp = HostInput(n_pairs=previous.n_pairs, n_matches=previous.n_matches, n_images=len(previous.image_names),
                    **{k: (v.ctypes.data if v.size else None) for k, v in arrs.items()})
    img = np.ascontiguousarray(g.node_image, dtype=np.uint32).reshape(-1)
    feat = np.ascontiguousarray(g.node_feat, dtype=np.uint32).reshape(-1)
    N = int(img.shape[0])
    pos = np.zeros((N, 2), np.float64)
    held = np.zeros(N, np.uint8)
    n, t, ch = C.c_uint64(), C.c_uint32(), C.c_uint32()
    if not _solution_parses(data):  # told apart from the other refusals
        raise ParseError("Failed to parse proto object.")
    rc = L.lfr_wire_update_solution_since(buf.ctypes.data if buf.size else None, buf.size, len(g.image_names),
                                          blob.ctypes.data, off.ctypes.data, C.addressof(s),
                                          img.ctypes.data if N else None, feat.ctypes.data if N else None,
                                          C.addressof(inp), pblob.ctypes.data, poff.ctypes.data,
                                          pos.ctypes.data if N else None, held.ctypes.data if N else None,
                                          C.byref(n), C.byref(t), C.byref(ch))
    del keep, arrs
    if rc != 0:
        raise RuntimeError("lfr_wire_update_solution_since failed (%d)" % rc)
    return pos, held.astype(bool), int(n.value), int(t.value), int(ch.value)


def _solution_parses(data: bytes) -> bool:
    """Whether the SolutionFile decoder accepts `data`."""
    L = _lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    ni, nd = C.c_uint64(), C.c_uint64()
    return L.lfr_wire_decode_solution(buf.ctypes.data if buf.size else None, buf.size, C.byref(ni), C.byref(nd),
                                      *([None] * 7)) == 0


RECORD_MAGIC = b"LFRPREC1"


def record_is_valid(record: bytes) -> bool:
    """Whether `record` is a well-formed problem record (include/lfr_graph.h): the magic "LFRPREC1", the length
    16 + 16 C for its count C, and the C digests in ascending (d0, d1) order."""
    if len(record) < 16 or record[:8] != RECORD_MAGIC:
        return False
    n = int.from_bytes(record[8:16], "little")
    if len(record) != 16 + 16 * n:
        return False
    d = np.frombuffer(record, dtype="<u8", offset=16).reshape(-1, 2)
    if n < 2:
        return True
    a0, a1, b0, b1 = d[:-1, 0], d[:-1, 1], d[1:, 0], d[1:, 1]
    return bool(np.all((b0 > a0) | ((b0 == a0) & (b1 >= a1))))


def _record_args(p, image_names):
    from .capi import Library
    g = p.graph
    s, keep = Library.marshal(p)
    blob, off = _names_blob(list(g.image_names if image_names is None else image_names))
    img = np.ascontiguousarray(g.node_image, dtype=np.uint32).reshape(-1)
    feat = np.ascontiguousarray(g.node_feat, dtype=np.uint32).reshape(-1)
    return s, keep, blob, off, img, feat


def problem_record(p, image_names=None) -> bytes:
    """The problem record of Problem `p` on the host (lfr_host_problem_record, include/lfr_host.h; the record is
    stated in include/lfr_graph.h), byte for byte Plan.problem_record().  `p.is_root` must be the reference's
    is_root, as build_problem() leaves it.  `image_names` by image id (default: p.graph.image_names)."""
    L = _lib()
    s, keep, blob, off, img, feat = _record_args(p, image_names)
    N = int(img.shape[0])
    args = (C.addressof(s), img.ctypes.data if N else None, feat.ctypes.data if N else None, len(off) - 1,
            blob.ctypes.data, off.ctypes.data)
    need = L.lfr_host_problem_record(*args, None, 0)
    if need < 0:
        raise RuntimeError("lfr_host_problem_record failed (%d)" % need)
    out = np.empty(max(int(need), 1), np.uint8)
    got = L.lfr_host_problem_record(*args, out.ctypes.data, int(need))
    del keep
    if got != need:
        raise RuntimeError("lfr_host_problem_record failed (%d)" % got)
    return out[:need].tobytes()


def update_solution_since_record(data: bytes, p, record: bytes):
    """The host form of Plan.update_solution(previous_record=...) (lfr_wire_update_solution_since_record,
    include/lfr_host.h): update_solution_since() with the earlier run's problem record in place of its
    MatchingFile.  Returns (positions [N, 2], held [N] bool, held nodes, touched components, changed
    components).  Raises ParseError on SolutionFile bytes the decoder rejects, ValueError on a malformed
    record, RuntimeError when the arrays are rejected."""
    L = _lib()
    if not record_is_valid(bytes(record)):
        raise ValueError("malformed problem record")
    if not _solution_parses(data):
        raise ParseError("Failed to parse proto object.")
    s, keep, blob, off, img, feat = _record_args(p, None)
    buf = np.frombuffer(data, dtype=np.uint8)
    rec = np.frombuffer(bytes(record), dtype=np.uint8)
    N = int(img.shape[0])
    pos = np.zeros((N, 2), np.float64)
    held = np.zeros(N, np.uint8)
    n, t, ch = C.c_uint64(), C.c_uint32(), C.c_uint32()
    rc = L.lfr_wire_update_solution_since_record(buf.ctypes.data if buf.size else None, buf.size, len(off) - 1,
                                                 blob.ctypes.data, off.ctypes.data, C.addressof(s),
                                                 img.ctypes.data if N else None, feat.ctypes.data if N else None,
                                                 rec.ctypes.data, rec.size, pos.ctypes.data if N else None,
                                                 held.ctypes.data if N else None, C.byref(n), C.byref(t), C.byref(ch))
    del keep
    if rc != 0:
        raise RuntimeError("lfr_wire_update_solution_since_record failed (%d)" % rc)
    return pos, held.astype(bool), int(n.value), int(t.value), int(ch.value)


def group_arrays(blobs):
    """The (pointer array, length array, keep-alive list) of a C call's per-group byte buffers (files[], file_len[]
    or records[], record_len[]): a NULL pointer where `blobs[g]` is None."""
    keep = [None if b is None else np.frombuffer(bytes(b) or b"\0", dtype=np.uint8) for b in blobs]
    ptrs = (C.c_void_p * max(len(blobs), 1))(*[None if k is None else k.ctypes.data for k in keep])
    lens = np.array([0 if b is None else len(b) for b in blobs] or [0], np.uint64)
    return ptrs, lens, keep


def update_solution_groups(solutions, p, image_group, records=None):
    """The host form of Plan.update_solution_groups (lfr_wire_update_solution_groups, include/lfr_host.h): every
    scene g of Problem `p` (image id k in scene image_group[k]) updated as its own run from solutions[g]
    (SolutionFile bytes, or None: every component of the scene is touched) and, where records[g] is not None, against
    that earlier problem record.  Returns (positions [N, 2], held [N] bool, held nodes, touched components, changed
    components).  Raises ValueError on a malformed record, ParseError on a SolutionFile the decoder rejects."""
    L = _lib()
    G = len(solutions)
    records = [None] * G if records is None else list(records)
    for r in records:
        if r is not None and not record_is_valid(bytes(r)):
            raise ValueError("malformed problem record")
    for sol in solutions:
        if sol is not None and not _solution_parses(bytes(sol)):
            raise ParseError("Failed to parse proto object.")
    s, keep, blob, off, img, feat = _record_args(p, None)
    group = np.ascontiguousarray(image_group, dtype=np.uint32).reshape(-1)
    fptr, flen, fkeep = group_arrays(solutions)
    rptr, rlen, rkeep = group_arrays(records)
    N = int(img.shape[0])
    pos = np.zeros((N, 2), np.float64)
    held = np.zeros(N, np.uint8)
    n, t, ch = C.c_uint64(), C.c_uint32(), C.c_uint32()
    rc = L.lfr_wire_update_solution_groups(len(off) - 1, blob.ctypes.data, off.ctypes.data,
                                           group.ctypes.data if group.size else None, G, fptr, flen.ctypes.data, rptr,
                                           rlen.ctypes.data, C.addressof(s), img.ctypes.data if N else None,
                                           feat.ctypes.data if N else None, pos.ctypes.data if N else None,
                                           held.ctypes.data if N else None, C.byref(n), C.byref(t), C.byref(ch))
    del keep, fkeep, rkeep
    if rc != 0:
        raise RuntimeError("lfr_wire_update_solution_groups failed (%d)" % rc)
    return pos, held.astype(bool), int(n.value), int(t.value), int(ch.value)


def problem_record_groups(p, image_group, n_groups: int) -> List[bytes]:
    """The problem record of every scene g < n_groups of Problem `p` on the host (lfr_host_problem_record_groups,
    include/lfr_host.h), each byte for byte problem_record() of the scene's own run and Plan.problem_record_groups()."""
    L = _lib()
    s, keep, blob, off, img, feat = _record_args(p, None)
    group = np.ascontiguousarray(image_group, dtype=np.uint32).reshape(-1)
    goff = np.zeros(n_groups + 1, np.uint64)
    N = int(img.shape[0])
    args = (C.addressof(s), img.ctypes.data if N else None, feat.ctypes.data if N else None, len(off) - 1,
            blob.ctypes.data, off.ctypes.data, group.ctypes.data if group.size else None, n_groups)
    cap = 16 * (n_groups + int(p.n_components))
    out = np.empty(max(cap, 1), np.uint8)
    got = L.lfr_host_problem_record_groups(*args, out.ctypes.data, cap, goff.ctypes.data)
    del keep
    if got != cap:
        raise RuntimeError("lfr_host_problem_record_groups failed (%d)" % got)
    data = out[:cap].tobytes()
    return [data[int(goff[g]):int(goff[g + 1])] for g in range(n_groups)]
