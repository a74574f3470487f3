"""MatchSet — the content of a MatchingFile (types.proto:3-28) as flat arrays.

The reference keeps the parsed protobuf objects around (solve.cc:438-480); here
the same information is a handful of numpy arrays so that the host graph stage
and the packer never loop over matches in Python.

    image_names[i], pair_name1/2 : strings
    pair_img1/2[p]   : image id of each side of pair p (ids index image_names)
    pair_fact1/2[p]  : float32 `fact1` / `fact2` of the pair (types.proto:6,8)
    pair_ptr[p..p+1] : matches of pair p
    feat1/feat2[m]   : uint32 feature_idx1 / feature_idx2 (types.proto:11-12)
    sim[m]           : float32 similarity (types.proto:13)
    disp1/disp2[m]   : float32 [18] = 9 x (di, dj), grid order 3*i+j
                       (types.proto:20-21, compute_match_graph.py:175-187);
                       shorter lists are zero-padded like solve.cc:460-472.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List

import numpy as np


@dataclass
class MatchSet:
    image_names: List[str]
    pair_img1: np.ndarray
    pair_img2: np.ndarray
    pair_fact1: np.ndarray
    pair_fact2: np.ndarray
    pair_ptr: np.ndarray
    feat1: np.ndarray
    feat2: np.ndarray
    sim: np.ndarray
    disp1: np.ndarray
    disp2: np.ndarray
    meta: dict = field(default_factory=dict)

    @property
    def n_pairs(self) -> int:
        return int(self.pair_img1.shape[0])

    @property
    def n_matches(self) -> int:
        return int(self.feat1.shape[0])

    def validate(self) -> None:
        m = self.n_matches
        assert self.pair_ptr.shape == (self.n_pairs + 1,)
        assert int(self.pair_ptr[-1]) == m and int(self.pair_ptr[0]) == 0
        assert self.feat2.shape == (m,) and self.sim.shape == (m,)
        assert self.disp1.shape == (m, 18) and self.disp2.shape == (m, 18)
        assert self.disp1.dtype == np.float32 and self.disp2.dtype == np.float32
        assert self.sim.dtype == np.float32

    # ---- packed on-disk form (SURVEY 8f row 4: the producer can emit this next to,
    # or instead of, the protobuf and skip serialise -> parse) --------------------
    def save_npz(self, path: str) -> None:
        """Write the flat arrays as one .npz (fp32 flows, exactly the wire content)."""
        # names as a fixed-width unicode array: loadable with allow_pickle=False (an object array would
        # make `solve --matches_file X.npz` unpickle whatever file it is handed)
        np.savez(path, image_names=np.array(self.image_names, dtype=np.str_), pair_img1=self.pair_img1,
                 pair_img2=self.pair_img2, pair_fact1=self.pair_fact1, pair_fact2=self.pair_fact2,
                 pair_ptr=self.pair_ptr, feat1=self.feat1, feat2=self.feat2, sim=self.sim, disp1=self.disp1,
                 disp2=self.disp2)

    @staticmethod
    def load_npz(path: str) -> "MatchSet":
        z = np.load(path, allow_pickle=False)
        ms = MatchSet(image_names=[str(x) for x in z["image_names"].tolist()],
                      pair_img1=z["pair_img1"].astype(np.int64), pair_img2=z["pair_img2"].astype(np.int64),
                      pair_fact1=z["pair_fact1"].astype(np.float32), pair_fact2=z["pair_fact2"].astype(np.float32),
                      pair_ptr=z["pair_ptr"].astype(np.int64), feat1=z["feat1"].astype(np.uint32),
                      feat2=z["feat2"].astype(np.uint32), sim=z["sim"].astype(np.float32),
                      disp1=z["disp1"].astype(np.float32), disp2=z["disp2"].astype(np.float32))
        ms.validate()
        return ms

    def without_images(self, banned) -> "MatchSet":
        """Drop every pair touching a banned image (solve.cc:444-446)."""
        banned = set(banned)
        if not banned:
            return self
        keep = np.array([
            (self.image_names[a] not in banned) and (self.image_names[b] not in banned)
            for a, b in zip(self.pair_img1.tolist(), self.pair_img2.tolist())
        ], dtype=bool) if self.n_pairs else np.zeros(0, dtype=bool)
        return self.select_pairs(np.nonzero(keep)[0])

    def select_pairs(self, idx: np.ndarray) -> "MatchSet":
        idx = np.asarray(idx, dtype=np.int64)
        counts = (self.pair_ptr[1:] - self.pair_ptr[:-1])[idx]
        new_ptr = np.zeros(idx.shape[0] + 1, dtype=np.int64)
        np.cumsum(counts, out=new_ptr[1:])
        if idx.shape[0]:
            sel = np.concatenate([np.arange(self.pair_ptr[p], self.pair_ptr[p + 1]) for p in idx.tolist()]) \
                if counts.sum() else np.zeros(0, dtype=np.int64)
        else:
            sel = np.zeros(0, dtype=np.int64)
        sel = sel.astype(np.int64)
        return MatchSet(
            image_names=self.image_names,
            pair_img1=self.pair_img1[idx], pair_img2=self.pair_img2[idx],
            pair_fact1=self.pair_fact1[idx], pair_fact2=self.pair_fact2[idx],
            pair_ptr=new_ptr,
            feat1=self.feat1[sel], feat2=self.feat2[sel], sim=self.sim[sel],
            disp1=self.disp1[sel], disp2=self.disp2[sel], meta=dict(self.meta),
        )

    def query_subscenes(self, query_images, banned_images=(), joint=False):
        """--query_images: (the pairs of every query group's sub-scene as one MatchSet, image_group).
        A group is one query; with `joint` (--joint_queries) it is a connected component of the queries under
        the kept pairs that name two of them, with or without matches.  After the banned images are dropped,
        a pair that names a query image belongs to that query's group's sub-scene and a pair that names none
        is dropped; each sub-scene gets its own id for every image it holds, in order of first appearance, so
        the sub-scenes share no node.  image_names of the result repeat a database image's name once per
        sub-scene; image_group[id] is the sub-scene (the group's lowest query image id in `self`).  Without
        `joint`, raises ValueError for a pair that names two queries."""
        queries = set(query_images)
        ms = self.without_images(banned_images)
        is_q = [n in queries for n in ms.image_names]
        pairs = list(zip(ms.pair_img1.tolist(), ms.pair_img2.tolist()))
        # the group of every query image: a union-find rooted at the group's lowest image id, run over all
        # pairs before any id is handed out (a later pair can merge two groups that already hold ids)
        group_of = list(range(len(ms.image_names)))

        def find(x):
            while group_of[x] != x:
                group_of[x] = group_of[group_of[x]]
                x = group_of[x]
            return x

        for a, b in pairs:
            if is_q[a] and is_q[b]:
                if not joint:
                    raise ValueError("the pair '%s' - '%s' names two query images" % (ms.image_names[a], ms.image_names[b]))
                ra, rb = find(a), find(b)
                group_of[max(ra, rb)] = min(ra, rb)
        keep = [p for p, (a, b) in enumerate(pairs) if is_q[a] or is_q[b]]
        return _sub_scenes(ms, keep, [find(a if is_q[a] else b) for a, b in (pairs[p] for p in keep)])

    def listed_pair_index(self, lines) -> np.ndarray:
        """--listed_pairs: the index of the pair that each line (name1, name2) of a match list names, in line
        order: the first pair whose image_name1 is name1 and image_name2 is name2 exactly.  A repeated line
        gives its pair again.  Raises UnheldPairError for the first line whose pair the set does not hold (a
        pair held only the other way round is not that pair: the network computes each direction on its own
        crops)."""
        first = {}
        for p, (a, b) in enumerate(zip(self.pair_img1.tolist(), self.pair_img2.tolist())):
            first.setdefault((self.image_names[a], self.image_names[b]), p)
        idx = []
        for k, (n1, n2) in enumerate(lines, 1):
            p = first.get((n1, n2))
            if p is None:
                raise UnheldPairError(k, n1, n2, (n2, n1) in first)
            idx.append(p)
        return np.array(idx, dtype=np.int64)

    def select_listed_pairs(self, lines) -> "MatchSet":
        """The MatchingFile a run of the two-view network over the match list `lines` ((name1, name2) per line)
        writes, taken from this superset: one pair per line, in line order (listed_pair_index)."""
        return self.select_pairs(self.listed_pair_index(lines))

    @staticmethod
    def join_scenes(scenes: List["MatchSet"], banned_images=()):
        """--additional_scenes: (the kept pairs of all `scenes` as one MatchSet, image_group).  Scene s's pairs
        follow scene s-1's; the banned images (by name) are dropped from every scene; each scene gets its own
        id for every image it holds, in order of first appearance, by query_subscenes' rule with the scene
        index as the label, so scenes that reuse image names share no node and each sub-scene is what a run on
        that scene alone stages."""
        kept = [s.without_images(banned_images) for s in scenes] + [MatchSet.empty()]
        names, label, ptr, base, m0 = [], [], [np.zeros(1, np.int64)], 0, 0
        for k, s in enumerate(kept):
            names += s.image_names
            label += [k] * s.n_pairs
            ptr.append(s.pair_ptr[1:].astype(np.int64) + m0)
            m0 += s.n_matches
        offs = np.cumsum([0] + [len(s.image_names) for s in kept])
        cat = lambda f, dt: np.concatenate([getattr(s, f) for s in kept]).astype(dt)
        flat = MatchSet(names, np.concatenate([s.pair_img1.astype(np.int64) + o for s, o in zip(kept, offs)]),
                        np.concatenate([s.pair_img2.astype(np.int64) + o for s, o in zip(kept, offs)]),
                        cat("pair_fact1", np.float32), cat("pair_fact2", np.float32), np.concatenate(ptr),
                        cat("feat1", np.uint32), cat("feat2", np.uint32), cat("sim", np.float32),
                        cat("disp1", np.float32).reshape(-1, 18), cat("disp2", np.float32).reshape(-1, 18))
        return _sub_scenes(flat, list(range(flat.n_pairs)), label)

    @staticmethod
    def empty() -> "MatchSet":
        """A MatchingFile with no pair: what the reference reads when the matches file is missing."""
        return MatchSet([], np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32),
                        np.zeros(0, np.float32), np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32),
                        np.zeros(0, np.float32), np.zeros((0, 18), np.float32), np.zeros((0, 18), np.float32))

    @staticmethod
    def concatenate(parts: List["MatchSet"]) -> "MatchSet":
        """Concatenate the `.part.N` files of one matching file (solve.cc:416-424):
        image ids are re-interned on the union of names, order of first use."""
        names: List[str] = []
        index = {}
        img1, img2 = [], []
        for ms in parts:
            remap = np.zeros(len(ms.image_names), dtype=np.int64)
            used = np.zeros(len(ms.image_names), dtype=bool)
            used[ms.pair_img1] = True
            used[ms.pair_img2] = True
            # intern in order of first use inside this part
            order = []
            seen = set()
            for a, b in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist()):
                for i in (a, b):
                    if i not in seen:
                        seen.add(i)
                        order.append(i)
            for i in order:
                nm = ms.image_names[i]
                if nm not in index:
                    index[nm] = len(names)
                    names.append(nm)
                remap[i] = index[nm]
            img1.append(remap[ms.pair_img1])
            img2.append(remap[ms.pair_img2])
        ptrs = [np.zeros(1, dtype=np.int64)]
        off = 0
        for ms in parts:
            ptrs.append(ms.pair_ptr[1:].astype(np.int64) + off)
            off += ms.n_matches
        cat = lambda xs, dt: (np.concatenate(xs).astype(dt) if xs else np.zeros(0, dtype=dt))
        return MatchSet(
            image_names=names,
            pair_img1=cat(img1, np.int64), pair_img2=cat(img2, np.int64),
            pair_fact1=cat([ms.pair_fact1 for ms in parts], np.float32),
            pair_fact2=cat([ms.pair_fact2 for ms in parts], np.float32),
            pair_ptr=np.concatenate(ptrs),
            feat1=cat([ms.feat1 for ms in parts], np.uint32),
            feat2=cat([ms.feat2 for ms in parts], np.uint32),
            sim=cat([ms.sim for ms in parts], np.float32),
            disp1=(np.concatenate([ms.disp1 for ms in parts]) if parts else np.zeros((0, 18), np.float32)),
            disp2=(np.concatenate([ms.disp2 for ms in parts]) if parts else np.zeros((0, 18), np.float32)),
            meta=dict(parts[0].meta) if parts else {},
        )


class UnheldPairError(ValueError):
    """A match-list line whose pair the MatchingFile does not hold: `line` counts from 1; `reverse` says whether
    the file holds the pair the other way round."""

    def __init__(self, line: int, name1: str, name2: str, reverse: bool):
        super().__init__("line %d: the matches file holds no pair '%s' '%s'%s"
                         % (line, name1, name2, "; it holds only '%s' '%s'" % (name2, name1) if reverse else ""))
        self.line, self.name1, self.name2, self.reverse = line, name1, name2, reverse


def _sub_scenes(ms: MatchSet, keep, label):
    """The pairs `keep` of `ms` (in order), pair keep[k] in the sub-scene labelled label[k]: every sub-scene
    gets its own id for each image it holds, in order of first appearance.  Returns (the MatchSet, whose
    image_names repeat a name once per sub-scene that holds it, image_group[id] = the label)."""
    keep = np.array(keep, dtype=np.int64)
    img1, img2, orig_of, group = sub_scene_ids(ms.pair_img1[keep], ms.pair_img2[keep], label)
    out = ms.select_pairs(keep)
    out.image_names = [ms.image_names[i] for i in orig_of]
    out.pair_img1 = img1
    out.pair_img2 = img2
    return out, group


def sub_scene_ids(pair_img1, pair_img2, label):
    """The id rule of _sub_scenes on the pair level alone: pair k in the sub-scene label[k] gets, on each side,
    that sub-scene's id for the image, handed out in order of first appearance.  Returns (pair_img1, pair_img2,
    orig_of: the original image of every id, image_group: the label of every id)."""
    img1, img2, group, orig_of, ids = [], [], [], [], {}

    def sub(g, i):
        if (g, i) not in ids:
            ids[(g, i)] = len(orig_of)
            orig_of.append(i)
            group.append(g)
        return ids[(g, i)]

    for a, b, g in zip(np.asarray(pair_img1).tolist(), np.asarray(pair_img2).tolist(), list(label)):
        img1.append(sub(g, a))
        img2.append(sub(g, b))
    return (np.array(img1, dtype=np.int64), np.array(img2, dtype=np.int64), orig_of, np.array(group, dtype=np.uint32))
