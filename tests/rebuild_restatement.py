"""A numpy restatement of the topology rtb200_scene_rebuild builds on the GPU (DESIGN.md §4.8), written from the documented
rules and sharing no code with csrc/: the recentring offset g and the oversize threshold from cub's radix order of the
columns, frame membership and the always-list, the 64-bit keys (oversized bit | Morton code | index), the top-down split
(radix split points on the first 13 wide levels, three rounds of halving below) and the numbering by scans. rebuild()
returns a dict in the layout of ResidentScene.bvh_records(), with placeholder boxes and records that
test_scene_update_cpu.refit fills in. check_tree() holds every invariant of a rebuilt topology that the traversal, the refit
and the rebuild's own buffer sizes (rebuild_carve) rely on; it is used on the restatement and on the device's arrays. Both
take the leaf size of the library (RT_LEAF_K, bvh_records()["leaf_size"]) as an argument; the node width is fixed."""
import bisect

import numpy as np

from test_bvh_cpu import _exact_hits, _traverse
from test_scene_update_cpu import refit, same_bits, sphere_boxes

K = 8                               # the default build's leaf size (RT_LEAF_K)
WIDE = 8                            # node width
MAX_DEPTH = 21                      # wide levels the trace's node stack reserve allows
RADIX_LEVELS = 13                   # wide levels split at radix split points; halving below
ID_BITS = 26                        # sphere index bits of a key
OVERSIZE = 16.0                     # default RTB200_REBUILD_OVERSIZE
EMPTY, LEAF, SKIP_NODE, NO_SKIP = 0xFFFFFFFF, 0x80000000, 0x80000000, 0xFFFFFFFF
_TOP = np.uint64(1 << 63)


def radix_rank_keys(x):
    """cub::DeviceRadixSort's key of each double: the sign-flip map of the IEEE bits (negative: all bits flipped; otherwise
    the sign bit set), after cub has mapped -0.0 onto +0.0. So -0.0 and +0.0 rank equal and a NaN ranks by its sign bit,
    below -inf or above +inf."""
    u = np.ascontiguousarray(x, np.float64).view(np.uint64).copy()
    u[u == _TOP] = 0
    return np.where(u & _TOP, ~u, u | _TOP)


def radix_median(x):
    """Element len(x) // 2 of x sorted by cub's stable radix sort: equal keys (both zeros among them) keep input order."""
    return x[np.argsort(radix_rank_keys(x), kind="stable")[len(x) // 2]]


def morton_codes(q):
    """30-bit Morton codes of cells q [m, 3] (0..1023): bit b of x, y, z goes to bit 3b + 2, 3b + 1, 3b."""
    code = np.zeros(len(q), np.uint64)
    for b in range(10):
        for a in range(3):
            code |= ((q[:, a].astype(np.uint64) >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + 2 - a)
    return code


def sort_keys(c, r, oversize=OVERSIZE):
    """g, r_big, the always-list and the sorted keys of the in-frame spheres."""
    n = len(r)
    g = np.array([radix_median(c[:, a]) for a in range(3)])
    g = np.where(np.isfinite(g), g, 0.0)
    ra = np.abs(r)
    r_big = oversize * radix_median(ra) if oversize > 0 else np.inf
    lo_b, _ = sphere_boxes(c, r, g)
    inside = np.isfinite(lo_b[:, 0])
    ids = np.nonzero(inside)[0]
    x = c[ids] - g
    with np.errstate(invalid="ignore"):
        big = ra[ids] > r_big
    box = x[~big]
    if len(box):
        lo = box.min(axis=0)
        ext = max(0.0, *(box.max(axis=0) - lo))
    if len(box) and ext > 0.0:
        t = np.clip((x - lo) / ext * 1024.0, 0.0, 1023.0)
    else:
        t = np.zeros_like(x)
    keys = big.astype(np.uint64) << np.uint64(63) | morton_codes(t.astype(np.uint32)) << np.uint64(ID_BITS) | ids.astype(np.uint64)
    return g, r_big, np.nonzero(~inside)[0].astype(np.uint32), np.sort(keys)


def _prefix(keys, f, l):
    """Length of the common prefix of the keys at positions f and l (keys are distinct)."""
    return 64 - (keys[f] ^ keys[l]).bit_length()


def _split_point(keys, f, l):
    """Size of the left part of keys[f..l] cut at their highest differing bit: the keys with that bit clear."""
    b = (keys[f] ^ keys[l]).bit_length() - 1
    return bisect.bisect_left(keys, ((keys[f] >> b) | 1) << b, f, l + 1) - f


def _children(keys, level, f, cnt, k):
    ch = [(f, cnt)]
    if level < RADIX_LEVELS:
        while len(ch) < WIDE:
            best = None                                  # shortest common prefix, then the larger range
            for i, (cf, cc) in enumerate(ch):
                if cc > k:
                    rank = (_prefix(keys, cf, cf + cc - 1), -cc)
                    if best is None or rank < best[0]:
                        best = (rank, i)
            if best is None:
                break
            i = best[1]
            cf, cc = ch[i]
            left = _split_point(keys, cf, cf + cc - 1)
            ch[i:i + 1] = [(cf, left), (cf + left, cc - left)]
    else:
        for _ in range(3):
            for i in range(len(ch) - 1, -1, -1):         # right to left: the new right part is not revisited this round
                cf, cc = ch[i]
                if cc > k:
                    left = cc - cc // 2
                    ch[i:i + 1] = [(cf, left), (cf + left, cc - left)]
    return ch


def rebuild(c, r, oversize=OVERSIZE, leaf_size=K):
    """The topology the GPU rebuild of a library with leaves of `leaf_size` makes of spheres (c [n, 3], r [n]) in the
    layout of ResidentScene.bvh_records(), with lo/hi (+inf, -inf) everywhere, leaf records zero with nk = -inf in padding slots, and "level_count" (nodes per level,
    root first) and "r_big" for the tests. Levels are built until no node is left: a depth above MAX_DEPTH is reported,
    not cut."""
    k = leaf_size
    assert k % 2 == 0 and 2 <= k <= 32, k
    c = np.asarray(c, np.float64).reshape(-1, 3)
    r = np.asarray(r, np.float64)
    n = len(r)
    g, r_big, always, skeys = sort_keys(c, r, oversize) if n else (np.zeros(3), np.inf, np.zeros(0, np.uint32), np.zeros(0, np.uint64))
    keys = skeys.tolist()
    n_in = len(keys)
    rows, level_count, leaves = [], [], []           # rows: per node its 8 child words, leaves: (first, count, node, slot)
    tasks = [(0, n_in)] if n_in else []
    level = 0
    while tasks:
        base, nxt = len(rows), []
        for f, cnt in tasks:
            row = [EMPTY] * WIDE
            for s, (cf, cc) in enumerate(_children(keys, level, f, cnt, k)):
                if cc > k:
                    row[s] = base + len(tasks) + len(nxt)
                    nxt.append((cf, cc))
                else:
                    leaves.append((cf, cc, len(rows), s))
            rows.append(row)
        level_count.append(len(tasks))
        tasks, level = nxt, level + 1
    nn, depth = len(rows), len(level_count)
    leaves.sort()                                    # leaves are numbered by their first key position
    nl = len(leaves)
    child = np.array(rows, np.uint32).reshape(nn, WIDE)
    ids = (skeys & np.uint64((1 << ID_BITS) - 1)).astype(np.int64)
    leaf_id = np.full((nl, k), EMPTY, np.uint32)
    skip = np.full(max(n, 1), NO_SKIP, np.uint32)
    for leaf, (f, cnt, node, s) in enumerate(leaves):
        child[node, s] = LEAF | leaf
        m = np.sort(ids[f:f + cnt])
        leaf_id[leaf, :cnt] = m
        skip[m] = leaf * k + np.arange(cnt)
        if cnt == 1:
            skip[m[0]] = SKIP_NODE | (node * WIDE + s)
    leaf_rec = np.zeros((nl, k // 2, 2, 4), np.float32)
    for j in range(k):
        leaf_rec[:, j // 2, 1, 2 + j % 2] = np.where(leaf_id[:, j] == EMPTY, -np.inf, 0.0)
    starts = np.concatenate([[0], np.cumsum(level_count)]).astype(np.int64)
    level_nodes = np.concatenate([np.arange(starts[j], starts[j + 1]) for j in range(depth - 1, -1, -1)] or [np.zeros(0)])
    level_off = np.concatenate([[0], np.cumsum(level_count[::-1])])
    return {"n": n, "leaf_size": k, "recentre": g, "r_big": r_big, "always": always, "n_nodes": nn, "n_leaves": nl,
            "depth": depth, "level_count": level_count, "child": child, "leaf_id": leaf_id, "skip_pos": skip,
            "level_nodes": level_nodes.astype(np.uint32), "level_off": level_off.astype(np.uint32),
            "lo": np.full((nn, 3, WIDE), np.inf, np.float32), "hi": np.full((nn, 3, WIDE), -np.inf, np.float32),
            "leaf_rec": leaf_rec, "flat": np.zeros((max((n + 1) // 2, 1), 2, 4), np.float32)}


def filled(t, c, r):
    """t with the values the refit computes on it for spheres (c, r)."""
    return refit(t, np.asarray(c, np.float64).reshape(-1, 3), np.asarray(r, np.float64))


def skip_rule(t, n):
    """build_records' skip_pos rule on topology t: a member's leaf slot, or its parent slot when it is alone in its leaf."""
    skip = np.full(max(n, 1), NO_SKIP, np.uint32)
    ids = t["leaf_id"].ravel()
    k = np.nonzero(ids != EMPTY)[0]
    skip[ids[k]] = k
    for node in range(t["n_nodes"]):
        for s, ref in enumerate(t["child"][node]):
            if ref != EMPTY and ref & LEAF:
                m = t["leaf_id"][ref & 0x7FFFFFFF]
                if (m != EMPTY).sum() == 1:
                    skip[m[0]] = SKIP_NODE | (node * WIDE + s)
    return skip


def check_tree(t, c, r, rays=0, cam=None, seed=11, leaf_size=K):
    """Every invariant of a rebuilt topology t (a dict in the layout of ResidentScene.bvh_records()) with leaves of
    `leaf_size` for spheres (c, r): leaves of that size, each sphere in exactly one leaf or on the always-list, members in
    increasing index, padding records that never hit, the level order and its depth, children deeper than their parents,
    the skip_pos rule, the sizes rebuild_carve allocates (n_leaves <= n, n_nodes <= max(n, 1), at most
    n // (leaf_size + 1) + 1 inner nodes per level), and values equal to the numpy refit. With rays, the float32 traversal emulation must reach every sphere the exact f64 test accepts."""
    c = np.asarray(c, np.float64).reshape(-1, 3)
    r = np.asarray(r, np.float64)
    n = len(r)
    assert t["leaf_size"] == leaf_size and t["leaf_id"].shape == (t["n_leaves"], leaf_size), (t["leaf_size"], t["leaf_id"].shape)
    ids = t["leaf_id"].ravel()
    assert sorted(np.concatenate([ids[ids != EMPTY], t["always"]]).tolist()) == list(range(n))   # in exactly one leaf or always
    assert np.all(np.diff(t["always"].astype(np.int64)) > 0), "the always-list is in increasing index order"
    for leaf in range(t["n_leaves"]):
        m = t["leaf_id"][leaf]
        cnt = int((m != EMPTY).sum())
        assert cnt >= 1 and np.all(m[cnt:] == EMPTY) and np.all(np.diff(m[:cnt].astype(np.int64)) > 0), (leaf, m)
        nk = np.concatenate([t["leaf_rec"][leaf][:, 1, 2], t["leaf_rec"][leaf][:, 1, 3]]).reshape(2, -1).T.ravel()
        assert np.all(nk[cnt:] == -np.inf), "padding records must never hit"
    depth, nn = t["depth"], t["n_nodes"]
    assert depth <= MAX_DEPTH and len(t["level_off"]) == depth + 1 and t["level_off"][-1] == nn
    assert t["n_leaves"] <= n and nn <= max(n, 1)
    per_level = np.diff(t["level_off"].astype(np.int64))
    assert np.all(per_level >= 1) and np.all(per_level <= n // (leaf_size + 1) + 1), per_level
    assert sorted(t["level_nodes"].tolist()) == list(range(nn))
    level = np.empty(nn, np.int64)
    for k in range(depth):                                     # deepest first
        level[t["level_nodes"][t["level_off"][k]:t["level_off"][k + 1]]] = depth - 1 - k
    seen_nodes, seen_leaves = np.zeros(nn, int), np.zeros(t["n_leaves"], int)
    for node in range(nn):
        for s, ref in enumerate(t["child"][node]):
            if ref == EMPTY:
                assert np.all(t["lo"][node][:, s] == np.inf) and np.all(t["hi"][node][:, s] == -np.inf)
            elif ref & LEAF:
                seen_leaves[ref & 0x7FFFFFFF] += 1
            else:
                assert ref > node and level[ref] == level[node] + 1
                seen_nodes[ref] += 1
    if nn:
        assert level[0] == 0 and seen_nodes[0] == 0 and np.all(seen_nodes[1:] == 1) and np.all(seen_leaves == 1)
    assert np.array_equal(t["skip_pos"], skip_rule(t, n))
    b = dict(t)
    b["flat"] = np.zeros((max((n + 1) // 2, 1), 2, 4), np.float32)   # a hierarchy handle has no flat records
    want = refit(b, c, r)
    for key in ("lo", "hi", "leaf_rec"):
        assert same_bits(t[key], want[key]), key
    if rays and nn:
        return sound(t, c, r, rays, cam, seed)
    return 0


def sound(t, c, r, rays, cam, seed=11):
    """The float32 traversal emulation of test_bvh_cpu on the filled topology t reaches every sphere the exact f64 test
    accepts, on `rays` rays of test_scene_update_cpu._rays; returns how many exact hits were checked."""
    from test_scene_update_cpu import _rays
    rng = np.random.default_rng(seed)
    n_exact = 0
    for i, (o, d) in enumerate(_rays(c, r, np.asarray(cam, np.float64), rng, rays)):
        with np.errstate(all="ignore"):
            exact = _exact_hits(c, r, o, d)
        cand, _ = _traverse(t, o, d)
        missing = set(exact.tolist()) - cand
        assert not missing, (i, sorted(missing)[:10])
        n_exact += len(exact)
    return n_exact
