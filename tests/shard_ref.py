"""NumPy restatement of the sharded index's merge (DESIGN.md, "Sharded index contract"), given each rank's results of
``search_ref`` / ``regions_ref`` on its own scenes and the directory.

A rank holds its scenes in ascending global id (``local_ids``), so its local row order is the global row order.  A
result slot's merge key is (order of its score, ~global row), global row = base[global id] + row within the scene,
padding slots below every real one; per query the m largest keys of all ranks win.  The per-scene outputs are placed by
global id, and the hit lists are sorted by (query, global row) with each hit's region rank taken through the merged list.

``rule`` selects deliberately wrong variants for the negative controls: 'tie_rank' (ties to the lower rank, then the
rank's own row), 'local_ids' (local scene ids in the keys and the outputs), 'no_base' (the row compared without its
scene's base), 'by_size' (regions ranked by size, then key), 'drop_sign' (the score taken from the key's order, which
maps -0 to +0) and 'add_order' (a rank keeps its scenes in the order they were added)."""
import numpy as np

MASK48 = (1 << 48) - 1


def local_ids(added, rule=None):
    """the local scene order of a rank that added the global ids ``added`` in this order"""
    return list(added) if rule == 'add_order' else sorted(added)


def shard(scores, off, ids, coords=None):
    """a rank's score matrix, scene offsets (and coordinates) for its scenes ``ids`` in this order"""
    off = np.asarray(off, np.int64)
    rows = np.concatenate([np.arange(off[g], off[g + 1]) for g in ids]) if len(ids) else np.zeros(0, np.int64)
    loff = np.concatenate([[0], np.cumsum([off[g + 1] - off[g] for g in ids])]).astype(np.int64)
    return scores[rows], loff, None if coords is None else np.asarray(coords)[rows]


def empty_search(nq, k, counted):
    """the results of a rank without scenes"""
    z = np.zeros((0, nq), np.int64)
    return dict(score=np.full((nq, k), -np.inf, np.float16), scene=np.full((nq, k), -1, np.int64),
                row=np.full((nq, k), -1, np.int64), scene_max=np.zeros((0, nq), np.float16), scene_argmax=z,
                scene_count=z if counted else None)


def empty_regions(nq, R):
    """the region results of a rank without scenes"""
    z = np.zeros(0, np.int64)
    return dict(score=np.full((nq, R), -np.inf, np.float16), scene=np.full((nq, R), -1, np.int64),
                row=np.full((nq, R), -1, np.int64), size=np.zeros((nq, R), np.int64),
                box_min=np.zeros((nq, R, 3), np.int32), box_max=np.zeros((nq, R, 3), np.int32),
                n_regions=np.zeros((0, nq), np.int64), hit_query=z, hit_scene=z, hit_row=z,
                hit_score=np.zeros(0, np.float16), hit_region=z)


def _order(bits):
    b = bits.astype(np.uint64)
    return np.where(b == 0x8000, np.uint64(0x8000), np.where(b & np.uint64(0x8000), ~b & np.uint64(0xffff),
                                                             b | np.uint64(0x8000)))


def keys(score, scene, row, ids, base, rank, rule=None):
    """uint64 merge keys of one rank's decoded slots (scene local, -1 padding) and their global scene ids"""
    bits = np.ascontiguousarray(score, np.float16).view(np.uint16)
    pad = scene < 0
    sc = np.where(pad, 0, scene)
    ids = np.asarray(ids, np.int64) if len(ids) else np.zeros(1, np.int64)
    g = np.where(pad, -1, ids[sc])
    if rule == 'local_ids':
        g = np.where(pad, -1, sc)
    if rule == 'no_base':
        grow = row
    elif rule == 'tie_rank':
        grow = (rank << 40) + np.where(pad, 0, np.asarray(base, np.int64)[np.where(pad, 0, ids[sc])]) + row
    else:
        grow = np.where(pad, 0, np.asarray(base, np.int64)[np.where(pad, 0, g)]) + row
    k = (_order(bits) << np.uint64(48)) | (~grow.astype(np.uint64) & np.uint64(MASK48))
    return np.where(pad | np.isnan(np.asarray(score, np.float16)), np.uint64(0), k), g


def _winners(klists):
    """klists uint64 [W, nq, m] -> positions w * m + j of the m largest per query (ties among zeros to the lower
    position)"""
    W, nq, m = klists.shape
    flat = klists.transpose(1, 0, 2).reshape(nq, W * m)
    pos = np.arange(W * m)
    return np.stack([np.lexsort((pos, ~flat[q]))[:m] for q in range(nq)]) if nq else np.zeros((0, m), np.int64)


def _take(cols, win):
    """cols [W, nq, m] -> [nq, m] at the winners"""
    W, nq, m = cols.shape
    flat = cols.transpose(1, 0, 2).reshape(nq, W * m)
    return np.take_along_axis(flat, win, 1)


def _place(per, parts_ids, S):
    """per-rank [S_w, nq] arrays -> [S, nq] by global id"""
    nq = next(p.shape[1] for p in per)
    out = np.zeros((S, nq), per[0].dtype)
    for p, ids in zip(per, parts_ids):
        for j, g in enumerate(ids):
            out[g] = p[j]
    return out


def merge_search(parts, base, rule=None):
    """parts: per rank (local ids, search_ref result on its scenes) -> the merged search_ref-shaped dict"""
    S = len(base)
    ks, cols = [], []
    for w, (ids, r) in enumerate(parts):
        k, g = keys(r['score'], r['scene'], r['row'], ids, base, w, rule)
        ks.append(k)
        bits = r['score'].view(np.uint16).astype(np.int64)
        if rule == 'drop_sign':
            bits = np.where(bits == 0x8000, 0, bits)
        cols.append(np.stack([g, r['row'], bits]))
    win = _winners(np.stack(ks))
    cols = np.stack(cols, 1)                                            # [3, W, nq, k]
    dec = [_take(c, win) for c in cols]
    ids_list = [p[0] for p in parts]
    out = dict(score=dec[2].astype(np.uint16).view(np.float16), scene=dec[0], row=dec[1],
               scene_max=_place([p[1]['scene_max'] for p in parts], ids_list, S),
               scene_argmax=_place([p[1]['scene_argmax'] for p in parts], ids_list, S),
               scene_count=None if parts[0][1]['scene_count'] is None else
               _place([p[1]['scene_count'] for p in parts], ids_list, S))
    return out


def merge_regions(parts, base, rule=None):
    """parts: per rank (local ids, regions_ref result on its scenes and coordinates) -> the merged regions_ref-shaped
    dict, hit list included"""
    S, W = len(base), len(parts)
    ks, cols = [], []
    for w, (ids, r) in enumerate(parts):
        k, g = keys(r['score'], r['scene'], r['row'], ids, base, w, rule)
        if rule == 'by_size':     # size above the key: the largest region first
            k = np.where(k > 0, (r['size'].astype(np.uint64) << np.uint64(40)) | (k >> np.uint64(24)), k)
        ks.append(k)
        bits = r['score'].view(np.uint16).astype(np.int64)
        if rule == 'drop_sign':
            bits = np.where(bits == 0x8000, 0, bits)
        cols.append(np.concatenate([np.stack([g, r['row'], r['size'], bits]), r['box_min'].transpose(2, 0, 1),
                                    r['box_max'].transpose(2, 0, 1)]))
    win = _winners(np.stack(ks))
    m = win.shape[1]
    cols = np.stack(cols, 1)                                            # [10, W, nq, R]
    dec = [_take(c, win) for c in cols]
    ids_list = [p[0] for p in parts]
    out = dict(score=dec[3].astype(np.uint16).view(np.float16), scene=dec[0], row=dec[1], size=dec[2],
               box_min=np.stack(dec[4:7], -1).astype(np.int32), box_max=np.stack(dec[7:10], -1).astype(np.int32),
               n_regions=_place([p[1]['n_regions'] for p in parts], ids_list, S))
    # hits: (query, global row) order; region rank through the winners
    hq, hg, hs, hr, hsc, hreg = [], [], [], [], [], []
    for w, (ids, r) in enumerate(parts):
        if not len(r['hit_query']):
            continue
        ids_a = np.asarray(ids, np.int64)
        g = ids_a[r['hit_scene']]
        hq.append(r['hit_query'])
        hg.append(np.asarray(base, np.int64)[g] + r['hit_row'])
        hs.append(g)
        hr.append(r['hit_row'])
        hsc.append(r['hit_score'].view(np.uint16))
        want = np.where(r['hit_region'] >= 0, w * m + r['hit_region'], -1)
        reg = np.full(len(want), -1, np.int64)
        for i, (q, t) in enumerate(zip(r['hit_query'], want)):
            if t >= 0:
                j = np.nonzero(win[q] == t)[0]
                reg[i] = j[0] if len(j) else -1
        hreg.append(reg)
    if hq:
        hq, hg = np.concatenate(hq), np.concatenate(hg)
        o = np.lexsort((hg, hq))
        out.update(hit_query=hq[o], hit_scene=np.concatenate(hs)[o], hit_row=np.concatenate(hr)[o],
                   hit_score=np.concatenate(hsc)[o].view(np.float16), hit_region=np.concatenate(hreg)[o])
    else:
        z = np.zeros(0, np.int64)
        out.update(hit_query=z, hit_scene=z, hit_row=z, hit_score=np.zeros(0, np.float16), hit_region=z)
    return out
