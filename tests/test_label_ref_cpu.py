"""The label restatement (tests/label_ref.py) against tests/topk_ref.py, torch's CPU argmax and brute forces over the labels
(per-scene bincounts and a breadth-first search per (scene, class)), on planted edge cases and against mutated rules; and
the C ABI's refusals of osb_match_topk_f8, osb_label_counts and osb_label_hits, in a child process (no GPU: they happen
before any CUDA call)."""
import json
import os
import subprocess
import sys
from collections import deque

import numpy as np
import pytest
import torch

from tests.label_ref import class_counts_ref, class_matrix, class_regions_ref, label_ref
from tests.search_ref import order_keys
from tests.topk_ref import topk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN, INF = np.float16(np.nan), np.float16(np.inf)


def _eq(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float16:
        return a.shape == b.shape and np.array_equal(a.view(np.uint16), b.view(np.uint16))
    return np.array_equal(a, b)


def _planted():
    """fp16 scores [N, K] of 5 scenes (one of 1 row) with ties, -0 / +0, NaN rows, inf, and coordinates"""
    s = np.array([
        [1, 3, 3, 0],                  # tie: column 1
        [-0.0, 0.0, -1, -2],           # -0 == +0: column 0, score -0
        [0.0, -0.0, -1, -2],           # column 0, score +0
        [NAN, 1, NAN, 2],              # first NaN: column 0
        [2, NAN, 5, 1],                # NaN ranks first: column 1
        [INF, 1, INF, 0],              # inf tie: column 0
        [-INF, -INF, -INF, -INF],      # all -inf: column 0
        [1, 2, 3, 3],                  # tie: column 2
        [0.5, 0.25, 0.75, 0.125],
        [NAN, NAN, NAN, NAN],
        [1, 4, 2, 0],
        [1, 4, 2, 0],
        [0, 0, 0, 0],
    ], np.float16)
    off = np.array([0, 3, 4, 8, 10, 13])
    xyz = np.array([[0, 0, 0], [1, 0, 0], [3, 0, 0],
                    [0, 0, 0],
                    [0, 0, 0], [1, 1, 1], [2, 2, 2], [5, 5, 5],
                    [0, 0, 0], [0, 0, 1],
                    [0, 0, 0], [1, 0, 0], [0, 2, 0]], np.int32)
    return s, off, xyz


def test_planted_labels():
    s, _, _ = _planted()
    lab, sc = label_ref(s)
    assert lab.tolist() == [1, 0, 0, 0, 1, 0, 0, 2, 2, 0, 1, 1, 0]
    assert sc[1].view(np.uint16) == 0x8000 and sc[2].view(np.uint16) == 0
    assert np.isnan(sc[3]) and np.isnan(sc[4]) and np.isnan(sc[9]) and np.isposinf(sc[5]) and np.isneginf(sc[6])


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_label_is_topk_one_and_torch_argmax(seed):
    rng = np.random.default_rng(seed)
    n, K = 4000, 37
    s = (rng.standard_normal((n, K)) * 4).astype(np.float16)        # fp16 rounding leaves many exact ties
    s[rng.random((n, K)) < 0.02] = np.float16(-0.0)
    s[rng.random((n, K)) < 0.02] = np.float16(0.0)
    s[rng.random((n, K)) < 0.01] = INF
    lab, sc = label_ref(s)
    tl, ts = topk(s, 1)
    assert np.array_equal(lab, tl[:, 0]) and _eq(sc, ts[:, 0])
    # on NaN-free rows: evaluate.py's torch.max(pred, 1)[1] (CPU)
    assert np.array_equal(lab, torch.from_numpy(s).float().max(1)[1].numpy())
    s[rng.random((n, K)) < 0.01] = NAN
    lab, sc = label_ref(s)
    tl, ts = topk(s, 1)
    assert np.array_equal(lab, tl[:, 0]) and _eq(sc, ts[:, 0])


def _brute_counts(lab, sc, off, classes, thr):
    S = len(off) - 1
    out = np.zeros((S, len(classes)), np.int64)
    for s in range(S):
        for r in range(off[s], off[s + 1]):
            for j, c in enumerate(classes):
                if lab[r] != c:
                    continue
                if thr is None or (not np.isnan(sc[r]) and float(sc[r]) >= float(np.float32(thr[j]))):
                    out[s, j] += 1
    return out


def _brute_regions(lab, sc, xyz, off, classes, thr, reach):
    """per class slot: the components (sets of global rows) by breadth-first search inside each scene"""
    comps = []
    for j, c in enumerate(classes):
        t = -np.inf if thr is None else thr[j]
        mine = []
        for s in range(len(off) - 1):
            rows = [r for r in range(off[s], off[s + 1])
                    if lab[r] == c and not np.isnan(sc[r]) and float(sc[r]) >= float(np.float32(t))]
            seen = set()
            for r0 in rows:
                if r0 in seen:
                    continue
                comp, todo = {r0}, deque([r0])
                seen.add(r0)
                while todo:
                    u = todo.popleft()
                    for v in rows:
                        if v not in seen and np.abs(xyz[u] - xyz[v]).max() <= reach:
                            seen.add(v)
                            comp.add(v)
                            todo.append(v)
                mine.append(frozenset(comp))
        comps.append(mine)
    return comps


def _ref_components(ref, off, m):
    grow = ref['hit_row'] + np.asarray(off)[ref['hit_scene']]
    out = []
    for j in range(m):
        sel = ref['hit_query'] == j
        groups = {}
        for r, g in zip(grow[sel], ref['hit_region'][sel]):
            groups.setdefault(g, set()).add(int(r))
        out.append(groups)
    return out


def _random_case(seed, n=600, K=9):
    rng = np.random.default_rng(seed)
    s = (rng.standard_normal((n, K)) * 2).astype(np.float16)
    s[rng.random((n, K)) < 0.01] = NAN
    s[rng.random((n, K)) < 0.02] = np.float16(-0.0)
    s[rng.random((n, K)) < 0.01] = INF
    s[:, K - 1] = s[:, 0]                         # class K-1 is absent: every tie with column 0 goes to 0
    cuts = np.sort(rng.choice(np.arange(1, n), 7, replace=False))
    off = np.concatenate([[0], cuts, [n - 1], [n]])            # a 1-row scene at the end
    xyz = np.concatenate([np.stack(np.unravel_index(rng.choice(9 ** 3, b - a, replace=False), (9,) * 3), 1)
                          for a, b in zip(off[:-1], off[1:])]).astype(np.int32)
    return s, off, xyz


@pytest.mark.parametrize('seed', [0, 1])
def test_counts_and_regions_against_brute_force(seed):
    s, off, xyz = _random_case(seed)
    lab, sc = label_ref(s)
    K = s.shape[1]
    classes = [K - 1, 2, 0, 5, 1]
    for thr in (None, [0.0, -1.0, 0.5, float('-inf'), 1.0]):
        got = class_counts_ref(lab, sc, off, classes, thr)
        assert np.array_equal(got, _brute_counts(lab, sc, off, classes, thr))
        assert got[:, 0].sum() == 0
        if thr is None:                                        # every row under its label, NaN scores included
            full = class_counts_ref(lab, sc, off, np.arange(K))
            assert np.array_equal(full.sum(1), np.diff(off))
            per = np.stack([np.bincount(lab[a:b], minlength=K) for a, b in zip(off[:-1], off[1:])])
            assert np.array_equal(full, per)
        for reach in (1, 2):
            ref = class_regions_ref(lab, sc, xyz, off, classes, thr, R=32, reach=reach)
            want = _brute_regions(lab, sc, xyz, off, classes, thr, reach)
            comps = _ref_components(ref, off, len(classes))
            for j in range(len(classes)):
                assert len(ref['hit_row'][ref['hit_query'] == j]) == sum(len(c) for c in want[j])
                listed = {frozenset(v) for g, v in comps[j].items() if g >= 0}
                assert listed <= set(want[j])
                assert len(listed) == min(32, len(want[j]))
                # the ranking: by the search key of the best hit
                keys = order_keys(class_matrix(lab, sc, classes))[:, j]
                best = sorted((max(keys[r] for r in c) for c in want[j]), reverse=True)[:32]
                got_best = [keys[ref['row'][j, i] + off[ref['scene'][j, i]]] for i in range(len(best))]
                assert got_best == best


def test_planted_counts_and_regions():
    s, off, xyz = _planted()
    lab, sc = label_ref(s)
    counts = class_counts_ref(lab, sc, off, [0, 1, 2, 3])
    assert counts.tolist() == [[2, 1, 0, 0], [1, 0, 0, 0], [2, 1, 1, 0], [1, 0, 1, 0], [1, 2, 0, 0]]
    # with a threshold NaN never counts (row 3 and row 9 are labelled 0 with NaN scores, row 4 is labelled 1)
    assert class_counts_ref(lab, sc, off, [0, 1], [-np.inf, -np.inf]).tolist() == \
        [[2, 1], [0, 0], [2, 0], [0, 0], [1, 2]]
    ref = class_regions_ref(lab, sc, xyz, off, [0, 1, 3], None, R=4, reach=1)
    # class 0: scene 2 rows 5 (inf), 6 touch and rank first; scene 0 rows 1 (-0), 2 (+0) are 2 apart, so two regions
    # tied at zero and ranked by row; scene 4 row 12 (+0) alone
    assert ref['size'][0].tolist() == [2, 1, 1, 1]
    assert ref['scene'][0].tolist() == [2, 0, 0, 4] and ref['row'][0].tolist() == [1, 1, 2, 2]
    assert ref['n_regions'][:, 0].tolist() == [2, 0, 1, 0, 1]
    # class 1 in scene 4: rows 10 and 11 touch; row 0 of scene 0; class 3 absent
    assert ref['size'][1].tolist()[:2] == [2, 1] and ref['size'][2].tolist() == [0, 0, 0, 0]
    assert (ref['scene'][2] == -1).all()


@pytest.mark.parametrize('rule', ['tie_high', 'second_best', 'nan_hit', 'merge_classes', 'cross_scene'])
def test_mutated_rules_fail(rule):
    s, off, xyz = _planted()
    lab, sc = label_ref(s)
    classes = [0, 1, 2]
    if rule in ('tie_high', 'second_best'):
        bl, bs = label_ref(s, rule)
        assert not (np.array_equal(lab, bl) and _eq(sc, bs))
        assert not np.array_equal(class_counts_ref(lab, sc, off, classes), class_counts_ref(bl, bs, off, classes))
    elif rule == 'nan_hit':
        thr = [-np.inf] * 3
        assert not np.array_equal(class_counts_ref(lab, sc, off, classes, thr),
                                  class_counts_ref(lab, sc, off, classes, thr, rule=rule))
    else:
        # rows 8, 9 of scene 3 touch; two classes side by side in one scene, and a region across scenes 0 / 1
        good = class_regions_ref(lab, sc, xyz, off, classes, None, R=8)
        bad = class_regions_ref(lab, sc, xyz, off, classes, None, R=8, rule=rule)
        assert any(not _eq(good[k], bad[k]) for k in ('size', 'n_regions', 'score', 'row', 'hit_region'))


_CHILD = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
from openscene_b200 import _cabi as C
L = C.lib()
out = {}
A = 1 << 20            # a 16-byte aligned non-NULL placeholder: never dereferenced, every call is refused first
def cls(*v):
    return (C.I64 * len(v))(*v)
def t(tag, codes=A, exp=A, n=10, c=768, text=A, K=20, topk=1, label=A):
    out[tag] = [L.osb_match_topk_f8(codes, exp, n, c, text, K, topk, None, label, None, None),
                (L.osb_last_error() or b'').decode()]
t('t_null_codes', codes=None); t('t_null_exp', exp=None); t('t_width', c=640); t('t_n0', n=0); t('t_K', K=0)
t('t_topk', topk=9); t('t_misaligned', codes=A + 8); t('t_null_label', label=None); t('t_n_big', n=1 << 31)
def c(tag, lab=A, sc=A, scene=A, n=10, S=2, K=20, classes=None, m=2, cnt=A, ws=A, wsb=1 << 30):
    classes = cls(1, 2) if classes is None else classes
    out[tag] = [L.osb_label_counts(lab, sc, scene, n, S, K, classes, m, None, cnt, ws, wsb, None),
                (L.osb_last_error() or b'').decode()]
c('c_K', K=0); c('c_m', m=0); c('c_m_big', m=21); c('c_n', n=0); c('c_S', S=11); c('c_null_lab', lab=None)
c('c_misaligned', lab=A + 4); c('c_class_range', classes=cls(1, 20)); c('c_class_neg', classes=cls(-1, 2))
c('c_dup', classes=cls(3, 3)); c('c_null_counts', cnt=None); c('c_ws', wsb=8); c('c_null_ws', ws=None)
c('c_too_many', n=1 << 30, S=1 << 22, K=64, m=64, classes=cls(*range(64)))
def h(tag, lab=A, n=10, S=2, K=200, classes=None, m=2, thr=A, cnt=A, nh=5, key=A, st=A, ws=A, wsb=1 << 30):
    classes = cls(1, 2) if classes is None else classes
    out[tag] = [L.osb_label_hits(lab, A, A, n, S, K, classes, m, thr, cnt, nh, key, A, st, ws, wsb, None),
                (L.osb_last_error() or b'').decode()]
h('h_m', m=97, classes=cls(*range(97))); h('h_hits', nh=0); h('h_null_thr', thr=None); h('h_null_counts', cnt=None)
h('h_null_key', key=None); h('h_misaligned', key=A + 4); h('h_dup', classes=cls(5, 5)); h('h_class', classes=cls(0, 200))
h('h_ws', wsb=16); h('h_S', S=0)
out['ws_counts_bad'] = [int(L.osb_label_counts_workspace_bytes(0, 1)), '']
out['ws_hits_bad'] = [int(L.osb_label_hits_workspace_bytes(20, 10, 2, 97)), '']
print('RESULT ' + json.dumps(out))
'''


def test_label_refusals_happen_on_the_host_with_a_message():
    p = subprocess.run([sys.executable, '-c', _CHILD, ROOT], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith('RESULT ')][-1][len('RESULT '):])
    expect = {'t_null_codes': 'NULL codes', 't_null_exp': 'NULL codes', 't_width': 'width', 't_n0': 'bad shape',
              't_K': 'K_text', 't_topk': 'topk', 't_misaligned': 'aligned', 't_null_label': 'NULL label',
              't_n_big': 'N=',
              'c_K': 'K=', 'c_m': 'm=', 'c_m_big': 'm=', 'c_n': 'N=', 'c_S': 'scenes', 'c_null_lab': 'NULL',
              'c_misaligned': 'misaligned', 'c_class_range': 'class 20', 'c_class_neg': 'class -1',
              'c_dup': 'class 3 listed twice', 'c_null_counts': 'counts', 'c_ws': 'workspace', 'c_null_ws': 'workspace',
              'c_too_many': 'exceed',
              'h_m': 'above 96', 'h_hits': 'n_hits', 'h_null_thr': 'NULL', 'h_null_counts': 'NULL', 'h_null_key': 'NULL',
              'h_misaligned': 'misaligned', 'h_dup': 'class 5 listed twice', 'h_class': 'class 200', 'h_ws': 'workspace',
              'h_S': 'scenes', 'ws_counts_bad': '', 'ws_hits_bad': ''}
    assert sorted(res) == sorted(expect)
    for tag, (rc, err) in res.items():
        if tag.startswith('ws_'):
            assert rc == 0, tag
            continue
        assert rc != 0, f"{tag}: accepted"
        assert expect[tag] in err, f"{tag}: {err!r}"
        assert err.startswith({'t': 'osb_match_topk_f8', 'c': 'osb_label_counts', 'h': 'osb_label_hits'}[tag[0]]), err


def test_python_refusals_before_any_launch():
    """SceneIndex's class arguments and refusals, checked on an object that never touches a device"""
    from openscene_b200.search import SceneIndex
    idx = SceneIndex.__new__(SceneIndex)
    for bad, msg in (([], 'no classes'), ([1, 1], 'listed twice'), ([0, 5], 'class 5 outside'), ([-1], 'class -1'),
                     ([1.5], 'integers'), ([True], 'integers'), ('ab', 'sequence'), (3, 'sequence'),
                     (torch.tensor([0.0]), 'integer CPU tensor')):
        with pytest.raises(ValueError, match=msg):
            idx._classes(bad, 5, 'class_counts')
    assert idx._classes(range(3), 5, 'x') == [0, 1, 2]
    assert idx._classes(torch.tensor([4, 0], dtype=torch.int32), 5, 'x') == [4, 0]
    assert idx._classes((np.int64(2),), 5, 'x') == [2]
    idx.vocab = None
    for what in ('labels', 'class_counts', 'class_regions'):
        with pytest.raises(RuntimeError, match='not labelled'):
            getattr(idx, what)(0) if what == 'labels' else getattr(idx, what)([0])
