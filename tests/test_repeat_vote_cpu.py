"""The test-time repeat vote without a GPU.

1. The torch CPU semantics the vote must reproduce (run/evaluate.py:400-417 and run/eval_mink.py:199-212 run them on the
   host): fp16 ``pred + store`` is one add rounded to nearest even, a zero store turns -0 into +0 and overflows to inf, and
   ``x.float().max(1)[1]`` takes the first NaN, else the first maximum.  The device's running argmax (csrc/vote.cuh),
   restated here with the same lane partitions as its two kernels, is checked against torch on rows full of ties, signed
   zeros, infinities and NaNs.
2. ``RepeatVote``'s host logic runs on CPU tensors with the library's entry points recorded instead of launched: one vote
   launch per scene per repeat, stores that never move, the begin/end protocol, and every refusal before any launch.
"""
import contextlib
import math
import types

import numpy as np
import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import repeat_eval
from tests import vote_oracle

NAN, INF = float('nan'), float('inf')


# ----------------------------------------------------------------------------------------------- torch CPU semantics
def _argmax(rows):
    return torch.tensor(rows, dtype=torch.float16).float().max(1)[1].tolist()


def test_torch_cpu_argmax_rules():
    assert _argmax([[1, 3, 3, 2]]) == [1]                       # first maximum
    assert _argmax([[-0.0, 0.0], [0.0, -0.0]]) == [0, 0]       # -0 == +0
    assert _argmax([[1, NAN, 5, NAN], [INF, NAN, 1, 1], [NAN, INF, NAN, 1]]) == [1, 1, 0]   # first NaN wins
    assert _argmax([[1, INF, 3, INF]]) == [1]                   # inf beats everything else
    assert _argmax([[-INF, -INF, -INF]]) == [0]
    assert _argmax([[-INF, -65504.0, -INF]]) == [1]


def test_torch_cpu_fp16_add():
    a = torch.tensor([-0.0, 60000.0, -60000.0, 1.0], dtype=torch.float16)
    z = a + 0.0                                                 # the reference's first `store = pred + store`
    assert z[0].item() == 0.0 and math.copysign(1.0, z[0].item()) == 1.0
    assert torch.equal((a + torch.zeros_like(a)).view(torch.int16), z.view(torch.int16))
    assert (a[1:2] + a[1:2]).item() == INF and (a[2:3] + a[2:3]).item() == -INF
    # correctly rounded: the fp64 sum of two fp16 values is exact, numpy's fp64 -> fp16 conversion rounds to nearest even
    rng = np.random.RandomState(0)
    bits = rng.randint(0, 1 << 16, size=(2, 400_000)).astype(np.uint16)
    x = bits.view(np.float16)
    fin = np.isfinite(x).all(0)
    x = x[:, fin]
    with np.errstate(over='ignore'):
        ref = (x[0].astype(np.float64) + x[1].astype(np.float64)).astype(np.float16)
    got = (torch.from_numpy(x[0].copy()) + torch.from_numpy(x[1].copy())).numpy()
    same = (ref.view(np.uint16) == got.view(np.uint16)) | (np.isnan(ref) & np.isnan(got))
    assert same.all(), int((~same).sum())


class _VoteArgmax:
    """csrc/vote.cuh, line by line"""

    def __init__(self):
        self.v, self.k = 0.0, -1

    def take(self, x, kx):
        if self.k < 0 or (not math.isnan(self.v) and (math.isnan(x) or x > self.v)):
            self.v, self.k = x, kx

    def merge(self, o):
        if o.k < 0:
            return
        if self.k < 0:
            self.v, self.k = o.v, o.k
            return
        n, on = math.isnan(self.v), math.isnan(o.v)
        if n or on:
            win = on and (not n or o.k < self.k)
        else:
            win = o.v > self.v or (o.v == self.v and o.k < self.k)
        if win:
            self.v, self.k = o.v, o.k


def _xor_reduce(states, width):
    o = 1
    while o < width:
        new = []
        for lane, s in enumerate(states):
            t = _VoteArgmax()
            t.v, t.k = s.v, s.k
            t.merge(states[lane ^ o])
            new.append(t)
        states, o = new, o * 2
    return states[0].k


def _device_argmax_simt(row):
    """k_vote_accumulate: lane l takes columns l, l + 32, ..., then a 32-lane xor tree"""
    st = [_VoteArgmax() for _ in range(32)]
    for k, x in enumerate(row):
        st[k % 32].take(x, k)
    return _xor_reduce(st, 32)


def _device_argmax_tc(row):
    """k_match_tc_vote: in pass p, lane q of a quad takes columns 96p + 8i + 2q + e (i < 12, e < 2), then a 4-lane tree"""
    st = [_VoteArgmax() for _ in range(4)]
    for p in range((len(row) + 95) // 96):
        for i in range(12):
            for q in range(4):
                for e in range(2):
                    k = 96 * p + 8 * i + 2 * q + e
                    if k < len(row):
                        st[q].take(row[k], k)
    return _xor_reduce(st, 4)


@pytest.mark.parametrize('k', [1, 16, 20, 21, 40, 80, 160, 200])
def test_device_argmax_rule_matches_torch(k):
    rng = np.random.RandomState(k)
    pool = np.array([0.0, -0.0, 1.0, -1.0, 2.0, INF, -INF, NAN, 65504.0], dtype=np.float16)
    rows = []
    for _ in range(300):
        mode = rng.randint(4)
        if mode == 0:
            r = pool[rng.randint(len(pool), size=k)]
        elif mode == 1:
            r = pool[rng.randint(len(pool) - 1, size=k)]               # no NaN
        elif mode == 2:
            r = rng.randint(-3, 4, size=k).astype(np.float16)          # many ties
        else:
            r = rng.randn(k).astype(np.float16)
        rows.append(r)
    rows = np.stack(rows)
    ref = torch.from_numpy(rows).float().max(1)[1].tolist()
    vals = rows.astype(np.float64).tolist()
    assert [_device_argmax_simt(r) for r in vals] == ref
    assert [_device_argmax_tc(r) for r in vals] == ref


def test_oracle_loops_restate_the_reference():
    g = torch.Generator().manual_seed(0)
    preds = [[(torch.randn(n, 5, generator=g) * 3).half() for n in (7, 4)] for _ in range(3)]
    gts = [torch.randint(0, 5, (7,), generator=g), torch.randint(0, 5, (4,), generator=g)]
    out = vote_oracle.evaluate_py(preds, gts, 5)
    for r in range(3):
        s = torch.cat(preds[r]) + (0.0 if r == 0 else out[r - 1]['store'])
        assert vote_oracle.same_bits(out[r]['store'], s)
    assert out[2]['store_logit'].tolist() == out[2]['store'].float().max(1)[1].tolist()


# ----------------------------------------------------------------------------------------------- recorded host logic
VOTES = ('osb_match_vote', 'osb_match_ensemble_vote', 'osb_vote_accumulate')


@pytest.fixture
def rec(monkeypatch):
    r = types.SimpleNamespace(calls=[])
    monkeypatch.setattr(C, 'call', lambda name, *a: r.calls.append((name, a)))
    monkeypatch.setattr(C, 'require_cuda', lambda t, what: None)
    monkeypatch.setattr(C, 'stream_ptr', lambda: None)
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    return r


def _val(p):
    return None if p is None else p.value


def check_plan(calls, n_scenes, n_repeats):
    """exactly one vote launch per scene per repeat, inside begin/end, each scene's store at the same address in every
    repeat.  ``calls`` = [('begin' | 'end', repeat) | (entry point, args)]; the store is the fourth argument from the end
    of every vote entry point."""
    stores0, per, repeat, done = None, None, -1, []
    for name, a in calls:
        if name == 'begin':
            assert per is None, "begin_repeat inside a repeat"
            per, repeat = [], a
        elif name == 'end':
            assert per is not None, "end_repeat outside a repeat"
            assert len(per) == len(set(per)), f"repeat {repeat} voted a store twice"
            assert len(per) == n_scenes, f"repeat {repeat} voted {len(per)} of {n_scenes} scenes"
            if stores0 is None:
                stores0 = set(per)
            assert set(per) == stores0, f"repeat {repeat}: a store moved"
            done.append(repeat)
            per = None
        elif name in VOTES:
            assert per is not None, f"{name} outside a repeat"
            per.append(_val(a[-4]))
    assert per is None and done == list(range(n_repeats))


def _distill_run(rec, n_scenes=3, n_repeats=3, drop=None):
    vote = repeat_eval.RepeatVote(20, device='cpu')
    g = torch.Generator().manual_seed(0)
    text = torch.zeros(20, 768, dtype=torch.float16)
    feats = [torch.zeros(50 + 10 * s, 768) for s in range(n_scenes)]
    log = []
    for r in range(n_repeats):
        vote.begin_repeat()
        log.append(('begin', r))
        for s in range(n_scenes):
            inv = torch.randint(0, feats[s].shape[0], (100 + s,), generator=g)
            n0 = len(rec.calls)
            vote.match_distill(s, feats[s], inv, text, gt=torch.zeros(100 + s, dtype=torch.int64))
            new = rec.calls[n0:]
            if drop == (r, s):
                new = [c for c in new if c[0] not in VOTES]
            log.extend(new)
        if drop is None or drop[0] != r:
            vote.end_repeat()
        else:
            vote._open = False
        log.append(('end', r))
    return vote, log


def test_one_vote_per_scene_per_repeat_and_stable_stores(rec):
    vote, log = _distill_run(rec)
    check_plan(log, 3, 3)
    names = [c[0] for c in log if c[0] not in ('begin', 'end')]
    assert names.count('osb_match_vote') == 9
    assert names.count('osb_confusion_accumulate') == 18                 # current and accumulated, per scene per repeat
    # every vote of scene s writes the same store, in every repeat
    stores = [_val(c[1][10]) for c in log if c[0] == 'osb_match_vote']
    assert stores[0:3] == stores[3:6] == stores[6:9] and len(set(stores[:3])) == 3
    assert [vote.scenes[s].store.data_ptr() for s in range(3)] == stores[:3]
    assert all(vote.scenes[s].store.dtype == torch.float16 and vote.scenes[s].store.shape == (100 + s, 20)
               for s in range(3))
    # each vote is followed by the two confusion updates of its labels, in the order current, accumulated
    for j, c in enumerate(log):
        if c[0] == 'osb_match_vote':
            assert [log[j + 1][0], log[j + 2][0]] == ['osb_confusion_accumulate'] * 2
            assert _val(log[j + 2][1][0]) == _val(c[1][12])              # the accumulated label feeds the second meter


def test_negative_control_dropped_vote_is_caught(rec):
    _, log = _distill_run(rec, drop=(1, 2))
    with pytest.raises(AssertionError, match='repeat 1 voted 2 of 3 scenes'):
        check_plan(log, 3, 3)


def test_ensemble_and_logits_launch_one_vote_each(rec):
    vote = repeat_eval.RepeatVote(20, device='cpu')
    text = torch.zeros(20, 512, dtype=torch.float16)
    for r in range(2):
        vote.begin_repeat()
        vote.match_ensemble(0, torch.zeros(30, 512), torch.zeros(30, 512, dtype=torch.float16), torch.zeros(40, dtype=torch.long), text)
        vote.end_repeat()
    names = [c[0] for c in rec.calls]
    assert names.count('osb_match_ensemble_vote') == 2 and names.count('osb_match_scores') == 4
    assert names.index('osb_match_ensemble_vote') > names.index('osb_match_scores')
    rec.calls.clear()
    mink = repeat_eval.RepeatVote(20, store_dtype=torch.float32, device='cpu')
    for r in range(2):
        mink.begin_repeat()
        mink.add_logits(0, torch.zeros(30, 20), torch.zeros(40, dtype=torch.long), gt=torch.zeros(40, dtype=torch.long))
        mink.end_repeat()
    assert [c[0] for c in rec.calls].count('osb_vote_accumulate') == 2
    assert mink.scenes[0].store.dtype == torch.float32 and mink.labels().shape == (40,)


def _refused(rec, fn, exc, match):
    n0 = len(rec.calls)
    with pytest.raises(exc, match=match):
        fn()
    assert len(rec.calls) == n0, "a refused call launched something"


def test_refusals_happen_before_any_launch(rec):
    text = torch.zeros(20, 768, dtype=torch.float16)
    feat = torch.zeros(10, 768)
    inv = torch.zeros(12, dtype=torch.long)
    vote = repeat_eval.RepeatVote(20, device='cpu')
    _refused(rec, lambda: vote.match_distill(0, feat, inv, text), RuntimeError, 'call begin_repeat')
    _refused(rec, lambda: vote.end_repeat(), RuntimeError, 'no repeat is open')
    vote.begin_repeat()
    _refused(rec, lambda: vote.begin_repeat(), RuntimeError, 'has not ended')
    vote.match_distill(0, feat, inv, text)
    vote.match_distill(1, feat, inv, text)
    _refused(rec, lambda: vote.match_distill(0, feat, inv, text), RuntimeError, 'already voted in repeat 0')
    _refused(rec, lambda: vote.add_logits(2, torch.zeros(10, 20), inv), TypeError, 'cannot add torch.float32')
    _refused(rec, lambda: vote.match_distill(2, feat, inv, torch.zeros(481, 768)), ValueError, r'K=481 outside 1\.\.480')
    _refused(rec, lambda: vote.match_ensemble(2, feat, feat.half(), inv, torch.zeros(481, 768)), ValueError,
             r'K=481 outside 1\.\.480')
    _refused(rec, lambda: vote.match_distill(2, feat, inv, text, gt=torch.zeros(5)), ValueError, 'gt has 5 labels')
    vote.end_repeat()
    vote.begin_repeat()
    _refused(rec, lambda: vote.match_distill(2, feat, inv, text), RuntimeError, 'scene 2 was not part of repeat 0')
    _refused(rec, lambda: vote.match_distill(0, feat, inv[:11], text), ValueError, '11 points x K=20 in repeat 1')
    _refused(rec, lambda: vote.match_distill(0, feat, inv, text[:16]), ValueError, 'K=16 in repeat 1')
    vote.match_distill(0, feat, inv, text)
    _refused(rec, lambda: vote.end_repeat(), RuntimeError, r'scene\(s\) \[1\] of repeat 0 were not voted in repeat 1')
    vote.match_distill(1, feat, inv, text)
    vote.end_repeat()
    with pytest.raises(TypeError, match='store_dtype'):
        repeat_eval.RepeatVote(20, store_dtype=torch.bfloat16, device='cpu')


def test_mapper_and_no_feature_override_reach_the_meters(rec, monkeypatch):
    seen = []
    monkeypatch.setattr(repeat_eval.metric.ConfusionMeter, 'update', lambda self, p, g: seen.append(p.clone()))
    vote = repeat_eval.RepeatVote(4, mapper=torch.arange(20) % 4, device='cpu')
    vote.begin_repeat()
    has_feat = torch.tensor([True, False, True, False])
    gt = torch.zeros(4, dtype=torch.long)
    sc = vote._slot('match_distill', 0, 4, 20, torch.float16, gt, has_feat)
    sc.label_acc.fill_(13)
    vote._count(0, torch.full((4,), 7), sc, gt, has_feat)
    assert seen[0].tolist() == [3, 256, 3, 256] and seen[1].tolist() == [1, 256, 1, 256]
    assert vote.scenes[0].label_acc.tolist() == [13] * 4                # the stored label stays unmapped


# the reference's labelsets as evaluate.py builds them: the class names, then the appended 'unlabeled'
_LABELSETS = {'scannet_3d': 20, 'matterport_3d': 21, 'matterport_3d_40': 40, 'matterport_3d_80': 80,
              'matterport_3d_160': 160, 'nuscenes_3d': 16}


@pytest.mark.parametrize('dataset', sorted(_LABELSETS))
def test_documented_binding_takes_the_metric_classes_from_the_dataset(dataset):
    n = _LABELSETS[dataset]
    labelset = [f'class {j}' for j in range(n)] + ['unlabeled']
    mapper = None
    if dataset == 'nuscenes_3d':                       # map_nuscenes_details: 43 detailed names -> 16 classes
        labelset = [f'detail {j}' for j in range(43)] + ['unlabeled']
        mapper = torch.arange(43) * 16 // 43
    vote = repeat_eval.RepeatVote(None, dataset=dataset, mapper=mapper, device='cpu')
    assert vote.num_classes == n and vote.meter_acc.C == n
    assert repeat_eval.RepeatVote(n, dataset=dataset, device='cpu').num_classes == n
    with pytest.raises(ValueError, match=f'num_classes={len(labelset)} disagrees with dataset'):
        repeat_eval.RepeatVote(len(labelset), dataset=dataset, mapper=mapper, device='cpu')
    with pytest.raises(ValueError, match='give num_classes or dataset'):
        repeat_eval.RepeatVote(None, device='cpu')


def test_logits_vote_takes_up_to_512_columns(rec):
    vote = repeat_eval.RepeatVote(20, store_dtype=torch.float32, device='cpu')
    vote.begin_repeat()
    vote.add_logits(0, torch.zeros(10, 512), torch.zeros(12, dtype=torch.long))
    _refused(rec, lambda: vote.add_logits(1, torch.zeros(10, 513), torch.zeros(12, dtype=torch.long)), ValueError,
             r'K=513 outside 1\.\.512')
    assert [c[0] for c in rec.calls] == ['osb_vote_accumulate']


def test_mapper_shorter_than_k_is_refused(rec):
    vote = repeat_eval.RepeatVote(16, mapper=torch.arange(20) % 16, device='cpu')
    vote.begin_repeat()
    _refused(rec, lambda: vote.match_distill(0, torch.zeros(10, 768), None, torch.zeros(21, 768)), ValueError,
             'the mapper has 20 entries')


def test_failed_launch_registers_no_scene(rec, monkeypatch):
    def fail_vote(name, *a):
        rec.calls.append((name, a))
        if name == 'osb_match_vote':
            raise RuntimeError('osb_match_vote failed: injected')
    monkeypatch.setattr(C, 'call', fail_vote)
    vote = repeat_eval.RepeatVote(20, device='cpu')
    vote.begin_repeat()
    with pytest.raises(RuntimeError, match='injected'):
        vote.match_distill(0, torch.zeros(10, 768), None, torch.zeros(20, 768))
    assert vote.scenes == {}
    vote.end_repeat()                                  # no scene was registered, so none is missing
