"""The validation tail of run/distill.py without a GPU: the fp64 restatement (tests/valce_ref.py) against torch's CPU
cross-entropy and the reference's own intersectionAndUnionGPU / AverageMeter arithmetic, the host replay of
``DeviceValidation.end`` (``distill.validation_result``) on fabricated per-scene state, its two-rank merge over gloo,
and the host-side argument checks of ``osb_match_ce``."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from openscene_b200 import distill
from tests import valce_ref as R


def _scene(n, k, seed, spread=4.0, ignore_frac=0.15):
    rng = np.random.default_rng(seed)
    s = (rng.standard_normal((n, k)) * spread).astype(np.float16)
    y = rng.integers(0, k, n)
    y[rng.random(n) < ignore_frac] = R.IGNORE
    return s, y


@pytest.mark.parametrize('k,spread', [(1, 1.0), (20, 4.0), (97, 0.5), (160, 8.0), (480, 3.0)])
def test_reference_terms_hold_torch_cpu_to_the_bound(k, spread):
    s, y = _scene(300, k, seed=k, spread=spread)
    y[y >= k] = R.IGNORE if k <= R.IGNORE else y[y >= k]
    lab = y != R.IGNORE
    t = R.logp_at_label(s, np.where(lab, y, 0))
    # torch's CPU kernel is not the CUDA one the device follows: it carries max + log(sum) in fp16 before the subtraction,
    # so it is held to the fp32 bound, half an fp16 ulp of T and one fp16 ulp of |max| + log(sum)
    f = s.astype(np.float64)
    m = f.max(axis=1)
    lse = np.log(np.exp(f - m[:, None]).sum(axis=1))
    bound = R.logp_bound(s, np.where(lab, y, 0)) + (0.5 * R.ulp16(t) + R.ulp16(np.abs(m) + lse)) * 1.001
    logp = F.log_softmax(torch.from_numpy(s), dim=1)
    assert logp.dtype == torch.float16
    got = logp.double().numpy()[np.arange(len(s)), np.where(lab, y, 0)]
    assert np.all(np.abs(got - t) <= bound), np.max(np.abs(got - t) - bound)
    # the scene loss of torch's fp16 cross-entropy against the fp64 mean of the reference terms
    ref = F.cross_entropy(torch.from_numpy(s), torch.from_numpy(y), ignore_index=R.IGNORE)
    v, _, terms = R.scene_loss(t, y)
    assert abs(float(ref) - v) <= R.loss_bound(terms, bound[lab])


def test_all_ignored_scene_is_nan_like_torch():
    s, _ = _scene(50, 20, seed=1)
    y = np.full(50, R.IGNORE)
    v, h, terms = R.scene_loss(np.zeros(50), y)
    assert len(terms) == 0 and np.isnan(v) and np.isnan(h)
    assert torch.isnan(F.cross_entropy(torch.from_numpy(s), torch.from_numpy(y), ignore_index=R.IGNORE))


def test_argmax_rule_matches_torch_on_finite_rows_and_single_nans():
    rng = np.random.default_rng(3)
    s = rng.integers(-3, 3, (400, 37)).astype(np.float32)        # many ties
    rows = rng.choice(400, 60, replace=False)
    s[rows, rng.integers(0, 37, 60)] = np.nan
    want = torch.from_numpy(s).max(1)[1].numpy()
    assert np.array_equal(R.argmax_nan_first(s), want)


@pytest.mark.parametrize('classes,k', [(20, 20), (13, 20), (160, 200), (2, 5)])
def test_device_counting_rule_equals_intersection_and_union(classes, k):
    rng = np.random.default_rng(classes)
    n = 5000
    pred = rng.integers(0, k, n)
    y = rng.integers(0, k, n)
    y[rng.random(n) < 0.15] = R.IGNORE
    got, bad = R.device_counts(pred, y, classes, k)
    assert bad == 0
    i, u, t = R.intersection_and_union(torch.from_numpy(pred), torch.from_numpy(y), classes)
    assert np.array_equal(got[0], i.numpy()) and np.array_equal(got[2], t.numpy())
    assert np.array_equal((got[1] + got[2] - got[0]).astype(np.float32), u.numpy())


def _fabricate(n_scenes, classes, seed, big=False):
    rng = np.random.default_rng(seed)
    hi = (1 << 23) if big else 5000                    # per-scene counts below 2^24; totals past 2^24 when big
    tgt = rng.integers(0, hi, (n_scenes, classes))
    inter = (tgt * rng.random((n_scenes, classes))).astype(np.int64)
    out = inter + rng.integers(0, hi // 4 + 1, (n_scenes, classes))
    tgt[:, rng.integers(0, classes)] = 0                 # a class absent everywhere: 0 / 1e-10
    inter[tgt == 0] = 0
    areas = np.stack([inter, out, tgt], axis=1).astype(np.int64)
    losses = (rng.random(n_scenes) * 5).astype(np.float16)
    return losses, areas


def _reference_scenes(losses, areas):
    scenes = []
    for s in range(len(losses)):
        i, o, t = (torch.from_numpy(areas[s, j]).float() for j in range(3))
        scenes.append((float(torch.tensor(losses[s]).item()), i.numpy(), (o + t - i).numpy(), t.numpy()))
    return scenes


@pytest.mark.parametrize('big', [False, True])
def test_replay_equals_the_reference_meters_bit_for_bit(big):
    losses, areas = _fabricate(40, 20, seed=7, big=big)
    if big:
        assert areas[:, 2].sum(0).max() > (1 << 24)       # float32 sums round past 2^24
    got = distill.validation_result(torch.from_numpy(losses), torch.from_numpy(areas),
                                    torch.zeros(40, dtype=torch.int32), weight=2)
    want = R.validate_tail(_reference_scenes(losses, areas), batch_size=2)
    assert R.same(got, want), (got, want)


def test_replay_refuses_bad_labels_and_names_the_first_scene():
    losses, areas = _fabricate(6, 5, seed=2)
    bad = torch.tensor([0, 0, 0, 2, 0, 1], dtype=torch.int32)
    with pytest.raises(IndexError, match='scene 3 '):
        distill.validation_result(torch.from_numpy(losses), torch.from_numpy(areas), bad)


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, case, ret):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        n = 9 if case == 'unequal' and rank == 1 else 8
        losses, areas = _fabricate(n, 12, seed=100 + rank, big=(case == 'big'))
        bad = torch.zeros(n, dtype=torch.int32)
        if case == 'bad' and rank == 1:
            bad[5] = 1
        try:
            ret[rank] = ('ok', distill.validation_result(torch.from_numpy(losses), torch.from_numpy(areas), bad, 3,
                                                         dist.group.WORLD))
        except (RuntimeError, IndexError) as e:
            ret[rank] = (type(e).__name__, str(e))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('case', ['equal', 'big', 'unequal', 'bad'])
def test_gloo_world2_merge_and_replay(case):
    world = 2
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), case, ret), nprocs=world, join=True)
    if case == 'unequal':
        assert ret[0][0] == ret[1][0] == 'RuntimeError' and 'same number of scenes' in ret[0][1]
        return
    if case == 'bad':
        assert ret[0][0] == ret[1][0] == 'IndexError'
        assert 'scene 5 ' in ret[1][1]
        return
    # the reference: per scene, the three vectors (union per rank) all-reduced, then the meters; the loss per rank
    for rank in range(world):
        per = [_fabricate(8, 12, seed=100 + r, big=(case == 'big')) for r in range(world)]
        scenes = []
        for s in range(8):
            vecs = [_reference_scenes(l[s:s + 1], a[s:s + 1])[0] for l, a in per]
            summed = [sum(v[j] for v in vecs) for j in (1, 2, 3)]
            scenes.append((vecs[rank][0], *summed))
        want = R.validate_tail(scenes, batch_size=3)
        assert ret[rank][0] == 'ok' and R.same(ret[rank][1], want), (rank, ret[rank], want)


def _abi(name, *args):
    from openscene_b200 import _cabi as C
    if not os.path.exists(C.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    L = C.lib()
    rc = getattr(L, name)(*args)
    return rc, (L.osb_last_error() or b'').decode()


def test_match_ce_refuses_bad_arguments_on_the_host():
    P = 0x1000                                               # never dereferenced: every call must fail before a launch

    def call(k=20, classes=20, feat=P, text=P, label=P, loss=P, areas=P, bad=P, ws=P, ws_bytes=16, n_pts=100, c=768,
             lab64=1):
        return _abi('osb_match_ce', feat, 0, 10, c, None, n_pts, text, k, label, lab64, 255, classes, None, None, loss,
                    areas, bad, ws, ws_bytes, None)

    cases = {
        'K=0': call(k=0), 'K=481': call(k=481), 'K=-1': call(k=-1),
        'classes=0': call(classes=0), 'classes=-3': call(classes=-3), 'classes=513': call(classes=513),
        'width': call(c=256), 'label dtype': call(lab64=2),
        'feat': call(feat=None), 'text': call(text=None), 'label': call(label=None), 'loss': call(loss=None),
        'areas': call(areas=None), 'bad': call(bad=None), 'ws': call(ws=None), 'ws small': call(ws_bytes=8),
    }
    for what, (rc, err) in cases.items():
        assert rc != 0 and err.startswith('osb_match_ce'), (what, rc, err)
    assert 'K_text=481' in cases['K=481'][1] and 'classes=0' in cases['classes=0'][1]
