"""CPU side of the supervised validation tail (osb_ce_head_eval, train_mink.DeviceMinkValidation) and of the training meter
(train_mink.DeviceTrainMeter): the fp64 restatement against torch CPU, the host replays bit for bit against the reference's
meters, a gloo world-2 merge, and the host-side argument checks of the new entry point."""
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from openscene_b200 import train_mink
from tests import minkval_ref as MR
from tests import valce_ref as R


def _scene(n_rows, n_pts, c, seed, scale=3.0, bad=0, ignored=0.15):
    g = np.random.default_rng(seed)
    z = (g.standard_normal((n_rows, c)) * scale).astype(np.float32)
    inv = g.integers(0, n_rows, n_pts)
    y = g.integers(0, c, n_pts)
    y[g.random(n_pts) < ignored] = R.IGNORE
    if bad:
        y[g.choice(n_pts, bad, replace=False)] = g.choice([-1, c, c + 7, 1000], bad)
    return z, inv, y


@pytest.mark.parametrize('c', [1, 20, 33, 160])
def test_point_head_terms_against_torch_cpu(c):
    z, inv, y = _scene(500, 1700, c, seed=c)
    z[7] = np.nan                                                  # a NaN row: its first class wins, the loss is NaN
    z[9, c // 2] = np.nan
    z[11, :] = 0.5                                                 # every class ties: class 0
    loss, pred, counts, bad = MR.point_head(z, inv, y)
    zt = torch.from_numpy(z)[torch.from_numpy(inv)]
    yt = torch.from_numpy(y)
    assert bad == 0
    assert np.array_equal(pred, zt.max(1)[1].numpy())               # torch CPU's first NaN / first maximum
    i, u, t = R.intersection_and_union(torch.from_numpy(pred), yt, c)
    if c > 1:                                                      # histc(bins=1) counts over the data's own range
        assert np.array_equal(counts[0], i.numpy()) and np.array_equal(counts[2], t.numpy())
        assert np.array_equal(counts[1] + counts[2] - counts[0], u.numpy())
    # loss: NaN through the NaN rows as in torch; without them within the fp32 bound of torch's own sum
    tl = float(F.cross_entropy(zt, yt, ignore_index=R.IGNORE))
    hit = np.isin(inv, [7, 9])
    assert math.isnan(loss) == math.isnan(tl) == bool((hit & (y != R.IGNORE)).any())
    keep = ~hit
    loss, _, _, _ = MR.point_head(z, inv[keep], y[keep])
    tl = float(F.cross_entropy(zt[torch.from_numpy(keep)], yt[torch.from_numpy(keep)], ignore_index=R.IGNORE))
    assert abs(loss - tl) <= MR.fp32_loss_bound(z, inv[keep], y[keep]), (loss, tl)


def test_point_head_drops_bad_labels_and_all_ignored_is_nan():
    z, inv, y = _scene(300, 900, 20, seed=3, bad=5)
    loss, pred, counts, bad = MR.point_head(z, inv, y)
    assert bad == 5
    ok = ~((y != R.IGNORE) & ((y < 0) | (y >= 20)))
    loss_ok, pred_ok, counts_ok, _ = MR.point_head(z, inv[ok], y[ok])
    assert loss == loss_ok and np.array_equal(counts, counts_ok) and np.array_equal(pred[ok], pred_ok)
    loss, _, counts, _ = MR.point_head(z, inv, np.full_like(y, R.IGNORE))
    assert math.isnan(loss) and not counts.any()


def _fabricate(n, c, seed, big=False, nan_scene=None):
    g = np.random.default_rng(seed)
    losses = (g.random(n) * 3).astype(np.float32)
    if nan_scene is not None:
        losses[nan_scene] = np.nan
    tgt = g.integers(0, (1 << 23) if big else 50000, (n, c))
    out = g.integers(0, (1 << 23) if big else 50000, (n, c))
    inter = np.minimum(np.minimum(tgt, out), g.integers(0, (1 << 23) if big else 50000, (n, c)))
    if nan_scene is not None:
        tgt[nan_scene] = out[nan_scene] = inter[nan_scene] = 0
    return losses, np.stack([inter, out, tgt], axis=1).astype(np.int64)


def _reference_scenes(losses, areas):
    scenes = []
    for s in range(len(losses)):
        i, o, t = (torch.from_numpy(areas[s, j]).float() for j in range(3))
        scenes.append((torch.tensor(losses[s]).item(), i.numpy(), (o + t - i).numpy(), t.numpy()))
    return scenes


@pytest.mark.parametrize('big', [False, True])
def test_validation_replay_equals_the_reference_meters_bit_for_bit(big):
    losses, areas = _fabricate(40, 20, seed=11, big=big, nan_scene=5)
    if big:
        assert areas[:, 2].sum(0).max() > (1 << 24)
    got = train_mink.validation_result(torch.from_numpy(losses), torch.from_numpy(areas), torch.zeros(40, dtype=torch.int32),
                                       weight=8, owner='DeviceMinkValidation')
    want = R.validate_tail(_reference_scenes(losses, areas), batch_size=8)
    assert R.same(got, want) and math.isnan(got[0]), (got, want)


def test_validation_replay_names_the_first_bad_scene():
    losses, areas = _fabricate(6, 5, seed=2)
    bad = torch.tensor([0, 0, 0, 0, 4, 1], dtype=torch.int32)
    with pytest.raises(IndexError, match='DeviceMinkValidation.end: scene 4 '):
        train_mink.validation_result(torch.from_numpy(losses), torch.from_numpy(areas), bad, owner='DeviceMinkValidation')


def _train_state(n, c, seed, big):
    losses, areas = _fabricate(n, c, seed, big)
    return torch.from_numpy(losses), torch.from_numpy(areas)


@pytest.mark.parametrize('big', [False, True])
def test_train_meter_replay_equals_the_reference_step_by_step(big):
    """fabricated per-step device state, read in three chunks; float32 epoch sums pass 2^24 with big"""
    c, n = 20, 30
    losses, areas = _train_state(n, c, 5, big)
    meter = train_mink.DeviceTrainMeter(c)
    ref = MR.TrainMeters()
    got = []
    for lo, hi in ((0, 7), (7, 8), (8, n)):
        meter._loss, meter._areas, meter._counted = losses[lo:hi].clone(), areas[lo:hi].clone(), [True] * (hi - lo)
        steps, totals = meter.read(weight=8)
        got += steps
    for s in range(n):
        i, o, t = (areas[s, j].float() for j in range(3))
        ref.step(losses[s].item(), i.numpy(), (o + t - i).numpy(), t.numpy(), batch_size=8)
    if big:
        assert float(ref.target.sum.max()) > (1 << 24)
    assert MR.same_steps(got, ref.steps)
    assert R.same(totals, ref.totals()), (totals, ref.totals())


def test_train_meter_without_counts_is_the_loss_meter():
    losses, _ = _train_state(9, 3, 1, False)
    meter = train_mink.DeviceTrainMeter(3)
    meter._loss, meter._areas, meter._counted = losses.clone(), None, [False] * 9
    steps, totals = meter.read(weight=2)
    ref = MR.TrainMeters()
    for s in range(9):
        ref.step(losses[s].item(), batch_size=2)
    assert MR.same_steps(steps, ref.steps) and totals[1:] == (None, None, None) and totals[0] == ref.loss.avg
    assert meter.read() == ([], totals)


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        losses, areas = _fabricate(8, 20, seed=200 + rank, big=True)
        ret[rank] = train_mink.validation_result(torch.from_numpy(losses), torch.from_numpy(areas),
                                                 torch.zeros(8, dtype=torch.int32), 4, dist.group.WORLD,
                                                 owner='DeviceMinkValidation')
    finally:
        dist.destroy_process_group()


def test_gloo_world2_merge_equals_the_per_scene_all_reduce():
    world = 2
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    per = [_fabricate(8, 20, seed=200 + r, big=True) for r in range(world)]
    for rank in range(world):
        scenes = []
        for s in range(8):
            vecs = [_reference_scenes(l[s:s + 1], a[s:s + 1])[0] for l, a in per]
            scenes.append((vecs[rank][0], *[sum(v[j] for v in vecs) for j in (1, 2, 3)]))
        want = R.validate_tail(scenes, batch_size=4)
        assert R.same(ret[rank], want), (rank, ret[rank], want)


def _abi(name, *args):
    from openscene_b200 import _cabi as C
    if not os.path.exists(C.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    L = C.lib()
    rc = getattr(L, name)(*args)
    return rc, (L.osb_last_error() or b'').decode()


def test_ce_head_eval_refuses_bad_arguments_on_the_host():
    P = 0x1000                                               # never dereferenced: every call must fail before a launch
    ws_ok = _abi('osb_ce_head_eval_workspace_bytes', 100, 96, 20)[0]
    assert ws_ok > 0
    assert _abi('osb_ce_head_eval_workspace_bytes', 100, 100, 20)[0] == 0
    assert _abi('osb_ce_head_eval_workspace_bytes', 100, 96, 161)[0] == 0
    assert _abi('osb_ce_head_eval_workspace_bytes', -1, 96, 20)[0] == 0

    def call(x=P, n_rows=100, cin=96, w=P, c=20, row_map=P, inv=P, n_pts=150, label=P, lab64=1, loss=P, areas=P, bad=P,
             ws=0x100000, ws_bytes=ws_ok):
        return _abi('osb_ce_head_eval', x, n_rows, cin, w, c, row_map, inv, n_pts, label, lab64, 255, None, loss, areas, bad,
                    ws, ws_bytes, None)

    cases = {
        'rows=0': call(n_rows=0), 'points<0': call(n_pts=-1), 'no inds_reverse': call(inv=None),
        'cin=0': call(cin=0), 'cin=100': call(cin=100), 'cin=416': call(cin=416),
        'C=0': call(c=0), 'C=161': call(c=161), 'label dtype': call(lab64=2),
        'x': call(x=None), 'w': call(w=None), 'row_map': call(row_map=None), 'labels': call(label=None),
        'loss': call(loss=None), 'areas': call(areas=None), 'bad': call(bad=None),
        'x misaligned': call(x=P + 8), 'ws': call(ws=None), 'ws small': call(ws_bytes=ws_ok - 1),
        'ws misaligned': call(ws=0x100000 + 64),
    }
    for what, (rc, err) in cases.items():
        assert rc != 0 and err.startswith('osb_ce_head_eval'), (what, rc, err)
    assert 'every row is one point' in cases['no inds_reverse'][1] and 'classes (161)' in cases['C=161'][1]


def test_meters_refuse_what_the_reference_never_does():
    class _Eng:
        batch_stats, out_channels, device = True, 20, torch.device('cpu')
    with pytest.raises(ValueError, match='eval mode'):
        train_mink.DeviceMinkValidation(_Eng(), 20)
    _Eng.batch_stats = False
    with pytest.raises(ValueError, match='classes=13'):
        train_mink.DeviceMinkValidation(_Eng(), 13)
    with pytest.raises(ValueError, match='positive'):
        train_mink.DeviceTrainMeter(0)
