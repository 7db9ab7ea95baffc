"""osb_ce_head_eval (k_ce_fwd_eval), FusedMinkUNet.forward_eval_ce, train_mink.DeviceMinkValidation and DeviceTrainMeter on
the GPU: the supervised validation tail of run/train_mink.py (validate(), :366-384) and train()'s per-step meters.

The kernel is checked against fp64 on the split rows it read (tests/minkval_ref.py): the loss within the CE forward's
bound (2^-20 relative, tests/test_gpu_ce_head.py), pred equal to the fp64 first argmax wherever the row's top-two gap exceeds
2^-18 max|z|, the counts equal to the counts of the kernel's own pred, outputs in poisoned buffers and bit-identical reruns.
Dyadic operands make every logit exact: pred and the counts then equal the exact values bit for bit, ties across the
31|32 and 127|128 chunk edges and at the last class included.  End to end, DeviceMinkValidation equals the reference's torch
tail on the eval engine's logits."""
import datetime
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from openscene_b200 import _cabi as C
from openscene_b200 import engine, synth, train_mink
from tests import minkval_ref as MR
from tests import valce_ref as R

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _split(v):
    n, c = v.shape
    rows = torch.empty((n, 4 * c), dtype=torch.uint8, device=DEV)
    C.call('osb_f32_to_split', C.ptr(v.float().contiguous()), n, c, C.ptr(rows), C.stream_ptr())
    return rows


def _joined(rows, c):
    out = torch.empty((rows.shape[0], c), dtype=torch.float32, device=DEV)
    C.call('osb_split_to_f32', C.ptr(rows), rows.shape[0], c, C.ptr(out), C.stream_ptr())
    return out


def head_eval(xs, cin, w, c, row_map, inv, y, ignore=R.IGNORE, want_pred=True):
    """one osb_ce_head_eval into poisoned buffers: (pred, loss, areas, bad)"""
    n_rows = xs.shape[0]
    n_pts = inv.numel() if inv is not None else n_rows
    ws_b = C.lib().osb_ce_head_eval_workspace_bytes(n_pts, cin, c)
    ws = torch.full((ws_b,), 0xFF, dtype=torch.uint8, device=DEV)
    pred = torch.full((n_pts,), -7, dtype=torch.int64, device=DEV) if want_pred else None
    loss = torch.full((1,), 1234.0, device=DEV)
    areas = torch.zeros((3, c), dtype=torch.int64, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    C.call('osb_ce_head_eval', C.ptr(xs), n_rows, cin, C.ptr(w), c, C.ptr(row_map), C.ptr(inv), n_pts, C.ptr(y),
           int(y.dtype == torch.int64), ignore, C.ptr(pred), C.ptr(loss), C.ptr(areas), C.ptr(bad), C.ptr(ws), ws_b,
           C.stream_ptr())
    return pred, loss, areas, bad


def points(n_pts, mode, g):
    """(n_rows, inds_reverse or None): no map, fewer points than rows, a permutation, heavy repeats"""
    if mode == 'none':
        return n_pts, None
    if mode == 'short':
        n_rows = n_pts + n_pts // 2 + 1
        return n_rows, torch.randperm(n_rows, generator=g)[:n_pts].to(DEV)
    if mode == 'equal':
        return n_pts, torch.randperm(n_pts, generator=g).to(DEV)
    n_rows = max(1, n_pts // 7)
    return n_rows, torch.randint(0, n_rows, (n_pts,), generator=g).to(DEV)


def labels(n, c, g, i64, ignored=0.15):
    y = torch.randint(0, c, (n,), generator=g)
    y[torch.rand(n, generator=g) < ignored] = R.IGNORE
    return y.to(torch.int64 if i64 else torch.int32).to(DEV)


# (n_pts, mode, cin, C, int64 labels, logit scale)
CASES = [(1, 'none', 32, 1, True, 1.0), (1, 'repeat', 96, 20, False, 1.0), (255, 'short', 384, 160, True, 1.0),
         (256, 'equal', 96, 31, False, 1.0), (257, 'repeat', 32, 32, True, 1.0), (257, 'none', 96, 33, False, 1.0),
         (70001, 'short', 96, 20, True, 1.0), (70001, 'repeat', 384, 33, False, 1000.0), (70001, 'equal', 32, 160, True, 1.0),
         (300000, 'repeat', 96, 20, False, 1.0), (300000, 'none', 384, 160, True, 1000.0), (300000, 'short', 32, 1, False, 1.0)]

NAN_ROWS = {(257, 'none'), (70001, 'equal'), (300000, 'repeat')}


@pytest.mark.parametrize('n_pts,mode,cin,c,i64,scale', CASES)
def test_kernel_against_fp64(n_pts, mode, cin, c, i64, scale):
    g = torch.Generator().manual_seed(n_pts + cin + c)
    n_rows, inv = points(n_pts, mode, g)
    x = torch.randn(n_rows, cin, generator=g)
    if (n_pts, mode) in NAN_ROWS:
        x[13] = float('nan')                                        # a NaN row: its first class, a NaN loss if labelled
    w = (torch.randn(cin, c, generator=g) / cin ** 0.5 * scale).to(DEV)
    xs = _split(x.to(DEV))
    row_map = torch.randperm(n_rows, generator=g).to(torch.int32).to(DEV)     # caller row -> internal (split) row
    y = labels(n_pts, c, g, i64)
    pred, loss, areas, bad = head_eval(xs, cin, w, c, row_map, inv, y)
    z = (_joined(xs, cin).double() @ w.double()).cpu().numpy()
    rows = (row_map.long()[inv] if inv is not None else row_map.long()).cpu().numpy()
    yc = y.long().cpu().numpy()
    l64, p64, _, nbad = MR.point_head(z, rows, yc)
    assert int(bad) == 0 and nbad == 0
    pc = pred.cpu().numpy()
    zp = z[rows]
    nan = np.isnan(zp).any(axis=1)
    top = np.sort(np.where(np.isnan(zp), -np.inf, zp), axis=1)
    gap = top[:, -1] - top[:, -2] if c > 1 else np.full(n_pts, np.inf)
    sure = nan | (gap > 2 ** -18 * np.nanmax(np.abs(zp), axis=1, initial=0.0))
    assert np.array_equal(pc[sure], p64[sure])
    assert np.array_equal(areas.cpu().numpy(), R.device_counts(pc, yc, c, c)[0])
    if math.isnan(l64):
        assert math.isnan(float(loss))
    else:
        assert abs(float(loss) - l64) <= 2 ** -20 * (abs(l64) + 1), (float(loss), l64)
    again = head_eval(xs, cin, w, c, row_map, inv, y)
    for a, b in zip((pred, loss, areas, bad), again):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                           b.view(torch.int32) if b.dtype == torch.float32 else b)


def test_all_ignored_empty_and_bad_labels():
    g = torch.Generator().manual_seed(4)
    cin, c, n = 96, 20, 5000
    xs = _split(torch.randn(n, cin, generator=g).to(DEV))
    w = (torch.randn(cin, c, generator=g) / 10).to(DEV)
    row_map = torch.arange(n, dtype=torch.int32, device=DEV)
    none = torch.full((n,), R.IGNORE, dtype=torch.int64, device=DEV)
    _, loss, areas, bad = head_eval(xs, cin, w, c, row_map, None, none)
    assert math.isnan(float(loss)) and int(areas.abs().sum()) == 0 and int(bad) == 0
    empty = torch.empty(0, dtype=torch.int64, device=DEV)
    _, loss, areas, bad = head_eval(xs, cin, w, c, row_map, empty, empty, want_pred=False)
    assert math.isnan(float(loss)) and int(areas.abs().sum()) == 0
    y = labels(n, c, g, True)
    planted = torch.tensor([3, 400, 4999])
    y[planted.to(DEV)] = torch.tensor([c, -1, 1000], device=DEV)
    pred, loss, areas, bad = head_eval(xs, cin, w, c, row_map, None, y)
    assert int(bad) == 3
    keep = torch.ones(n, dtype=torch.bool)
    keep[planted] = False
    keep = keep.to(DEV)
    inv = torch.arange(n, device=DEV)[keep]
    pred_ok, loss_ok, areas_ok, bad_ok = head_eval(xs, cin, w, c, row_map, inv, y[keep])
    assert torch.equal(areas, areas_ok) and torch.equal(loss, loss_ok) and torch.equal(pred[keep], pred_ok)


@pytest.mark.parametrize('cin,c', [(96, 160), (384, 33), (32, 129)])
def test_exact_probes_chunk_edge_ties(cin, c):
    """x in (1/8) Z and W in (1/16) Z, small: every product and partial sum is exact in fp32, so z is exact.  Columns
    31 / 32, 127 / 128 and 5 / C-1 are equal and dominate the rows of one group each: the first maximum must win."""
    g = torch.Generator().manual_seed(cin + c)
    n = 3000
    x = torch.randint(-4, 5, (n, cin), generator=g).double() / 8
    w = torch.randint(-4, 5, (cin, c), generator=g).double() / 16
    pairs = [(31, 32), (127, 128), (5, c - 1)]
    for k, (a, b) in enumerate(pairs):
        if b < c:
            w[k, a] = w[k, b] = 8.0
            w[:, b] = w[:, a]
            x[k * 1000:(k + 1) * 1000, k] = 8.0
    xs = _split(x.float().to(DEV))
    row_map = torch.randperm(n, generator=g).to(torch.int32).to(DEV)
    inv = torch.randint(0, n, (2 * n,), generator=g).to(DEV)
    y = labels(2 * n, c, g, False)
    pred, loss, areas, bad = head_eval(xs, cin, w.float().to(DEV), c, row_map, inv, y)
    z = x.to(DEV)[row_map.long()[inv]] @ w.to(DEV)                # exact in fp64 as in fp32
    assert torch.equal(_joined(xs, cin).double(), x.to(DEV))
    want = z.argmax(1)                                              # first maximum
    assert torch.equal(pred, want)
    for k, (a, b) in enumerate(pairs):
        if b < c:
            grp = (row_map.long()[inv] >= 0) & (x.to(DEV)[row_map.long()[inv], k] == 8.0)
            assert bool((pred[grp] != b).all()) and bool((pred[grp] == a).any())
    yc = y.long().cpu().numpy()
    assert np.array_equal(areas.cpu().numpy(), R.device_counts(want.cpu().numpy(), yc, c, c)[0]) and int(bad) == 0
    l64, _, _, _ = MR.point_head(x[row_map.long().cpu()].numpy() @ w.numpy(), inv.cpu().numpy(), yc)
    assert abs(float(loss) - l64) <= 2 ** -20 * (abs(l64) + 1)


def _scenes(config, count, c, seed0=0):
    out = []
    for s in range(count):
        coords = torch.from_numpy(synth.scene(config, seed=seed0 + s))
        g = torch.Generator().manual_seed(seed0 + s)
        n_vox = coords.shape[0]
        inv = torch.cat([torch.randperm(n_vox, generator=g), torch.randint(0, n_vox, (n_vox // 2,), generator=g)])
        z = coords[:, 3].float()
        label = (z / (z.max() + 1) * c).long()[inv]
        label[torch.rand(len(inv), generator=g) < 0.15] = R.IGNORE
        out.append((coords, torch.rand(n_vox, 3, generator=g), inv, label))
    return out


def _torch_tail(eng, scenes, c):
    """the reference's validate() body after the forward, per scene: (loss.item(), i, u, t) and the logits / pred"""
    rows, extra = [], []
    for coords, feats, inv, label in scenes:
        with torch.no_grad():
            output = eng(coords.to(DEV), feats.to(DEV))[inv.to(DEV)]
        lab = label.to(DEV)
        loss = F.cross_entropy(output, lab, ignore_index=R.IGNORE)
        pred = output.max(1)[1]
        i, u, t = R.intersection_and_union(pred.cpu(), lab.cpu(), c)
        rows.append((loss.item(), i.numpy(), u.numpy(), t.numpy()))
        extra.append((output, pred))
    return rows, extra


def _device(eng, scenes, c):
    meter = train_mink.DeviceMinkValidation(eng, c)
    preds = []
    for coords, feats, inv, label in scenes:
        meter.add(coords, feats, inv, label)
        pred = torch.empty(len(inv), dtype=torch.int64, device=DEV)
        slot_l, slot_a, slot_b = (torch.zeros(1, device=DEV), torch.zeros((3, c), dtype=torch.int64, device=DEV),
                                  torch.zeros(1, dtype=torch.int32, device=DEV))
        eng.forward_eval_ce(coords.to(DEV), feats.to(DEV), label, inv, slot_l, slot_a, slot_b, pred=pred)
        preds.append(pred)
    return meter.end(weight=1), meter, preds


@pytest.mark.parametrize('arch,config', [('MinkUNet18A', 'config1_50k'), ('MinkUNet34C', 'config2_200k')])
def test_device_validation_equals_the_torch_tail(arch, config):
    torch.cuda.set_device(0)
    c = 20
    model = synth.build_model(arch, c, seed=0).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    scenes = _scenes(config, 3, c)
    want_rows, extra = _torch_tail(eng, scenes, c)
    got, meter, preds = _device(eng, scenes, c)
    want = R.validate_tail(want_rows, batch_size=1)
    near, bounds = 0, []
    for (output, pt), pd, (_, _, inv, label) in zip(extra, preds, scenes):
        diff = pd != pt
        if bool(diff.any()):
            top = output[diff].topk(2, 1).values
            assert bool((top[:, 0] - top[:, 1] <= 2 ** -16 * output[diff].abs().max(1).values).all())
            near += int(diff.sum())
        zc = output.double().cpu().numpy()
        bounds.append(2 * MR.fp32_loss_bound(zc, np.arange(len(zc)), label.numpy())
                      + 2 ** -15 * float(output.abs().max()))
    if near == 0:
        assert R.same(got[1:], want[1:]), (got, want)
    else:                                                          # every differing point moves each count by at most one
        a = meter._areas[:meter.n].sum(0).cpu()
        ref = torch.stack([torch.from_numpy(np.sum([r[j] for r in want_rows], axis=0)) for j in (1, 3)])
        assert float((a[0].double() - ref[0].double()).abs().max()) <= near
    assert abs(got[0] - want[0]) <= float(np.mean(bounds)), (got[0], want[0])
    # probe weights: logit c is trunk channel 3 c exactly on both paths, so everything but the loss is bit for bit
    with torch.no_grad():
        model.final.kernel.zero_()
        model.final.kernel[torch.arange(c) * 3, torch.arange(c)] = 1.0
    want_rows, extra = _torch_tail(eng, scenes, c)
    got, _, preds = _device(eng, scenes, c)
    for (_, pt), pd in zip(extra, preds):
        assert torch.equal(pt, pd)
    assert R.same(got[1:], R.validate_tail(want_rows, batch_size=1)[1:])


def test_stale_weights_are_refolded_after_device_optimiser_steps():
    from openscene_b200 import optim
    torch.cuda.set_device(0)
    c = 20
    model = synth.build_model('MinkUNet18A', c, seed=1).to(DEV)
    model.eval()
    stale = engine.FusedMinkUNet(model)
    scenes = _scenes('config1_50k', 2, c, seed0=7)
    first, _, _ = _device(stale, scenes, c)                        # packs folded from the initial weights
    model.train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    coords = torch.from_numpy(synth.scene('config1_50k', seed=3)).to(DEV)
    feats = torch.rand(coords.shape[0], 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    lab = (coords[:, 3].long() * 7 + coords[:, 1].long()) % c
    for opt in (optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4),
                optim.Adam(model.parameters(), lr=1e-3)):
        opt.bind(eng)
        for _ in range(2):
            train_mink.fused_train_step(eng, opt, coords, feats, lab)
    model.eval()
    got, _, preds = _device(stale, scenes, c)
    fresh, _, fresh_preds = _device(engine.FusedMinkUNet(model), scenes, c)
    assert R.same(got, fresh), (got, fresh)
    assert not R.same(got, first)
    for a, b in zip(preds, fresh_preds):
        assert torch.equal(a, b)


def test_side_stream_and_poisoned_workspace_equal_a_serialised_run():
    torch.cuda.set_device(0)
    c = 20
    model = synth.build_model('MinkUNet18A', c, seed=2).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    scenes = [(co.to(DEV), f.to(DEV), i.to(DEV), l.to(DEV)) for co, f, i, l in _scenes('config1_50k', 3, c, seed0=11)]
    ref = train_mink.DeviceMinkValidation(eng, c)
    for s in scenes:
        ref.add(*s)
        torch.cuda.synchronize()
    want = ref.end()
    meter = train_mink.DeviceMinkValidation(eng, c)
    meter._loss.fill_(float('nan'))
    eng._ce_ws.fill_(0xFF)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    torch.cuda._sleep(50_000_000)                                   # the default stream is busy while the side stream runs
    with torch.cuda.stream(side):
        for s in scenes:
            meter.add(*s)
    side.synchronize()
    torch.cuda.synchronize()
    got = meter.end()
    assert R.same(got, want), (got, want)
    assert torch.equal(meter._areas[:3], ref._areas[:3]) and torch.equal(meter._loss[:3].view(torch.int32),
                                                                          ref._loss[:3].view(torch.int32))


def test_train_meter_equals_the_reference_meters_over_fused_steps():
    torch.cuda.set_device(0)
    c = 20
    model = synth.build_model('MinkUNet18A', c, seed=0).train().to(DEV)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    coords = torch.cat([torch.from_numpy(synth.scene('config1_50k', seed=i, batch_index=i)) for i in range(2)]).to(DEV)
    feats = torch.rand(coords.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    lab = ((coords[:, 3].long() // 8) * 5 + coords[:, 1].long() // 16) % c
    lab[(coords[:, 1] * 7 + coords[:, 2] * 13).long() % 10 == 0] = R.IGNORE
    meter, ref = train_mink.DeviceTrainMeter(c), MR.TrainMeters()
    got = []
    for step in range(5):
        loss, pred = train_mink.fused_train_step(eng, opt, coords, feats, lab)
        meter.add(loss, pred, lab)
        i, u, t = R.intersection_and_union(pred.cpu(), lab.cpu(), c)
        ref.step(loss.item(), i.numpy(), u.numpy(), t.numpy(), batch_size=8)
        if step in (1, 4):
            steps, totals = meter.read(weight=8)
            got += steps
    assert MR.same_steps(got, ref.steps), (got, ref.steps)
    assert R.same(totals, ref.totals())


def _free_port():
    sk = socket.socket()
    sk.bind(('127.0.0.1', 0))
    port = sk.getsockname()[1]
    sk.close()
    return port


def _pg_worker(rank, world, backend, port, devices):
    """each rank validates its own scenes with a process group; the reference all-reduces the three vectors of every scene"""
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dev = torch.device(devices[rank])
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(minutes=3))
    try:
        c = 20
        model = synth.build_model('MinkUNet18A', c, seed=0).eval().to(dev)
        with torch.no_grad():                    # probe weights: both tails see the same logits, so the metrics are exact
            model.final.kernel.zero_()
            model.final.kernel[torch.arange(c) * 3, torch.arange(c)] = 1.0
        eng = engine.FusedMinkUNet(model)
        scenes = _scenes('config1_50k', 2, c, seed0=20 + 5 * rank)
        meter = train_mink.DeviceMinkValidation(eng, c, process_group=dist.group.WORLD)
        rows = []
        for coords, feats, inv, label in scenes:
            meter.add(coords, feats, inv, label)
            with torch.no_grad():
                output = eng(coords.to(dev), feats.to(dev))[inv.to(dev)]
            lab = label.to(dev)
            loss = F.cross_entropy(output, lab, ignore_index=R.IGNORE)
            vecs = [v.to(dev) if backend == 'nccl' else v for v in R.intersection_and_union(output.max(1)[1].cpu(), lab.cpu(), c)]
            for v in vecs:
                dist.all_reduce(v)
            rows.append((loss.item(), *(v.cpu().numpy() for v in vecs)))
        got = meter.end(weight=1)
        want = R.validate_tail(rows, batch_size=1)
        assert R.same(got[1:], want[1:]), (rank, got, want)
        assert abs(got[0] - want[0]) <= 1e-5 * abs(want[0]), (rank, got, want)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_process_group_gloo_two_ranks_on_one_device():
    mp.spawn(_pg_worker, args=(2, 'gloo', _free_port(), ['cuda:0', 'cuda:0']), nprocs=2, join=True)


def test_process_group_nccl_two_devices():
    if torch.cuda.device_count() < 2:
        pytest.skip(f"NCCL needs one device per rank: {torch.cuda.device_count()} visible")
    mp.spawn(_pg_worker, args=(2, 'nccl', _free_port(), ['cuda:0', 'cuda:1']), nprocs=2, join=True)
