"""Static check of the data-parallel backward of the fused engine (``FusedMinkUNet(model, batch_stats=True, process_group=pg)``,
openscene_b200/engine_train.py), without a GPU: the launch recorder of tests/test_engine_train_plan_cpu.py, plus a fake process
group of two ranks that records every collective with the number of launches issued before it.  For all ten architectures and
three scene sizes:
  * the all-reduce buckets cover every parameter gradient exactly once, contiguous in the flat buffer, in reverse parameter
    order, with DistributedDataParallel's size caps;
  * each bucket is issued after the last launch (kernel or copy) that writes one of its slots, and the last one holds the stem;
  * the backward waits on every collective, after its last launch;
plus the ordering guard as a negative control, the construction refusals (with a simulated gathered signature) and the buffer
broadcast rule."""
import types

import pytest
import torch
import torch.distributed as dist

from openscene_b200 import engine, engine_train, minkunet, synth
from tests.test_engine_plan_cpu import SCENES
from tests.test_engine_train_plan_cpu import _CM, _check, _i, _run, recorded  # noqa: F401  (recorded: fixture)

_LAUNCH_FREE = ('all_reduce', 'wait', 'broadcast', 'all_gather')


class _Group:
    def __init__(self, world=2, rank=0):
        self.world, self.rank = world, rank


@pytest.fixture
def dp(recorded, monkeypatch):
    """recorded + a fake group: collectives and device copies go into recorded.calls"""
    rec = recorded
    rec.gathered = None                            # signatures the fake all_gather returns (None: every rank holds this one)
    rec.sigs = []

    def world(group=None):
        assert isinstance(group, _Group), "a collective outside the engine's own group"
        return group.world

    def all_gather(out, t, group=None):
        world(group)
        rec.sigs.append(t.clone())
        rec.calls.append(('all_gather', ()))
        for r, o in enumerate(out):
            o.copy_(t if rec.gathered is None or r == group.rank else rec.gathered)

    def broadcast_coalesced(group, tensors, bucket_bytes, src):
        world(group)
        assert src == 0
        rec.calls.append(('broadcast', tuple(x.data_ptr() for x in tensors)))

    def all_reduce(t, group=None, async_op=False):
        world(group)
        assert async_op and t.is_contiguous()
        rec.calls.append(('all_reduce', (t.data_ptr(), t.numel())))
        return types.SimpleNamespace(wait=lambda: rec.calls.append(('wait', ())))

    copy = torch.Tensor.copy_

    def copy_(self, src, non_blocking=False):
        rec.calls.append(('copy_', (self.data_ptr(),)))
        return copy(self, src, non_blocking)

    monkeypatch.setattr(dist, 'get_world_size', world)
    monkeypatch.setattr(dist, 'get_rank', lambda group=None: group.rank)
    monkeypatch.setattr(dist, 'all_gather', all_gather)
    monkeypatch.setattr(dist, '_broadcast_coalesced', broadcast_coalesced)
    monkeypatch.setattr(dist, 'all_reduce', all_reduce)
    monkeypatch.setattr(torch.Tensor, 'copy_', copy_)
    return rec


def _collectives(rec):
    return [c for c in rec.calls if c[0] in _LAUNCH_FREE]


def _slot_writes(name, a):
    a = [_i(x) for x in a]
    if name == 'osb_conv_wgrad_tc':
        return [a[8]]
    if name == 'osb_bn_backward_reduce':
        return [a[8], a[9]]
    if name == 'copy_':
        return [a[0]]
    return []


def _check_buckets(bwd, model):
    params = list(model.parameters())
    slots = [(p.grad.data_ptr(), 4 * p.numel()) for p in params]

    def slot_of(ptr):
        hit = [i for i, (a, nb) in enumerate(slots) if a <= ptr < a + nb]
        return hit[0] if hit else None
    last_write = {}
    launches = [k for k, (name, _) in enumerate(bwd) if name not in _LAUNCH_FREE]
    for k, (name, a) in enumerate(bwd):
        for ptr in _slot_writes(name, a):
            s = slot_of(ptr)
            if s is not None:
                last_write[s] = k
    assert sorted(last_write) == list(range(len(params))), "every slot written in the backward"
    issued = [(k, a) for k, (name, a) in enumerate(bwd) if name == 'all_reduce']
    hi, sizes = len(params), []
    for k, (ptr, numel) in issued:
        idx = [i for i, (a, nb) in enumerate(slots) if ptr <= a < ptr + 4 * numel]
        assert idx == list(range(idx[0], idx[-1] + 1)) and idx[-1] == hi - 1, "contiguous, in reverse parameter order"
        assert slots[idx[0]][0] == ptr and sum(slots[i][1] for i in idx) == 4 * numel, "the bucket is exactly its slots"
        assert k > max(last_write[i] for i in idx), "a bucket issued before the last launch writing one of its slots"
        hi = idx[0]
        sizes.append([slots[i][1] for i in idx])
    assert hi == 0, "the buckets cover every parameter"
    stem = next(i for i, p in enumerate(params) if p is model.conv0p1s1.kernel)
    assert stem == 0 and slots[stem][0] == issued[-1][1][0], "the last bucket holds the stem"
    for j, sz in enumerate(sizes[:-1]):                          # DistributedDataParallel's caps: closed once reached
        cap = engine_train._FIRST_BUCKET_BYTES if j == 0 else engine_train._BUCKET_BYTES
        assert sum(sz) >= cap > sum(sz) - sz[0]
    waits = [k for k, (name, _) in enumerate(bwd) if name == 'wait']
    assert len(waits) == len(issued) and min(waits) > max(launches), "every collective waited on, after the last launch"
    if len(issued) > 1:
        assert issued[0][0] < last_write[stem], "the first bucket overlaps the rest of the backward"
    return len(issued)


@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_dp_bucket_plan(dp, arch, scene):
    n = dp.n = SCENES[scene]
    model = synth.build_model(arch, 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True, process_group=_Group())
    rows = torch.arange(n[0]) % 7 == 0
    for _ in range(2):
        dp.calls.clear()
        model.zero_grad(set_to_none=True)
        out = _run(eng, n, rows)
        nf = len(dp.calls)
        out.sum().backward()
        _check(dp.calls, nf, model)                              # the launches themselves are those of the local backward
        nb = _check_buckets(dp.calls[nf:], model)
        assert nb >= 2


def test_local_engine_issues_no_collective(dp):
    n = dp.n = SCENES['tiny']
    model = synth.build_model('MinkUNet18A', 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    _run(eng, n).sum().backward()
    assert not [c for c in dp.calls if c[0] in _LAUNCH_FREE]


def test_ordering_guard_raises(dp, monkeypatch):
    """negative control: the first bucket's boundary moved down to the stem, slots the backward has not written yet"""
    n = dp.n = SCENES['tiny']
    model = synth.build_model('MinkUNet18A', 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True, process_group=_Group())
    plan = engine_train.plan_buckets

    def moved(tape, params):
        (lo, hi, t), = plan(tape, params)[:1]
        return [(0, hi, t)]
    monkeypatch.setattr(engine_train, 'plan_buckets', moved)
    out = _run(eng, n)
    with pytest.raises(RuntimeError, match='still unwritten'):
        out.sum().backward()


def test_construction_refusals_and_broadcast(dp):
    n = dp.n = SCENES['tiny']
    with pytest.raises(ValueError, match='batch_stats=True'):
        engine.FusedMinkUNet(synth.build_model('MinkUNet18A', 768, seed=0).eval(), process_group=_Group())
    assert _collectives(dp) == []
    engine.FusedMinkUNet(synth.build_model('MinkUNet34C', 768, seed=0).train(), batch_stats=True, process_group=_Group())
    sig34 = dp.sigs[-1]
    dp.gathered = sig34                                          # the other rank holds MinkUNet34C
    for rank in (0, 1):
        dp.calls.clear()
        model = synth.build_model('MinkUNet18A', 768, seed=rank).train()
        before = {k: v.clone() for k, v in model.state_dict().items()}
        with pytest.raises(RuntimeError, match='differ from rank 0'):
            engine.FusedMinkUNet(model, batch_stats=True, process_group=_Group(rank=rank))
        assert [c[0] for c in _collectives(dp)] == ['all_gather'], "refused before any broadcast"
        assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
    dp.gathered = None
    dp.calls.clear()
    model = synth.build_model('MinkUNet18A', 768, seed=0).train()
    engine.FusedMinkUNet(model, batch_stats=True, process_group=_Group(rank=1))
    assert [c[0] for c in _collectives(dp)] == ['all_gather', 'broadcast']
    assert _collectives(dp)[1][1] == tuple(t.data_ptr() for t in list(model.parameters()) + list(model.buffers()))


def test_buffer_broadcast_rule(dp):
    """DistributedDataParallel's broadcast_buffers rule: before the first forward and after a grad-enabled one"""
    n = dp.n = SCENES['tiny']
    model = synth.build_model('MinkUNet14A', 64, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True, process_group=_Group())
    bufs = tuple(b.data_ptr() for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)
                 for b in (m.running_mean, m.running_var, m.num_batches_tracked))
    coords, feats = torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3)

    def fwd_train():
        eng.forward_train(coords, feats).sum().backward()

    def fwd_eval():
        with torch.no_grad():
            eng(coords, feats, coordinate_manager=_CM(n))
    seen = []
    for fn in (fwd_train, fwd_train, fwd_eval, fwd_eval, fwd_train, fwd_train):
        dp.calls.clear()
        fn()
        b = [c for c in dp.calls if c[0] == 'broadcast']
        assert all(c[1] == bufs for c in b)
        assert not b or dp.calls[0][0] == 'broadcast', "the buffers are broadcast before the forward's first launch"
        seen.append(len(b))
    assert seen == [1, 1, 1, 0, 0, 1]
