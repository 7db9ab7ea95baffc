"""The PDL window rule (tests/launch_order.py) over the launch plans of the fused engine, without a GPU.

The engine's Python runs on CPU tensors with the device entry points recorded (the fixtures of tests/test_engine_plan_cpu.py
and tests/test_engine_train_plan_cpu.py), here with one more layer that keeps every recorded call in stream order and with
kernel maps the size the kernels read.  For every launch with the PDL attribute, what it reads before ``griddepcontrol.wait``
(``k_conv_tc``: its kernel-map rows and BatchNorm scale / shift) must not be written by any launch of its PDL window: the
eval forward on the persistent chain and on one launch per layer, the training forward and backward, and the cosine
distillation step (``forward_train_cosine`` and its backward), for all ten architectures and three scene sizes.  The table of pre-wait reads is checked against the comments the kernels carry next to
their waits.  Negative controls: the persistent chain's former read of its grid-barrier generation before the wait, and a
kernel map produced inside the window of the layer that reads it."""
import pytest
import torch

from openscene_b200 import _cabi as C
from openscene_b200 import engine, engine_train, minkunet, synth
from tests import launch_order as LO
from tests import test_engine_train_plan_cpu as tp
from tests.test_engine_plan_cpu import SCENES, _FakeCM
from tests.test_engine_plan_cpu import recorded as eval_recorded        # noqa: F401 (fixture)
from tests.test_engine_train_plan_cpu import recorded as train_recorded  # noqa: F401 (fixture)


class _SizedMap:
    """a kernel map whose storage has the [K, n_out] int32 rows the kernels read (uninitialised: only addresses matter)"""

    def __init__(self, K, n_in, n_out):
        self.K, self.n_in, self.n_out = K, n_in, n_out
        self.nbr = torch.empty(K * n_out, dtype=torch.int32)
        self._t = None

    def transposed(self):
        if self._t is None:
            self._t = _SizedMap(self.K, self.n_out, self.n_in)
        return self._t


class _SizedCM(_FakeCM):
    def __init__(self, n):
        super().__init__(n)
        self.perm = torch.arange(n[0], dtype=torch.int32)
        self.inv_perm = self.perm.clone()

    def kernel_map(self, ts_in, ts_out, ks, dilation=1):
        key = (ts_in, ts_out, ks, dilation)
        if key not in self.kmaps:
            self.kmaps[key] = _SizedMap(ks ** 3, self.sets[ts_in].n, self.sets[ts_out].n)
        return self.kmaps[key]


def _in_order(monkeypatch):
    """wrap the recording library once more: every device entry point, in the order the engine issues it"""
    seq = []
    inner_lib, inner_call = C.lib(), C.call

    class Lib:
        def __getattr__(self, name):
            fn = getattr(inner_lib, name)
            if LO.is_host_only(name):
                return fn

            def rec(*a):
                seq.append(LO.launch_of(name, a))
                return fn(*a)
            return rec

    lib = Lib()
    monkeypatch.setattr(C, 'lib', lambda: lib)

    def call(name, *a):
        if not LO.is_host_only(name):
            seq.append(LO.launch_of(name, a))
        return inner_call(name, *a)
    monkeypatch.setattr(C, 'call', call)
    return seq


def _eval_plan(monkeypatch, arch, scene, chain):
    seq = _in_order(monkeypatch)
    n = SCENES[scene]
    eng = engine.FusedMinkUNet(synth.build_model(arch, 768, seed=0).eval())
    eng.use_chain = chain
    cm = _SizedCM(n)
    for _ in range(2):                                  # two forwards: the second one's windows reach back into the first
        eng(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), coordinate_manager=cm)
    return seq


def _summary(seq, table=None):
    n_win, n_in, bad = LO.check_windows(seq, table)
    return dict(launches=len(seq), pdl=sum(1 for L in seq if L.pdl), windows=n_win, in_windows=n_in, bad=bad)


@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_eval_plan_respects_pdl_windows(eval_recorded, monkeypatch, arch, scene):  # noqa: F811
    for chain in (True, False):
        s = _summary(_eval_plan(monkeypatch, arch, scene, chain))
        assert not s['bad'], s['bad'][:3]
        assert s['pdl'] > 0 and s['windows'] == s['pdl']
        if not chain:
            assert s['in_windows'] > s['windows']            # one launch per layer: long windows, all of them checked


@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_train_plan_respects_pdl_windows(train_recorded, monkeypatch, arch, scene):  # noqa: F811
    n = train_recorded.n = SCENES[scene]
    monkeypatch.setattr(engine_train, 'CoordinateManager', lambda coords, pyramid_levels=0: _SizedCM(n))
    seq = _in_order(monkeypatch)
    model = synth.build_model(arch, 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    rows = torch.arange(n[0]) % 7 == 0
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        out = eng.forward_train(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), rows=rows)
        out.sum().backward()
    s = _summary(seq)
    assert not s['bad'], s['bad'][:3]
    # the forward's convolutions run with PDL, each behind a BatchNorm launch that closes its window; the final layer reads
    # the selected rows' map before its wait
    assert s['pdl'] > 0 and s['windows'] == s['pdl']
    heads = [L for L in seq if L.name == 'osb_conv_fwd_tc' and L.pdl and L.operands['nbr']
             and L.operands['nbr'][0][1] - L.operands['nbr'][0][0] == 4 * int(rows.sum())]
    assert len(heads) == 2


@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('arch', sorted(minkunet.ARCHS))
def test_cosine_plan_respects_pdl_windows(train_recorded, monkeypatch, arch, scene):  # noqa: F811
    assert LO.is_host_only('osb_cos_head_workspace_bytes')
    monkeypatch.setattr(tp, '_HOST', tp._HOST | {'osb_cos_head_workspace_bytes'})
    n = train_recorded.n = SCENES[scene]
    monkeypatch.setattr(engine_train, 'CoordinateManager', lambda coords, pyramid_levels=0: _SizedCM(n))
    seq = _in_order(monkeypatch)
    model = synth.build_model(arch, 768, seed=0).train()
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    rows = torch.arange(n[0]) % 7 == 0
    target = torch.ones(int(rows.sum()), 768, dtype=torch.float16)
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        loss = eng.forward_train_cosine(torch.zeros(n[0], 4, dtype=torch.int32), torch.ones(n[0], 3), target, rows)
        (0.75 * loss).backward()
    s = _summary(seq)
    assert not s['bad'], s['bad'][:3]
    assert s['pdl'] > 0 and s['windows'] == s['pdl']
    # the head is two plain launches per step, each closing the window of what follows it; no tensor-core head launch
    heads = [L for L in seq if L.name in ('osb_cos_head_fwd', 'osb_cos_head_bwd')]
    assert [L.name for L in heads] == ['osb_cos_head_fwd', 'osb_cos_head_bwd'] * 2 and not any(L.pdl or L.triggers for L in heads)
    assert not any(L.name == 'osb_conv_fwd_tc' and L.writes and any(w[2] == 'out_f32' for w in L.writes) for L in seq)


def test_prewait_table_matches_the_kernels():
    """every kernel that triggers its dependents early carries a pre-wait comment, and the comments are the test's table"""
    marks, triggers = LO.source_prewait()
    assert marks == LO.PREWAIT, (marks, LO.PREWAIT)
    assert triggers == set(LO.PREWAIT), triggers
    assert {k for ks in LO.PDL_ENTRY.values() for k in ks} == set(LO.PREWAIT)


def test_window_check_catches_a_producer_in_the_window(eval_recorded, monkeypatch):  # noqa: F811
    """Negative controls.  (1) The persistent chain as it read its grid-barrier generation before its wait: every chain launch
    after the first reads a word the launch before it writes.  (2) One launch per layer, with a layer's kernel map written
    by a triggering PDL launch just before it (a map built lazily between layers): the map is a pre-wait read."""
    seq = _eval_plan(monkeypatch, 'MinkUNet34C', 'bench', True)
    assert not LO.check_windows(seq)[2]
    old = dict(LO.PREWAIT, k_conv_chain=('gbar',))
    bad = LO.check_windows(seq, old)[2]
    n_chain = sum(1 for L in seq if L.name == 'osb_conv_chain_launch')
    readers = {b.split(' reads ')[0] for b in bad}
    assert n_chain > 4 and len(readers) == n_chain - 2, (n_chain, bad[:2])     # all but the first of each forward (the stem)
    assert all('k_conv_chain.gbar' in b and 'grid barrier' in b for b in bad)

    seq = _eval_plan(monkeypatch, 'MinkUNet34C', 'bench', False)
    assert not LO.check_windows(seq)[2]
    i = next(i for i, L in enumerate(seq) if L.name == 'osb_conv_fwd_tc' and L.operands['nbr'] and i > 10)
    lo, hi = seq[i].operands['nbr'][0]
    producer = LO.Launch('osb_conv_fwd_tc', True, {}, [(lo, hi, 'a kernel map')])
    bad = LO.check_windows(seq[:i] + [producer] + seq[i:])[2]
    assert bad and all('k_conv_tc.nbr' in b and 'a kernel map' in b for b in bad), bad[:2]
    # the same producer behind a launch that closes the window is ordered
    closer = LO.Launch('osb_kernel_map_transpose', False)
    assert not LO.check_windows(seq[:i] + [producer, closer] + seq[i:])[2]
