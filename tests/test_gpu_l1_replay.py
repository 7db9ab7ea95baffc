"""Replay of the L1 distillation step launch by launch: the BatchNorm replay harness of tests/test_gpu_norm_replay.py (its
worker script and ``Harness`` class, imported, with the L1 head's two entry points added), driven by
``forward_train_l1`` under ``(0.75 * loss).backward()`` so that a dropped upstream gradient shows.  On top of what that harness
checks for every BatchNorm launch:

* ``osb_l1_head_fwd`` reads the last apply's output with its rows and width, ``final.kernel``, the caller's targets and, as
  supervised rows, the inverse of the input gather's permutation at the caller's mask rows in caller order.  Its loss is
  within ``l1_ref.head``'s bound, and every stored sign equals the fp64 sign of f - t wherever the forward bound decides it;
* ``osb_l1_head_bwd`` reads the forward's rows, weights, row index and signs, the signs unchanged since the forward wrote
  them, and g = 0.75.  Its dx (exactly 0 on the unsupervised rows) and dW are within ``l1_ref.head``'s bounds on the stored
  signs; its dW is ``final.kernel.grad`` bit for bit and its dx is the gradient the first BatchNorm backward reduce and apply
  read.

Reference-side negative controls must fail: rows taken through the permutation instead of its inverse, targets rolled by one
row, and g = 1.  Runs on MinkUNet34C at config1_50k (the shipped 96 -> 768 head), MinkUNet14D with a 512-wide head (input
width 384) and all ten architectures at the tiny scene."""
import subprocess
import sys

import pytest

from tests.test_gpu_norm_replay import ARCHS, ROOT, WORKER

pytestmark = pytest.mark.gpu

_BASE = WORKER.rstrip()
assert _BASE.endswith('\nmain()')
_BASE = _BASE[:-len('main()')]

L1_WORKER = r'''
from tests import l1_ref as LR

PASS.add('osb_l1_head_workspace_bytes')
HANDLED = HANDLED + ('osb_l1_head_fwd', 'osb_l1_head_bwd')


class L1Harness(Harness):
    def __init__(self, model):
        super().__init__(model)
        self.l1 = {}
        self.l1_caller = None                              # (caller rows of the mask, feat_3d, g)
        self.l1_dx_readers = {}                            # BatchNorm backward entry point -> the dx it must read as g

    def l1_fails(self, got, ref, signs=None):
        """outside a bound, or a stored sign the forward bound decides that differs from the reference's"""
        if any(LR.ratio(v, *ref[k]) > 1 for k, v in got.items()):
            return True
        return signs is not None and not bool((signs[LR.certain(ref)] == LR.sgn(ref['d'][0])[LR.certain(ref)]).all())

    def _l1_head_fwd(self, *args):
        a = [_i(v) for v in args]
        x_a, n, cin, w_a, c, rows_a, m, t_a, s_a, loss_a = a[:10]
        torch.cuda.synchronize()
        A = self.applies[-1] if self.applies else None
        assert A is not None and (A['y'], A['n'], A['c']) == (x_a, n, cin), "the L1 head does not read the trunk's last activation"
        assert w_a == self.model.final.kernel.data_ptr() and (cin, c) == tuple(self.model.final.kernel.shape[-2:]), \
            "the L1 head does not read final.kernel"
        caller, feat, _ = self.l1_caller
        assert t_a == feat.data_ptr() and m == feat.shape[0] == caller.numel(), "the L1 head does not read the caller's targets"
        assert self.gather_perm is not None and self.gather_perm[1] == n, "no input gather before the L1 head"
        perm = snap(self.gather_perm[0], 4 * n).view(torch.int32).long()
        inv = torch.empty_like(perm)
        inv[perm] = torch.arange(n, device=dev)
        sel = snap(rows_a, 4 * m).view(torch.int32)
        assert torch.equal(sel.long(), inv[caller]), "the L1 head's rows are not the inverse gather permutation at the caller's rows"
        x, w = rows(x_a, n, cin), f32(w_a, cin * c).view(cin, c)
        t = snap(t_a, 2 * m * c).view(torch.float16).view(m, c).double()
        rc = self.real.osb_l1_head_fwd(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_l1_head_fwd'] += 1
        words = snap(s_a, 4 * m * (c // 16)).view(torch.int32).view(m, c // 16)
        S = LR.decode(words, c)
        got = dict(loss=f32(loss_a, 1)[0])
        ref = LR.head(x, w, t, sel, signs=S)
        assert not self.l1_fails(got, ref, S), "the L1 head's loss or signs are outside their bounds"
        self.worst['l1-loss'] = max(self.worst['l1-loss'], LR.ratio(got['loss'], *ref['loss']))
        if not self.neg['l1_rows_through_perm']:
            assert self.l1_fails(got, LR.head(x, w, t, perm[caller], signs=S), S), "negative control: rows through perm passed"
            self.neg['l1_rows_through_perm'] += 1
        if not self.neg['l1_targets_rolled']:
            assert self.l1_fails(got, LR.head(x, w, t.roll(1, 0), sel, signs=S), S), "negative control: rolled targets passed"
            self.neg['l1_targets_rolled'] += 1
        self.l1 = dict(args=(x_a, n, cin, w_a, c, rows_a, m, s_a), x=x, w=w, t=t, sel=sel, words=words, S=S)
        return 0

    def _l1_head_bwd(self, *args):
        a = [_i(v) for v in args]
        x_a, n, cin, w_a, c, rows_a, m, s_a, g_a, dx_a, dw_a = a[:11]
        torch.cuda.synchronize()
        F = self.l1
        assert F and F['args'] == (x_a, n, cin, w_a, c, rows_a, m, s_a), \
            "the L1 backward does not read its forward's rows, weights, row index and signs"
        assert torch.equal(rows(x_a, n, cin), F['x']) and torch.equal(f32(w_a, cin * c).view(cin, c), F['w']), \
            "the L1 head's rows or weights changed between forward and backward"
        assert torch.equal(snap(rows_a, 4 * m).view(torch.int32), F['sel'])
        assert torch.equal(snap(s_a, 4 * m * (c // 16)).view(torch.int32).view(m, c // 16), F['words']), \
            "the L1 signs changed between forward and backward"
        g = float(f32(g_a, 1))
        assert g == self.l1_caller[2], f"the L1 backward reads g = {g}, not the upstream gradient {self.l1_caller[2]}"
        rc = self.real.osb_l1_head_bwd(*args)
        torch.cuda.synchronize()
        if rc:
            return rc
        self.counts['osb_l1_head_bwd'] += 1
        dx = rows(dx_a, n, cin)
        r = F['sel'].long()
        others = torch.ones(n, dtype=torch.bool, device=dev)
        others[r] = False
        assert bool((dx[others] == 0).all()), "the L1 dx is not 0 on the unsupervised rows"
        dw = f32(dw_a, cin * c).view(cin, c)
        got = dict(dx=dx[r], dW=dw)
        ref = LR.head(F['x'], F['w'], F['t'], F['sel'], signs=F['S'], g=g)
        for k, v in got.items():
            q = LR.ratio(v, *ref[k])
            assert q <= 1, f"l1-{k}: {q:.3g} of the bound"
            self.worst['l1-' + k] = max(self.worst['l1-' + k], q)
        if not self.neg['l1_g_one']:
            assert self.l1_fails(got, LR.head(F['x'], F['w'], F['t'], F['sel'], signs=F['S'], g=1.0)), "negative control: g = 1 passed"
            self.neg['l1_g_one'] += 1
        self.l1['dW'] = dw
        self.l1_dx_readers = {'osb_bn_backward_reduce': dx_a, 'osb_bn_backward_apply': dx_a}
        self.written.add(dx_a)
        return 0

    def cos_gradient_read(self, name, g_a):
        """the first BatchNorm backward reduce / apply after the L1 backward reads its dx as g"""
        super().cos_gradient_read(name, g_a)
        want = self.l1_dx_readers.pop(name, None)
        if want is not None:
            assert g_a == want, f"{name}: the first BatchNorm backward does not read the L1 head's dx"


def main_l1():
    kind, arch, scene = cfg.split(':')[:3]
    assert kind == 'l1', cfg
    head = int(cfg.split(':')[3]) if cfg.count(':') > 2 else 768
    model = synth.build_model(arch, head, seed=0).to(dev).train()
    H = L1Harness(model)
    C.lib = lambda: H
    C.call = H.call
    coords = torch.from_numpy(synth.scene(scene)).to(dev)
    n = coords.shape[0]
    gen = torch.Generator(device=dev).manual_seed(1)
    feats = torch.rand(n, 3, device=dev, generator=gen)
    eng = engine.FusedMinkUNet(model, batch_stats=True)
    bns = [nm for nm, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm1d)]
    caller = (torch.arange(n, device=dev) % 7 == 0).nonzero().squeeze(1)
    feat = torch.randn(caller.numel(), head, device=dev, generator=gen).half()
    H.l1_caller = (caller, feat, 0.75)
    mask = torch.zeros(n, dtype=torch.bool, device=dev)
    mask[caller] = True
    loss = eng.forward_train_l1(coords, feats, feat, mask)
    assert sorted(s['bn'] for s in H.stats) == sorted(bns), "not exactly one statistics launch per BatchNorm"
    (0.75 * loss).backward()
    torch.cuda.synchronize()
    mods = dict(model.named_modules())
    for nm in bns:
        dw, db = H.reduce_last[nm]
        assert torch.equal(dw, mods[nm].weight.grad) and torch.equal(db, mods[nm].bias.grad), f"{nm}: dweight / dbias not in its gradient slot"
    assert H.counts['osb_l1_head_fwd'] == H.counts['osb_l1_head_bwd'] == 1, dict(H.counts)
    assert not H.l1_dx_readers, f"no BatchNorm backward read the L1 dx: {sorted(H.l1_dx_readers)}"
    assert torch.equal(H.l1['w'], model.final.kernel.detach().view(H.l1['w'].shape))
    assert torch.equal(H.l1['dW'], model.final.kernel.grad.view(H.l1['dW'].shape)), "the L1 dW is not final.kernel.grad"
    print('SLOTS every BatchNorm\'s dweight / dbias and the L1 dW equal their .grad bit for bit', flush=True)
    print('CONFIG', cfg, 'rows', n, 'supervised', caller.numel(), 'BatchNorms', len(bns), flush=True)
    print('COUNTS', dict(H.counts), flush=True)
    for op, r in sorted(H.worst.items()):
        print('WORST %-16s %.3f of the bound' % (op, r), flush=True)
    downsample = any(A['res_bn'] for A in H.applies)
    assert H.neg['swapped_form'] == H.neg['own_bn_on_downsample'] == (1 if downsample else 0), dict(H.neg)
    assert H.neg['dropped_mask'] == 1, dict(H.neg)
    assert [H.neg[k] for k in ('l1_rows_through_perm', 'l1_targets_rolled', 'l1_g_one')] == [1, 1, 1], dict(H.neg)
    print('NEGATIVE controls failed as they must:', dict(H.neg), flush=True)
    print('OK')


main_l1()
'''

CONFIGS = [
    'l1:MinkUNet34C:config1_50k',                      # the shipped distillation shape: 768-wide head on 96 channels
    'l1:MinkUNet14D:config1_50k:512',                  # cin 384: the head's largest shared-memory plan
]


def _run(cfg, timeout=900):
    script = _BASE % {'root': ROOT} + L1_WORKER
    r = subprocess.run([sys.executable, '-c', script, cfg], capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-4000:], r.stderr[-3000:])
    assert r.returncode == 0 and r.stdout.rstrip().endswith('OK'), r.stdout[-2500:] + r.stderr[-2500:]


@pytest.mark.parametrize('cfg', CONFIGS)
def test_l1_replay(cfg):
    _run(cfg)


@pytest.mark.parametrize('arch', ARCHS)
def test_l1_replay_every_architecture(arch):
    _run(f'l1:{arch}:tiny')
