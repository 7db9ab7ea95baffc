"""When each launch of the L1 distillation step reads its inputs, relative to the launch that produces them: the free-running
against serialised harness of tests/test_gpu_launch_order.py (its worker script, ``Wrapper``, poisoning and comparisons,
imported), with the L1 head's sign state filled with 0xFF (code 3, never written by the kernel) before
``osb_l1_head_fwd`` writes it.  Cases, one subprocess each:

  * free against serialised, every reused buffer poisoned: ``forward_train_l1`` + ``(0.75 * loss).backward()``, and
    ``distill.fused_l1_step`` with a bound Adam followed by the next L1 loss, each twice on the same engine;
  * one engine through ``tiny -> config1_50k -> tiny -> config2_200k -> config1_50k`` against a fresh serialised engine per
    scene;
  * the step run/distill.py makes with the L1 loss (voxeliser, batch-statistics forward, device validation,
    ``fused_l1_step`` with a bound Adam, the next L1 loss) on a side stream while the legacy default stream sleeps;
  * the PDL window rule (tests/launch_order.py) on every free-running launch sequence.

Negative control, on the test side only: the signs poisoned between forward and backward; the outputs must then differ."""
import subprocess
import sys

import pytest

from tests.test_gpu_launch_order import ROOT, WORKER

pytestmark = pytest.mark.gpu

_BASE = WORKER.rstrip()
assert _BASE.endswith('\nmain()')
_BASE = _BASE[:-len('main()')]

L1_WORKER = r'''
POISON_L1_SIGNS_IN_BACKWARD = [False]
W.l1_signs = None                                        # (pointer, bytes) of the latest L1 sign state
_getattr = Wrapper.__getattr__


def _l1_getattr(self, name):
    fn = _getattr(self, name)
    if name != 'osb_l1_head_fwd':
        return fn

    def run(*a):
        self.l1_signs = (LO.ival(a[8]), 4 * LO.ival(a[6]) * (LO.ival(a[4]) // 16))
        self.poison_raw(*self.l1_signs)
        return fn(*a)
    return run


Wrapper.__getattr__ = _l1_getattr
_bwd_poisoned = engine_train._run_backward


def _l1_run_backward(eng, *a):
    if POISON_L1_SIGNS_IN_BACKWARD[0]:
        W.poison_raw(*W.l1_signs)
    return _bwd_poisoned(eng, *a)


engine_train._run_backward = _l1_run_backward
_run_case = run_case


def run_case(case, arch, scene, mode, eng=None, model=None):
    if case not in ('l1', 'l1_adam'):
        return _run_case(case, arch, scene, mode, eng, model)
    coords, feats, labels, gout = inputs(scene)
    if eng is None:
        model, eng = make(arch, True, 768)
    set_mode(eng, mode)
    out = {}
    rows = torch.arange(coords.shape[0], device=dev) % 7 == 0
    for it in range(2):
        if case == 'l1':
            model.zero_grad(set_to_none=True)
            loss = eng.forward_train_l1(coords, feats, target(scene, rows), rows)
            (0.75 * loss).backward()
        else:
            if it == 0:
                opt = optim.Adam(model.parameters(), lr=1e-3)
                opt.bind(eng)
            loss = distill.fused_l1_step(eng, opt, coords, feats, target(scene, rows), rows, translate=False)
            out.update({f'{it} param {k}': cl(p) for k, p in model.named_parameters()})
            out[f'{it} next loss'] = cl(eng.forward_train_l1(coords, feats, target(scene, rows), rows))
        out[f'{it} loss'] = cl(loss)
        out.update({f'{it} {k}': v for k, v in state(model).items()})
    torch.cuda.synchronize()
    return out


def l1_step_all(arch, scene, mode):
    """the step run/distill.py makes with the L1 loss: the voxeliser, a batch-statistics forward with a device validation,
    distill.fused_l1_step with a bound Adam, then the next L1 loss"""
    coords, feats, labels, gout = inputs(scene)
    pts, vox = synth.scene_points('tiny')
    P = torch.from_numpy(pts).to(dev)
    M = np.diag([1 / vox, 1 / vox, 1 / vox, 1.0])
    model, eng = make(arch, True, 768)
    text = torch.from_numpy(synth.text_embeddings(20)).to(dev)
    torch.cuda.synchronize()

    def body():
        set_mode(eng, mode)
        out = {}
        cv, inds, inv, mn = voxelize.voxelize_points(P, M)
        out.update({'vox coords': cv, 'vox inds': inds, 'vox inv': inv})
        with torch.no_grad():
            y = eng(coords, feats)
        out['bs out'] = y
        val = distill.DeviceValidation(text, 20, 255)
        val.add(y, None, labels)
        out['validation'] = torch.tensor(val.end(), dtype=torch.float64)
        rows = torch.arange(coords.shape[0], device=dev) % 7 == 0
        opt = optim.Adam(model.parameters(), lr=1e-3)
        opt.bind(eng)
        out['train loss'] = distill.fused_l1_step(eng, opt, coords, feats, target(scene, rows), rows, translate=False)
        out.update(state(model))
        out.update({'param ' + k: cl(p) for k, p in model.named_parameters()})
        out['next loss'] = cl(eng.forward_train_l1(coords, feats, target(scene, rows), rows))
        return out
    return body


def main_l1():
    arch = 'MinkUNet34C'
    if cfg == 'l1_train':
        for case in ('l1', 'l1_adam'):
            ref = free_vs_serial(case, arch, 'config1_50k')
            if case == 'l1':
                POISON_L1_SIGNS_IN_BACKWARD[0] = True
                bad = run_case(case, arch, 'config1_50k', 'free')
                POISON_L1_SIGNS_IN_BACKWARD[0] = False
                W.seq = []
                k = same(bad, ref, 'negative control', allow_nonfinite=True)
                assert k is not None, "negative control: the L1 signs poisoned between forward and backward were not detected"
                print('NEGATIVE control failed as it must: L1 signs poisoned before the backward ->', k, 'differs', flush=True)
    elif cfg == 'l1_interleave':
        order = ['tiny', 'config1_50k', 'tiny', 'config2_200k', 'config1_50k']
        a = 'MinkUNet18A'
        refs = {sc: run_case('l1', a, sc, 'serial') for sc in sorted(set(order))}
        W.seq = []
        model, eng = make(a, True, 768)
        for sc in order:
            got = {k: v for k, v in run_case('l1', a, sc, 'free', eng, model).items() if 'buffer' not in k}
            must_equal(got, {k: v for k, v in refs[sc].items() if 'buffer' not in k}, f'interleaved l1 {sc}')
        windows()
        print('OK interleaved l1', a, ' -> '.join(order), '== a fresh serialised engine per scene', flush=True)
    elif cfg == 'l1_stream':
        ref = l1_step_all('MinkUNet18A', 'config1_50k', 'serial')()
        W.seq = []
        got = on_side_stream(l1_step_all('MinkUNet18A', 'config1_50k', 'free'))
        windows()
        must_equal(got, ref, 'L1 training iteration on a side stream behind a sleeping default stream')
        print('OK side stream L1 iteration (voxeliser, batch statistics, validation, fused_l1_step, Adam, next loss)',
              flush=True)
    else:
        raise ValueError(cfg)
    torch.cuda.synchronize()
    print('CONFIG', cfg, flush=True)
    print('STATS', dict(W.stats), dict(COMPARED), flush=True)
    print('TIME %.1f s' % (time.time() - T0), flush=True)
    print('OK')


main_l1()
'''

CONFIGS = ['l1_train', 'l1_interleave', 'l1_stream']


def _run(cfg, timeout=1200):
    script = _BASE % {'root': ROOT} + L1_WORKER
    r = subprocess.run([sys.executable, '-c', script, cfg], capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-5000:], r.stderr[-3000:])
    assert r.returncode == 0 and r.stdout.rstrip().endswith('OK'), r.stdout[-2500:] + r.stderr[-2500:]


@pytest.mark.parametrize('cfg', CONFIGS)
def test_l1_launch_order(cfg):
    _run(cfg)
