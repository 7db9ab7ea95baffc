"""When each launch of the fused engine reads its inputs, relative to the launch that produces them.

The replays (tests/test_gpu_launch_replay.py, tests/test_gpu_norm_replay.py) synchronise around every launch, so they pin
what a launch computes but cannot see one that reads too early; repeated calls on the same scene read stale buffers that
happen to hold the right numbers.  Here the library seen by the engine is a wrapper with two modes:

  * serialised (the reference): ``torch.cuda.synchronize()`` after every device entry point, the engine built with
    ``use_pdl = False``;
  * free: pass-through, recording every entry point, its arguments and its PDL flag.

Both run under poison: every byte of the engine's reused buffers is set to 0xFF (NaN in fp32 and in both bf16 halves of a
split row, -1 = "no row" in int32 / int64 indices) at the start of every forward (the activation arena, the split-K
workspace, the batch-statistics and cross-entropy workspaces, the gradient-row chunks) and of every backward (the same but
the arena, which holds the saved activations, plus the weight-gradient workspaces).  The chain's grid-barrier words are
never poisoned (their generation is carried from launch to launch); every poisoned range is checked against them.  A read
that overtakes its producer then reads NaN, or the previous scene's rows, and every comparison is bitwise with every output
finite.  The cosine head's per-row state is filled with 0xFF before ``osb_cos_head_fwd`` writes it.  Cases, one subprocess
each:

  * free against serialised: eval on the persistent chain and with ``OSB_CHAIN=0``, ``forward_scores`` with a folded head,
    the batch-statistics forward, ``forward_train`` + backward (row mask, all rows), ``forward_train_ce`` + backward, an Adam
    step with its in-place re-pack followed by the next forward, ``forward_train_cosine`` + ``(0.75 * loss).backward()``, and
    ``distill.fused_cosine_step`` with a bound Adam followed by the next cosine loss;
  * one engine through ``tiny -> config1_50k -> tiny -> config2_200k -> config1_50k`` (eval and training) against a fresh
    engine per scene;
  * the whole step on a side stream while the legacy default stream sleeps, with ``forward_train`` and with the cosine step
    run/distill.py makes: work that lands on the default stream queues behind the sleep and its consumer reads poison;
  * plan switches: order-only ones (``OSB_PDL``, ``OSB_PYRAMID``, ``OSB_OCCGRID``) bitwise across settings, the others
    (``OSB_DENSE_UP``, ``OSB_CHAIN_MAX_TILES``, ``OSB_TC_LAZY``, the chain grid) free against serialised per setting;
  * the PDL window rule (tests/launch_order.py) on every free-running launch sequence.

Negative controls change only the test side: the arena poisoned between forward and backward, the cosine state poisoned
between forward and backward, and one mid-network ``osb_conv_fwd_tc`` routed to the legacy stream behind the sleep."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import collections, os, sys, time
cfg = sys.argv[1]
for kv in sys.argv[2:]:
    k, v = kv.split('=')
    os.environ[k] = v
sys.path.insert(0, %(root)r)
import numpy as np
import torch
from openscene_b200 import distill, engine, engine_train, optim, synth, tc, voxelize, _cabi as C
from tests import launch_order as LO

dev = torch.device('cuda:0')
REAL = C.lib()
T0 = time.time()


class _Raw:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {'shape': (nbytes,), 'typestr': '|u1', 'data': (ptr, False), 'version': 3}


class Wrapper:
    """the library as the engine sees it: serialised or free-running, recording, poisoning"""

    def __init__(self):
        self.mode = 'free'
        self.seq = []
        self.stats = collections.Counter()
        self.fwd_eng = None              # engine whose forward has started: poison at its first row gather
        self.bwd = False
        self.wg_seen = set()
        self.reroute = None              # index of the osb_conv_fwd_tc call to send to the legacy stream (negative control)
        self.n_conv = 0
        self.gbars = []
        self.cos_state = None            # (pointer, bytes) of the latest cosine head state

    def __getattr__(self, name):
        fn = getattr(REAL, name)
        if LO.is_host_only(name):
            return fn

        def run(*a):
            if name == 'osb_gather_rows_f32' and self.fwd_eng is not None:
                eng, self.fwd_eng = self.fwd_eng, None
                self.poison_engine(eng, arena=True)
            if name == 'osb_conv_wgrad_tc' and self.bwd:
                p, nb = LO.ival(a[9]), LO.ival(a[10])
                if p and p not in self.wg_seen:
                    self.wg_seen.add(p)
                    self.poison_raw(p, nb)
            if name == 'osb_cos_head_fwd':
                self.cos_state = (LO.ival(a[8]), 24 * LO.ival(a[6]))
                self.poison_raw(*self.cos_state)
            L = LO.launch_of(name, a)
            self.seq.append(L)
            self.stats['launches'] += 1
            self.stats['PDL launches'] += int(L.pdl)
            if name == 'osb_conv_fwd_tc':
                if self.reroute is not None and self.n_conv == self.reroute:
                    a = list(a[:-1]) + [None]                    # the legacy default stream
                    self.stats['rerouted'] += 1
                self.n_conv += 1
            rc = fn(*a)
            if self.mode == 'serial':
                torch.cuda.synchronize()
                self.seq.append(LO.Launch('host synchronise', False))
            return rc
        return run

    def call(self, name, *a):
        C.check(getattr(self, name)(*a), name)

    # ------------------------------------------------------------------ poison
    def _guard(self, lo, hi):
        for g in self.gbars:
            glo = g.data_ptr()
            assert hi <= glo or glo + g.numel() * g.element_size() <= lo, "a poisoned range covers the grid-barrier words"

    def poison(self, t):
        if t is None or t.numel() == 0:
            return
        b = t.view(-1).view(torch.uint8)
        self._guard(b.data_ptr(), b.data_ptr() + b.numel())
        b.fill_(255)
        self.stats['bytes poisoned'] += b.numel()

    def poison_raw(self, p, nb):
        self._guard(p, p + nb)
        torch.as_tensor(_Raw(p, nb), device=dev).fill_(255)
        self.stats['bytes poisoned'] += nb

    def poison_engine(self, eng, arena):
        self.gbars = [ch.gbar for ch in [eng._chain] + list(tc._CHAINS.values()) if ch is not None]
        if arena:
            self.poison(eng._arena)
        self.poison(eng._bs_ws)
        self.poison(eng._ws)
        self.poison(eng._ce_ws)
        for t in eng._garena:
            self.poison(t)


W = Wrapper()
C.lib = lambda: W
C.call = W.call
tc._CHAINS.clear()
tc._PACK_CACHE.clear()
POISON_ARENA_IN_BACKWARD = [False]
POISON_COS_STATE_IN_BACKWARD = [False]

_fwd = engine.FusedMinkUNet._forward


def _forward(self, *a):
    W.fwd_eng = self
    return _fwd(self, *a)


engine.FusedMinkUNet._forward = _forward
_run_forward = engine_train._run_forward


def run_forward(eng, *a, **k):
    W.fwd_eng = eng
    return _run_forward(eng, *a, **k)


engine_train._run_forward = run_forward
_run_backward = engine_train._run_backward


def run_backward(eng, *a):
    W.poison_engine(eng, arena=POISON_ARENA_IN_BACKWARD[0])
    if POISON_COS_STATE_IN_BACKWARD[0]:
        W.poison_raw(*W.cos_state)
    W.bwd, W.wg_seen = True, set()
    try:
        return _run_backward(eng, *a)
    finally:
        W.bwd = False


engine_train._run_backward = run_backward

# ---------------------------------------------------------------------- inputs and cases
_SCENES = {}


def inputs(scene):
    if scene not in _SCENES:
        coords = torch.from_numpy(synth.scene(scene)).to(dev)
        n = coords.shape[0]
        g = torch.Generator(device=dev).manual_seed(1)
        feats = torch.rand(n, 3, device=dev, generator=g)
        labels = torch.randint(0, 20, (n,), device=dev, generator=g)
        labels[::9] = 255
        _SCENES[scene] = (coords, feats, labels, torch.randn(n, 96, device=dev, generator=g))
    return _SCENES[scene]


def target(scene, rows):
    """fp16 distillation targets of the rows selected by the mask rows"""
    key = ('target', scene)
    if key not in _SCENES:
        g = torch.Generator(device=dev).manual_seed(2)
        _SCENES[key] = torch.randn(rows.numel(), 768, device=dev, generator=g).half()
    return _SCENES[key][rows]


def make(arch, train, head=768):
    model = synth.build_model(arch, head, seed=0).to(dev)
    model.train() if train else model.eval()
    eng = engine.FusedMinkUNet(model, batch_stats=train)
    return model, eng


def set_mode(eng, mode):
    W.mode = mode
    eng.use_pdl = eng.use_pdl and mode == 'free'


def cl(t):
    return t.detach().clone()


def state(model, grads=True):
    out = {}
    for n, p in model.named_parameters():
        if grads and p.grad is not None:
            out['grad ' + n] = cl(p.grad)
    for n, b in model.named_buffers():
        out['buffer ' + n] = cl(b)
    return out


def run_case(case, arch, scene, mode, eng=None, model=None):
    """-> {name: tensor} of one case, run twice on the same engine (the second run reuses every buffer)"""
    coords, feats, labels, gout = inputs(scene)
    train = case not in ('eval', 'scores')
    if eng is None:
        model, eng = make(arch, train, 20 if case == 'ce' else (96 if case in ('train_mask', 'train_all', 'adam') else 768))
    set_mode(eng, mode)
    out = {}
    n = coords.shape[0]
    rows = None if case == 'train_all' else (torch.arange(n, device=dev) %% 7 == 0)
    for it in range(2):
        if case == 'eval':
            out[f'{it} out'] = eng(coords, feats)
        elif case == 'scores':
            folded = eng.fold_head(torch.from_numpy(synth.text_embeddings(20)).float().to(dev))
            s, lab, smax = eng.forward_scores(coords, feats, folded)
            out.update({f'{it} scores': s, f'{it} label': lab, f'{it} smax': smax})
        elif case == 'bs':
            out[f'{it} out'] = eng(coords, feats)
        elif case in ('train_mask', 'train_all', 'adam'):
            model.zero_grad(set_to_none=True)
            y = eng.forward_train(coords, feats, rows=rows)
            y.backward(gout[:y.shape[0]] if rows is None else gout[rows])
            out[f'{it} out'] = cl(y)
            out.update({f'{it} {k}': v for k, v in state(model).items()})
            if case == 'adam':
                opt = optim.Adam(model.parameters(), lr=1e-3)
                opt.bind(eng)
                opt.step()
                out.update({f'{it} param {k}': cl(p) for k, p in model.named_parameters()})
                y = eng.forward_train(coords, feats, rows=rows)
                out[f'{it} next out'] = cl(y)
        elif case == 'cos':
            model.zero_grad(set_to_none=True)
            loss = eng.forward_train_cosine(coords, feats, target(scene, rows), rows)
            (0.75 * loss).backward()
            out[f'{it} loss'] = cl(loss)
            out.update({f'{it} {k}': v for k, v in state(model).items()})
        elif case == 'cos_adam':
            if it == 0:
                opt = optim.Adam(model.parameters(), lr=1e-3)
                opt.bind(eng)
            loss = distill.fused_cosine_step(eng, opt, coords, feats, target(scene, rows), rows, translate=False)
            out[f'{it} loss'] = cl(loss)
            out.update({f'{it} {k}': v for k, v in state(model).items()})
            out.update({f'{it} param {k}': cl(p) for k, p in model.named_parameters()})
            out[f'{it} next loss'] = cl(eng.forward_train_cosine(coords, feats, target(scene, rows), rows))
        elif case == 'ce':
            model.zero_grad(set_to_none=True)
            loss, pred = eng.forward_train_ce(coords, feats, labels, 255)
            loss.backward()
            out.update({f'{it} loss': cl(loss), f'{it} pred': pred})
            out.update({f'{it} {k}': v for k, v in state(model).items()})
        else:
            raise ValueError(case)
    if case in ('bs',):
        out.update(state(model, grads=False))
    torch.cuda.synchronize()
    return out


COMPARED = collections.Counter()


def same(a, b, what, allow_nonfinite=False):
    assert a.keys() == b.keys(), (what, sorted(set(a) ^ set(b))[:5])
    for k in a:
        x, y = a[k], b[k]
        assert x.shape == y.shape and x.dtype == y.dtype, (what, k)
        if x.is_floating_point():
            assert allow_nonfinite or bool(torch.isfinite(x).all()), f"{what}: {k} is not finite"
            iv = {2: torch.int16, 4: torch.int32, 8: torch.int64}[x.element_size()]
            ok = torch.equal(x.view(iv), y.view(iv))
        else:
            ok = torch.equal(x, y)
        if not ok:
            return k
        COMPARED['tensors compared bitwise'] += 1
    return None


def must_equal(a, b, what):
    k = same(a, b, what)
    assert k is None, f"{what}: {k} differs bitwise"


def windows():
    n_win, n_in, bad = LO.check_windows(W.seq)
    assert not bad, bad[:3]
    COMPARED['PDL windows checked'] += n_win
    COMPARED['launches in windows'] += n_in
    W.seq = []


def free_vs_serial(case, arch, scene):
    ref = run_case(case, arch, scene, 'serial')
    W.seq = []
    got = run_case(case, arch, scene, 'free')
    windows()
    must_equal(got, ref, f'{case} {arch} {scene}')
    print('OK free == serialised:', case, arch, scene, flush=True)
    return ref


# ---------------------------------------------------------------------- side stream
def on_side_stream(fn, sleep=True):
    """fn() on a fresh stream that waited for the default stream, while the default stream sleeps"""
    torch.cuda.synchronize()
    default = torch.cuda.current_stream()
    s = torch.cuda.Stream()
    s.wait_stream(default)
    if sleep:
        torch.cuda._sleep(200_000_000)                     # about 0.1 s at the H100's clocks
    with torch.cuda.stream(s):
        out = fn()
    default.wait_stream(s)
    torch.cuda.synchronize()
    return out


def train_step_all(arch, scene, mode, cos=False):
    """one training iteration as run/train_mink.py and run/distill.py make it: the voxeliser, a batch-statistics forward
    with a device validation, forward_train + backward, an Adam step with re-pack, the next forward.  cos: the step
    run/distill.py makes with the cosine loss, distill.fused_cosine_step with a bound Adam, then the next cosine loss"""
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
        if cos:
            rows = torch.arange(coords.shape[0], device=dev) %% 7 == 0
            opt = optim.Adam(model.parameters(), lr=1e-3)
            opt.bind(eng)
            out['train loss'] = distill.fused_cosine_step(eng, opt, coords, feats, target(scene, rows), rows, translate=False)
            out.update(state(model))
            out.update({'param ' + k: cl(p) for k, p in model.named_parameters()})
            out['next loss'] = cl(eng.forward_train_cosine(coords, feats, target(scene, rows), rows))
            return out
        model.zero_grad(set_to_none=True)
        y = eng.forward_train(coords, feats, rows=None)
        y.backward(gout[:, :1].expand(-1, 768).contiguous() if y.shape[1] == 768 else gout)
        out['train out'] = cl(y)
        out.update(state(model))
        opt = optim.Adam(model.parameters(), lr=1e-3)
        opt.bind(eng)
        opt.step()
        out.update({'param ' + k: cl(p) for k, p in model.named_parameters()})
        out['next out'] = cl(eng.forward_train(coords, feats, rows=None))
        return out
    return body


def main():
    kind = cfg
    arch = 'MinkUNet34C'
    if kind == 'eval_chain':
        ref = free_vs_serial('eval', arch, 'config2_200k')
        free_vs_serial('scores', arch, 'config2_200k')
        # the persistent chain on a side stream (no concurrent kernel: its grid barrier needs every SM)
        model, eng = make(arch, False)
        got = on_side_stream(lambda: run_case('eval', arch, 'config2_200k', 'free', eng, model), sleep=False)
        windows()
        must_equal(got, ref, 'eval chain on a side stream')
        print('OK side stream (chain, no sleep) == serialised default stream', flush=True)
    elif kind == 'eval_nochain':
        ref = free_vs_serial('eval', arch, 'config2_200k')
        free_vs_serial('scores', arch, 'config2_200k')
        model, eng = make(arch, False)
        got = on_side_stream(lambda: run_case('eval', arch, 'config2_200k', 'free', eng, model))
        windows()
        must_equal(got, ref, 'eval on a side stream behind a sleeping default stream')
        print('OK side stream behind the sleep == serialised default stream', flush=True)
        # negative control: one mid-network convolution on the legacy stream
        model, eng = make(arch, False)
        W.reroute, W.n_conv = 12, 0
        bad = on_side_stream(lambda: run_case('eval', arch, 'config2_200k', 'free', eng, model))
        W.reroute, W.seq = None, []
        assert W.stats['rerouted'] == 1
        k = same(bad, ref, 'negative control', allow_nonfinite=True)
        assert k is not None, "negative control: a convolution on the legacy stream behind the sleep was not detected"
        print('NEGATIVE control failed as it must: osb_conv_fwd_tc #12 on the legacy stream ->', k, 'differs', flush=True)
    elif kind == 'train':
        for case, a, sc in (('bs', arch, 'config1_50k'), ('train_mask', arch, 'config1_50k'), ('train_all', 'MinkUNet18A', 'tiny'),
                            ('ce', 'MinkUNet18A', 'config1_50k'), ('adam', arch, 'config1_50k'), ('cos', arch, 'config1_50k'),
                            ('cos_adam', arch, 'config1_50k')):
            ref = free_vs_serial(case, a, sc)
            if case == 'train_mask':
                POISON_ARENA_IN_BACKWARD[0] = True
                bad = run_case(case, a, sc, 'free')
                POISON_ARENA_IN_BACKWARD[0] = False
                W.seq = []
                k = same(bad, ref, 'negative control', allow_nonfinite=True)
                assert k is not None, "negative control: the arena poisoned between forward and backward was not detected"
                print('NEGATIVE control failed as it must: arena poisoned before the backward ->', k, 'differs', flush=True)
            if case == 'cos':
                POISON_COS_STATE_IN_BACKWARD[0] = True
                bad = run_case(case, a, sc, 'free')
                POISON_COS_STATE_IN_BACKWARD[0] = False
                W.seq = []
                k = same(bad, ref, 'negative control', allow_nonfinite=True)
                assert k is not None, "negative control: the cosine state poisoned between forward and backward was not detected"
                print('NEGATIVE control failed as it must: cosine state poisoned before the backward ->', k, 'differs', flush=True)
    elif kind == 'interleave':
        order = ['tiny', 'config1_50k', 'tiny', 'config2_200k', 'config1_50k']
        for case, a in (('eval', arch), ('train_mask', 'MinkUNet18A'), ('cos', 'MinkUNet18A')):
            refs = {sc: run_case(case, a, sc, 'serial') for sc in sorted(set(order))}
            W.seq = []
            model, eng = make(a, case != 'eval', 96 if case == 'train_mask' else 768)
            for sc in order:
                got = run_case(case, a, sc, 'free', eng, model)
                if case != 'eval':
                    got = {k: v for k, v in got.items() if 'buffer' not in k}       # running buffers moved by earlier scenes
                    ref = {k: v for k, v in refs[sc].items() if 'buffer' not in k}
                else:
                    ref = refs[sc]
                must_equal(got, ref, f'interleaved {case} {sc}')
            windows()
            print('OK interleaved', case, a, ' -> '.join(order), '== a fresh serialised engine per scene', flush=True)
    elif kind == 'stream_train':
        ref = train_step_all('MinkUNet18A', 'config1_50k', 'serial')()
        W.seq = []
        got = on_side_stream(train_step_all('MinkUNet18A', 'config1_50k', 'free'))
        windows()
        must_equal(got, ref, 'training iteration on a side stream behind a sleeping default stream')
        print('OK side stream training iteration (voxeliser, batch statistics, validation, step, Adam, next forward)',
              flush=True)
        ref = train_step_all('MinkUNet18A', 'config1_50k', 'serial', cos=True)()
        W.seq = []
        got = on_side_stream(train_step_all('MinkUNet18A', 'config1_50k', 'free', cos=True))
        windows()
        must_equal(got, ref, 'cosine training iteration on a side stream behind a sleeping default stream')
        print('OK side stream cosine iteration (voxeliser, batch statistics, validation, fused_cosine_step, Adam, next loss)',
              flush=True)
    elif kind == 'switches_order':
        from openscene_b200 import coords as CO
        results = {}
        for name, vals in (('OSB_PDL', '01'), ('OSB_PYRAMID', '01'), ('OSB_OCCGRID', '01')):
            for v in vals:
                os.environ[name] = v
                for case, a, sc in (('eval', arch, 'config1_50k'), ('train_mask', 'MinkUNet18A', 'config1_50k')):
                    got = run_case(case, a, sc, 'free')
                    windows()
                    key = (case, a, sc)
                    if key in results:
                        must_equal(got, results[key], f'{case} with {name}={v}')
                    else:
                        results[key] = got
                os.environ.pop(name)
                print('OK', name, '=', v, 'bitwise equal to the other settings', flush=True)
    elif kind == 'switches_kernel':
        for name, v in (('OSB_DENSE_UP', '0'), ('OSB_CHAIN_MAX_TILES', '0'), ('OSB_CHAIN_MAX_TILES', '1000000')):
            os.environ[name] = v
            free_vs_serial('eval', arch, 'config1_50k')
            if name == 'OSB_DENSE_UP':
                free_vs_serial('train_mask', 'MinkUNet18A', 'config1_50k')
            os.environ.pop(name)
            print('OK', name, '=', v, flush=True)
        os.environ['OSB_CHAIN'] = '0'
        for lazy in (0, 1, 2):
            tc.debug_set_tc(lazy=lazy)
            free_vs_serial('eval', arch, 'config1_50k')
            print('OK OSB_TC_LAZY =', lazy, flush=True)
        tc.debug_set_tc(lazy=1)
        os.environ.pop('OSB_CHAIN')
        for grid in (3, 148):
            tc.tuning_set('chain_grid', grid)
            free_vs_serial('eval', arch, 'config1_50k')
            print('OK chain grid', grid, '->', REAL.osb_conv_chain_grid(), 'CTAs', flush=True)
        tc.tuning_set('chain_grid', 0)
    else:
        raise ValueError(kind)
    torch.cuda.synchronize()
    print('CONFIG', cfg, ' '.join(sys.argv[2:]), flush=True)
    print('STATS', dict(W.stats), dict(COMPARED), flush=True)
    print('TIME %%.1f s' %% (time.time() - T0), flush=True)
    print('OK')


main()
'''

CONFIGS = ['eval_chain', 'eval_nochain', 'train', 'interleave', 'stream_train', 'switches_order', 'switches_kernel']


def _run(cfg, env=(), timeout=1200):
    args = [sys.executable, '-c', WORKER % {'root': ROOT}, cfg] + list(env)
    if cfg == 'eval_nochain':
        args.append('OSB_CHAIN=0')
    r = subprocess.run(args, capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-5000:], r.stderr[-3000:])
    assert r.returncode == 0 and r.stdout.rstrip().endswith('OK'), r.stdout[-2500:] + r.stderr[-2500:]


@pytest.mark.parametrize('cfg', CONFIGS)
def test_launch_order(cfg):
    _run(cfg)
