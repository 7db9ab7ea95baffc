"""Fused inference engine (tensor-core path end to end) against the reference-topology golden activations and
against the module-by-module surface.  Tolerance 1e-3 relative per point (north star); observed ~1e-5."""
import numpy as np
import pytest
import torch

from openscene_b200 import synth
from tests.util import golden, rel_row_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.mark.parametrize('arch', ['MinkUNet18A', 'MinkUNet34C'])
def test_engine_matches_reference_golden(arch):
    from openscene_b200 import engine
    g = golden(f'unet_{arch}.npz')
    model = synth.build_model(arch, 768, seed=0).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    out = eng(torch.from_numpy(g['coords']).to(DEV), torch.from_numpy(g['feats']).to(DEV)).cpu().numpy()
    err = rel_row_err(out[g['rows']], g['out_rows'])
    print(arch, 'engine rel err', err)
    assert err < 1e-3
    assert np.allclose(np.linalg.norm(out, axis=1), g['row_norm'], rtol=1e-3)


def test_engine_equals_module_path_on_batched_scene_and_odd_head():
    import MinkowskiEngine as ME
    from openscene_b200 import engine
    c = synth.random_cloud(3000, 36, seed=4, batch=3)
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(2))
    for arch, head in (('MinkUNet14A', 512), ('MinkUNet18B', 20)):
        model = synth.build_model(arch, head, seed=3).eval().to(DEV)
        with torch.no_grad():
            ref = model(ME.SparseTensor(f.to(DEV), torch.from_numpy(c).to(DEV)))
        out = engine.FusedMinkUNet(model)(torch.from_numpy(c).to(DEV), f.to(DEV))
        assert out.shape == ref.shape
        assert rel_row_err(out.cpu().numpy(), ref.cpu().numpy()) < 1e-3


def test_engine_refuses_train_mode():
    from openscene_b200 import engine
    model = synth.build_model('MinkUNet14A', 64, seed=0).to(DEV).train()
    with pytest.raises(RuntimeError, match='eval'):
        engine.FusedMinkUNet(model)


def test_engine_follows_weight_changes():
    """The engine's packed weights / folded BatchNorm are copies: in-place updates and load_state_dict must show up in the next
    forward, and a head folded from the old weights must be refused (ADVICE r1: stale outputs with no error)."""
    import MinkowskiEngine as ME
    from openscene_b200 import engine
    c = torch.from_numpy(synth.random_cloud(2500, 40, seed=6)).to(DEV)
    f = torch.rand(c.shape[0], 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    model = synth.build_model('MinkUNet14A', 64, seed=1).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    text = torch.nn.functional.normalize(torch.randn(8, 64, device=DEV), dim=1)
    head = eng.fold_head(text)
    out0 = eng(c, f)
    with torch.no_grad():
        model.final.kernel.mul_(1.5)                                     # optimiser-style in-place update
        model.bn0.bn.running_mean.add_(0.05)                             # a buffer, not a parameter
        model.block2[0].conv1.kernel.add_(0.01)
        ref = model(ME.SparseTensor(f, c))
    out1 = eng(c, f)
    assert rel_row_err(out1.cpu().numpy(), ref.cpu().numpy()) < 1e-3
    assert rel_row_err(out1.cpu().numpy(), out0.cpu().numpy()) > 1e-2   # it really changed
    with pytest.raises(RuntimeError, match='fold_head again'):
        eng.forward_scores(c, f, head)
    other = synth.build_model('MinkUNet14A', 64, seed=2).state_dict()
    model.load_state_dict(other)
    with torch.no_grad():
        ref2 = model(ME.SparseTensor(f, c))
    assert rel_row_err(eng(c, f).cpu().numpy(), ref2.cpu().numpy()) < 1e-3


def test_folded_head_scores_match_materialised_path():
    """engine.forward_scores (final conv folded with the text matrix) against normalise + match on the 768-d features."""
    from openscene_b200 import engine, matching
    c = torch.from_numpy(synth.scene('tiny')).to(DEV)
    f = torch.rand(c.shape[0], 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    model = synth.build_model('MinkUNet18A', 768, seed=0).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    text = torch.from_numpy(synth.text_embeddings(20)).to(DEV)
    s_ref, l_ref, m_ref = matching._scores(eng(c, f), None, text, normalize=True, want_smax=True)
    s, l, m = eng.forward_scores(c, f, eng.fold_head(text.float()))
    assert s.shape == s_ref.shape and s.dtype == torch.float16
    assert (s.float() - s_ref.float()).abs().max() < 2e-3          # both are fp16 roundings of the same cosine
    assert (l == l_ref).float().mean() > 0.99
    assert torch.equal(l, s.float().max(1)[1])


def test_steady_state_makes_no_device_allocations():
    """A serving loop (GC disabled, as in bench.py) must not grow device memory: no reference cycles holding kernel maps,
    one grow-only activation arena.  Regression test for 10-120 ms cudaMalloc stalls inside steps."""
    import gc
    from openscene_b200 import engine, matching
    c = torch.from_numpy(synth.scene('tiny')).to(DEV)
    f = torch.ones(c.shape[0], 3, device=DEV)
    text = torch.from_numpy(synth.text_embeddings(20)).to(DEV)
    eng = engine.FusedMinkUNet(synth.build_model('MinkUNet18A', 768, seed=0).eval().to(DEV))
    step = lambda: matching._scores(eng(c, f), None, text, normalize=True)
    for _ in range(5):
        step()
    torch.cuda.synchronize()
    gc.collect(); gc.disable()
    try:
        before = torch.cuda.memory_stats()['num_device_alloc']
        reserved = torch.cuda.memory_reserved()
        for _ in range(40):
            step()
        torch.cuda.synchronize()
        assert torch.cuda.memory_stats()['num_device_alloc'] == before
        assert torch.cuda.memory_reserved() == reserved
    finally:
        gc.enable()


def test_occupancy_grid_and_hash_engines_are_bit_identical(monkeypatch):
    """Stem probes and kernel maps through the occupancy grid or the hash table: same maps, same accumulation order."""
    from openscene_b200 import engine
    c = synth.scene('config1_50k')
    f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(5))
    model = synth.build_model('MinkUNet18A', 96, seed=1).eval().to(DEV)
    eng = engine.FusedMinkUNet(model)
    outs = {}
    for flag in ('1', '0'):
        monkeypatch.setenv('OSB_OCCGRID', flag)
        outs[flag] = eng(torch.from_numpy(c).to(DEV), f.to(DEV)).clone()
        assert (eng.last_cm.sets[1].grid is not None) == (flag == '1')
    assert torch.equal(outs['1'], outs['0'])
