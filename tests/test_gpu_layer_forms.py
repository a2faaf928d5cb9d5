"""The layer forms (num_x2h, num_h2x, sync_twoup; reference models/uni_transformer.py:143-210) and forward(..., return_all=True)
(models/molopt_score_model.py:360-367) on the engine (run with -m gpu): against the CPU oracle, which is pinned bit for bit against
the unmodified reference for the same forms (tests/test_layer_forms.py), layer by layer against float64, and bit for bit against the
engine's own reduced paths (no ligand-free cache, no relevant-node restriction, no CUDA graph)."""
import math

import pytest
import torch

from oracle import layer_forms, layerwise, restate, synth
from oracle.make_layer_form_pins import LAYER_FORM_CONFIGS
from oracle.make_reference_pins import option_id

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _model(weight_seed, cfg):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg))
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))


@pytest.mark.parametrize('cfgd', LAYER_FORM_CONFIGS, ids=option_id)
def test_layer_form_vs_oracle(cfgd):
    """Forward (with the per-block lists of return_all), and a 6-step noise-tape chain against the oracle, at the tolerances of the
    other backbone options (tests/test_gpu_reference_golden.py::test_backbone_options_vs_oracle)."""
    torch.set_num_threads(16)
    model, sd = _model(2, cfgd)
    b = synth.make_batch(9, 3, n_protein=70, ligand_sizes=[12, 5, 9])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    want = layer_forms.forward(sd, cfgd, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr,
                           return_all=True)
    out = model(pp.to(DEV), b['protein_v'].to(DEV), b['batch_protein'].to(DEV), lp.to(DEV), b['init_ligand_v'].to(DEV),
                b['batch_ligand'].to(DEV), return_all=True)
    ei, want_ei = out['edge_index'].cpu(), tr['block_edge_index'][-1]
    if cfgd.get('cutoff_mode') == 'hybrid':           # the engine's slot list is destination-sorted; the edge SET must agree
        ei, want_ei = layerwise._sorted_edges(ei), layerwise._sorted_edges(want_ei)
    assert torch.equal(ei, want_ei)
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=1e-3)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=1e-4, atol=1e-4)
    nb = cfgd.get('num_blocks', 1)
    assert len(out['layer_pred_ligand_pos']) == len(out['layer_pred_ligand_v']) == nb + 1
    for g, w in zip(out['layer_pred_ligand_pos'], want['layer_pred_ligand_pos']):
        torch.testing.assert_close(g.cpu(), w, rtol=1e-4, atol=1e-5)
    for g, w in zip(out['layer_pred_ligand_v'], want['layer_pred_ligand_v']):
        torch.testing.assert_close(g.cpu(), w, rtol=0, atol=1e-3)
    assert torch.equal(out['layer_pred_ligand_pos'][-1], out['pred_ligand_pos'])
    assert torch.equal(out['layer_pred_ligand_v'][-1], out['pred_ligand_v'])
    if cfgd.get('num_h2x', 1) == 0:                   # x never moves
        assert all(torch.equal(p.cpu(), lp) for p in out['layer_pred_ligand_pos'])
    if cfgd.get('num_x2h', 1) == 0:                   # h never changes: the head sees the initial embeddings after every block
        assert all(torch.equal(v, out['layer_pred_ligand_v'][0]) for v in out['layer_pred_ligand_v'])
    S = 6
    pn, vu = synth.make_tape(4, S, len(b['batch_ligand']))
    w = layer_forms.sample_diffusion(sd, cfgd, *_args(b, 'cpu'), pn, vu, num_steps=S)
    got = model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', noise_tape=(pn, vu))
    assert torch.equal(torch.stack(got['v_traj']), torch.stack(w['v_traj']))
    torch.testing.assert_close(torch.stack(got['pos_traj']), torch.stack(w['pos_traj']), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(torch.stack(got['v0_traj']), torch.stack(w['v0_traj']), rtol=0, atol=1e-3)


@pytest.mark.parametrize('cfgd', LAYER_FORM_CONFIGS, ids=option_id)
def test_layer_form_every_layer_vs_float64(cfgd):
    """Every layer of the engine against oracle.layer_forms.LayerFormRef in float64 on the engine's own previous layer, within LAYER_TOL
    (block 0 of the form)."""
    torch.set_num_threads(16)
    cfg = dict(cfgd, num_blocks=1)
    sd = synth.make_state_dict(4, cfg, schedules=restate.make_schedules(cfg))
    b = synth.make_batch(12, 3, n_protein=80, ligand_sizes=[11, 3, 17])

    def make_model(c, s):
        from targetdiff_b200.config import default_model_config
        from targetdiff_b200.score_model import ScorePosNet3D
        mc = default_model_config()
        mc.update(c)
        m = ScorePosNet3D(mc, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
        m.load_state_dict(s, strict=True)
        return m.to(DEV)

    rows = layer_forms.engine_layer_parity(option_id(cfgd), cfg, sd, b, synth.DEFAULT_MODEL_CONFIG['num_layers'], make_model, DEV)
    th, tx = layerwise.LAYER_TOL['tc3']
    for r in rows:
        # with num_x2h = 0 (num_h2x = 0) the layer leaves h (x) as it is: layerwise.row_error is then 0 / 0 = nan on every row when the
        # engine's value equals the input exactly, and inf on a row where it does not
        if cfg.get('num_x2h', 1) > 0:
            assert r[1] <= th, 'layer %d: h %.3e (limit %.1e)' % (r[0], r[1], th)
        else:
            assert math.isnan(r[1]), 'layer %d: h moved (%.3e)' % (r[0], r[1])
        if cfg.get('num_h2x', 1) > 0:
            assert r[3] <= tx, 'layer %d: x %.3e (limit %.1e)' % (r[0], r[3], tx)
        else:
            assert math.isnan(r[3]), 'layer %d: x moved (%.3e)' % (r[0], r[3])


REDUCED_FORMS = [{'num_x2h': 2}, {'num_h2x': 2, 'sync_twoup': True}, {'num_x2h': 2, 'num_h2x': 3, 'sync_twoup': True, 'ew_net_type': 'r'}]


def _chain(monkeypatch, cfgd, env, b, pn, vu):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    model, _ = _model(3, cfgd)
    r = model.sample_diffusion(*_args(b), num_steps=pn.shape[0], center_pos_mode='protein', noise_tape=(pn, vu))
    for k in env:
        monkeypatch.delenv(k)
    return r


def _assert_same(a, r):
    assert torch.equal(a['pos'], r['pos']) and torch.equal(a['v'], r['v'])
    for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
        assert torch.equal(torch.stack(a[k]), torch.stack(r[k])), k


@pytest.mark.parametrize('cfgd', REDUCED_FORMS, ids=option_id)
def test_layer_form_reduced_paths_bit_identical(monkeypatch, cfgd):
    """The ligand-free cache (counted in x2h sub-layer evaluations, depths 1-3 and the default), the relevant-node restriction of the
    last x2h sub-layer and the CUDA-graph replay change no bit of the chain: it equals the one without cache (TDIFF_FREE_DEPTH=0),
    without restriction (TDIFF_NO_RESTRICT=1) and launched eagerly (TDIFF_NO_GRAPH=1)."""
    b = synth.make_batch(6, 4, n_protein=150, ligand_sizes=[20, 7, 33, 12])
    S = 8
    pn, vu = synth.make_tape(11, S, int(b['init_ligand_pos'].shape[0]))
    base = _chain(monkeypatch, cfgd, {'TDIFF_FREE_DEPTH': '0', 'TDIFF_NO_RESTRICT': '1', 'TDIFF_NO_GRAPH': '1'}, b, pn, vu)
    for env in ({}, {'TDIFF_FREE_DEPTH': '1'}, {'TDIFF_FREE_DEPTH': '2'}, {'TDIFF_FREE_DEPTH': '3'}, {'TDIFF_FREE_DEPTH': '0'},
                {'TDIFF_NO_RESTRICT': '1'}, {'TDIFF_NO_GRAPH': '1'}):
        _assert_same(base, _chain(monkeypatch, cfgd, env, b, pn, vu))


def _launches_per_step(cfgd, b):
    from targetdiff_b200 import _lib
    model, _ = _model(3, cfgd)
    lib = _lib.load()
    counts = []
    for S in (3, 5):
        model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', return_traj=False)
        eng = model.engine(DEV)
        counts.append(lib.tdiff_launch_count(eng))
        model._drop_engine()
    return counts


# Kernel launches of one sampling step of the default form (9 layers, k = 32, ligand-free cache depth 2) on the batch below, as the
# engine issued them before the layer forms existed (measured on an NVIDIA H100 80GB HBM3); the default form keeps that launch sequence.
DEFAULT_FORM_LAUNCHES_PER_STEP = 108


def test_default_form_launches_per_step():
    b = synth.make_batch(6, 2, n_protein=150, ligand_sizes=[20, 7])
    c3, c5 = _launches_per_step({}, b)
    per_step = (c5 - c3) // 2
    print('default form: %d launches per step' % per_step)
    assert per_step == DEFAULT_FORM_LAUNCHES_PER_STEP
    # the default form spelt out explicitly takes the same path
    e3, e5 = _launches_per_step({'num_x2h': 1, 'num_h2x': 1, 'sync_twoup': False}, b)
    assert (e3, e5) == (c3, c5)
    # a second x2h / h2x sub-layer adds launches (edge MLPs, node GEMMs, the ligand-slot edge lengths)
    x3, x5 = _launches_per_step({'num_h2x': 2}, b)
    assert (x5 - x3) // 2 > per_step
