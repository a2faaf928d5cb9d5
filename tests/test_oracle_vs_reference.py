"""Pins oracle/restate.py against the UNMODIFIED reference (run under oracle/shims): the restatement must reproduce, bit for bit,
what the reference returned on the same inputs, stored in tests/golden/reference_pins.pt by oracle/make_reference_pins.py."""
import os
import sys

import pytest
import torch

from oracle import make_reference_pins as pins_mod
from oracle import refload, restate, synth
from oracle.make_reference_pins import OPTION_CONFIGS, equal, option_id

if refload.SHIMS not in sys.path:           # torch_geometric / easydict stand-ins
    sys.path.insert(0, refload.SHIMS)


@pytest.fixture(scope='module', autouse=True)
def pins():
    n = torch.get_num_threads()
    torch.set_num_threads(pins_mod.THREADS)       # the thread count the pins were computed with
    yield torch.load(pins_mod.OUT, weights_only=True)
    torch.set_num_threads(n)


def test_state_dict_layout_matches_reference(pins):
    spec = synth.state_dict_spec()
    assert equal([(k, tuple(shape)) for k, shape, _ in spec], pins['state_dict_layout'])
    assert len(spec) == pins['state_dict_size'] == 384


def test_schedules_bit_exact(pins):
    sched = restate.make_schedules()
    for k in synth.SCHEDULE_KEYS:
        assert equal(sched[k], pins['schedules'][k]), k


def _assert_chain(got, want, keys=('pos_traj', 'v_traj', 'v0_traj', 'vt_traj')):
    assert equal(got['pos'], want['pos']) and equal(got['v'], want['v'])
    for k in keys:
        assert equal(list(got[k]), want[k]), k


def test_knn_shim_equals_canonical_restatement():
    from torch_geometric.nn import knn_graph  # the shim
    b = synth.make_batch(11, 3, n_protein=70, ligand_sizes=[5, 9, 1])
    x = torch.cat([b['protein_pos'], b['init_ligand_pos']])
    batch = torch.cat([b['batch_protein'], b['batch_ligand']])
    order = torch.sort(batch, stable=True).indices
    x, batch = x[order], batch[order]
    for k in (8, 32, 48):
        assert torch.equal(knn_graph(x, k=k, batch=batch, flow='source_to_target'), restate.knn_graph_canonical(x, k, batch))


def test_knn_small_graph_and_ties():
    from torch_geometric.nn import knn_graph
    # graph 0 has 5 nodes (< k+1) incl. exact duplicate points and equidistant neighbours; graph 1 has 40 on a lattice
    g0 = torch.tensor([[0., 0, 0], [1, 0, 0], [-1, 0, 0], [0, 0, 0], [0, 1, 0]])
    g1 = torch.stack(torch.meshgrid(torch.arange(5.), torch.arange(4.), torch.arange(2.), indexing='ij'), -1).reshape(-1, 3)
    x = torch.cat([g0, g1])
    batch = torch.cat([torch.zeros(5, dtype=torch.long), torch.ones(40, dtype=torch.long)])
    a = knn_graph(x, k=32, batch=batch)
    b = restate.knn_graph_canonical(x, 32, batch)
    assert torch.equal(a, b)
    assert (a[1] < 5).sum() == 5 * 4              # fewer than k edges per node in the small graph
    assert ((a[1] >= 5).sum()) == 40 * 32


def test_forward_bit_exact(pins):
    want = pins['forward']
    sd = synth.make_state_dict(0, schedules=restate.make_schedules())
    b = synth.make_batch(1, 2, n_protein=60, ligand_sizes=[9, 7])
    pp2, lp2, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    assert equal(pp2, want['protein_pos']) and equal(lp2, want['ligand_pos'])
    got = restate.forward(sd, None, pp2, b['protein_v'], b['batch_protein'], lp2, b['init_ligand_v'], b['batch_ligand'])
    for k in ('pred_ligand_pos', 'pred_ligand_v', 'final_h', 'final_ligand_h'):
        assert equal(got[k], want[k]), k


def test_sampling_chain_bit_exact(pins):
    sd = synth.make_state_dict(3, schedules=restate.make_schedules())
    b = synth.make_batch(2, 2, n_protein=48, ligand_sizes=[8, 6])
    S = 3
    pn, vu = synth.make_tape(7, S, len(b['batch_ligand']))
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    got = restate.sample_diffusion(sd, None, *args, pn, vu, num_steps=S)
    _assert_chain(got, pins['chain'])


@pytest.mark.parametrize('steps', [[0, 999], [417, 3], None])
def test_likelihood_estimation_matches_reference(pins, steps):
    """SURVEY 8(f) n3: the second consumer of `forward` (reference models/molopt_score_model.py:565-617), incl. the decoder
    branch (t = 0) and the prior branch (time_step == T)."""
    sd = synth.make_state_dict(5, schedules=restate.make_schedules())
    b = synth.make_batch(4, 2, n_protein=52, ligand_sizes=[7, 10])
    Nl = len(b['batch_ligand'])
    pn, vu = synth.make_tape(9, 1, Nl)
    t = torch.tensor(steps) if steps is not None else torch.full((2,), 1000)
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    want = pins['likelihood'][str(steps)]
    got = restate.likelihood_estimation(sd, None, *args, t, pn[0], vu[0])
    for w, g in zip(want, got):
        assert w.shape == g.shape == (2,)
        torch.testing.assert_close(g, w, rtol=1e-6, atol=1e-7)


def test_sampling_chain_noise_mean_type_bit_exact(pins):
    """SURVEY 8(f) n2: model_mean_type='noise' (reference models/molopt_score_model.py:663-666, :419-422)."""
    sd = synth.make_state_dict(6, schedules=restate.make_schedules())
    b = synth.make_batch(8, 2, n_protein=48, ligand_sizes=[8, 6])
    S = 3
    pn, vu = synth.make_tape(7, S, len(b['batch_ligand']))
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    got = restate.sample_diffusion(sd, {'model_mean_type': 'noise'}, *args, pn, vu, num_steps=S)
    _assert_chain(got, pins['chain_noise'])


@pytest.mark.parametrize('cfgd', OPTION_CONFIGS, ids=option_id)
def test_backbone_options_restatement_bit_exact(pins, cfgd):
    """SURVEY 8(f) n2: num_blocks > 1, ew_net_type r / m / none, x2h_out_fc, time_emb_mode 'simple', cutoff_mode 'hybrid' -- state_dict layout (key order and
    shapes) and a 3-step sampling chain of the restatement against the unmodified reference, bit for bit."""
    want = pins['options'][option_id(cfgd)]
    sd = synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd))
    assert equal(list(sd.keys()), want['keys'])
    b = synth.make_batch(3, 2, n_protein=60, ligand_sizes=[9, 7])
    S = 3
    pn, vu = synth.make_tape(5, S, 16)
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    w = restate.sample_diffusion(sd, cfgd, *args, pn, vu, num_steps=S)
    _assert_chain(w, want, keys=('v0_traj', 'vt_traj', 'pos_traj'))


def test_sampling_driver_restatement_bit_exact(pins):
    """a1: oracle.restate.sample_diffusion_ligand against the UNMODIFIED reference driver (scripts/sample_diffusion.py:31-116, imported with
    placeholders for rdkit / openbabel / lmdb) on the 1h36 pocket: same seeds -> the same prior sizes, positions, types and trajectories."""
    import json
    import random
    import numpy as np
    from targetdiff_b200.pocket import pdb_to_pocket_data
    want = pins['driver']
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    # the product's PDB ingest gives the reference's tensors
    data = pdb_to_pocket_data(os.path.join(root, 'tests', 'golden', '1h36_pocket10.pdb'))
    assert equal(data.protein_pos, want['protein_pos']) and equal(data.protein_atom_feature, want['protein_atom_feature'])
    sd = synth.make_state_dict(0, schedules=restate.make_schedules())
    prior = json.load(open(os.path.join(root, 'targetdiff_b200', 'data', 'atom_num_prior.json')))
    # the reference driver's global seeding (utils/misc.py seed_all)
    torch.manual_seed(2021)
    np.random.seed(2021)
    random.seed(2021)
    out2 = restate.sample_diffusion_ligand(sd, None, data.protein_pos, data.protein_atom_feature, 3, prior, batch_size=2, num_steps=2)
    for a, b in zip(want['outputs'], out2[:6]):
        assert len(a) == len(b) == 3 and all(equal(torch.from_numpy(np.asarray(y)), x) for x, y in zip(a, b))


def test_check_stability_restatement_equals_reference(pins):
    """n4: the bond-count stability screen (utils/evaluation/analyze.py:106-143) on random molecule-like point sets."""
    import numpy as np
    assert len(pins['stability']) == 2 * len(pins_mod.STABILITY_SIZES)
    for case in pins['stability']:
        got = restate.check_stability(case['pos'].numpy(), case['z'].numpy(), hs=case['hs'])
        assert [bool(got[0]), int(got[1]), int(got[2])] == case['result']
        assert np.array_equal(case['nr_bonds'].numpy(), np.asarray(got[3]))
