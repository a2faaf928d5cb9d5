"""GPU path against vectors the UNMODIFIED reference produced in the build container (oracle/make_golden.py, long cases):
the full 1000-step chain of BASELINE configs[0], the 1h36 pocket through the sampling driver on identical CPU RNG streams
(configs[1]), the k = 48 large pocket chain (configs[4]), plus the options the reference's sampler exposes (pos_only,
center_pos_mode='none') against the live CPU oracle.  Run with -m gpu.

Tolerances (BASELINE.json north_star): positions 1e-4 relative (atol 1e-4 A for near-zero coordinates), log-probabilities 1e-3,
sampled atom types identical.  A free-running chain contains discrete decisions (k-NN membership, Gumbel arg-max), so each long
test first reports where -- if anywhere -- the discrete trajectories part."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import restate, synth
from oracle.make_golden import GOLDEN, LONG_CASES

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
PDB_1H36 = os.path.join(GOLDEN, '1h36_pocket10.pdb')


def _model(weight_seed=0, cfg=None, gain=1.0):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg), gain=gain)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))


def _golden(name):
    path = os.path.join(GOLDEN, name + '.npz')
    if not os.path.exists(path):
        pytest.skip('golden %s.npz not generated' % name)
    return {k: torch.from_numpy(v) for k, v in np.load(path).items()}


def chain_divergence(pos_traj, v_traj, want_pos, want_v):
    """First step at which the sampled types differ, and the worst position error (relative to the coordinate scale) per 100 steps."""
    S = want_pos.shape[0]
    bad = (v_traj != want_v).flatten(1).any(1).nonzero()
    err = (pos_traj - want_pos).abs().flatten(1).max(1).values
    scale = want_pos.abs().flatten(1).max(1).values.clamp(min=1.0)
    rel = (err / scale)
    return {'steps': S, 'first_type_mismatch_step': int(bad[0]) if len(bad) else None,
            'type_mismatch_fraction': float((v_traj != want_v).float().mean()),
            'max_abs_pos_err': float(err.max()), 'max_rel_pos_err': float(rel.max()),
            'max_rel_pos_err_per_100_steps': [float(rel[i:i + 100].max()) for i in range(0, S, 100)]}


def run_chain_case(name, mode_env=None):
    case = LONG_CASES[name]
    g = _golden(name)
    model, sd = _model(case['weight_seed'], case['cfg'], gain=case.get('gain', 1.0))
    b = synth.make_batch(**case['batch'])
    T = sd['betas'].shape[0]
    S = case['num_steps'] or T
    pn, vu = synth.make_tape(case['tape_seed'], S, len(b['batch_ligand']))
    got = model.sample_diffusion(*_args(b), num_steps=case['num_steps'], center_pos_mode='protein', noise_tape=(pn, vu), stack_traj=True)
    rep = chain_divergence(got['pos_traj'], got['v_traj'], g['pos_traj'], g['v_traj'].long())
    return got, g, rep, case


def test_full_1000_step_chain_cfg1_vs_reference():
    """configs[0] shape, t = 999 ... 0 on one noise tape: the reference's own trajectory (unmodified code under the shims)."""
    got, g, rep, case = run_chain_case('chain_1000_cfg1')
    print('chain_1000_cfg1:', json.dumps(rep))
    assert rep['first_type_mismatch_step'] is None, rep
    torch.testing.assert_close(got['pos_traj'], g['pos_traj'], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(got['pos'].cpu(), g['pos'], rtol=1e-4, atol=1e-4)
    assert torch.equal(got['v'].cpu(), g['v'])
    st = case['stride']
    torch.testing.assert_close(got['v0_traj'][::st], g['v0_traj'], rtol=0, atol=1e-3)
    torch.testing.assert_close(got['vt_traj'][::st], g['vt_traj'], rtol=0, atol=1e-3)


def test_cfg5_large_pocket_k48_chain_vs_reference():
    """configs[4]: 1200 + 40 atoms, knn = 48, 20 denoising steps."""
    got, g, rep, case = run_chain_case('chain_cfg5')
    print('chain_cfg5:', json.dumps(rep))
    assert rep['first_type_mismatch_step'] is None, rep
    torch.testing.assert_close(got['pos_traj'], g['pos_traj'], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(got['v0_traj'], g['v0_traj'], rtol=0, atol=1e-3)
    torch.testing.assert_close(got['vt_traj'], g['vt_traj'], rtol=0, atol=1e-3)


def _run_driver(case):
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand, seed_all
    model, _ = _model(case['weight_seed'], case['cfg'])
    data = pdb_to_pocket_data(PDB_1H36)
    seed_all(case['seed'])
    return sample_diffusion_ligand(model, data, case['num_samples'], batch_size=case['batch_size'], device=DEV, num_steps=case['num_steps'],
                                   pos_only=False, center_pos_mode='protein', sample_num_atoms='prior', rng='cpu')


@pytest.mark.parametrize('name', ['pocket_1h36_s50', 'pocket_1h36_full'])
def test_1h36_pocket_driver_vs_reference_same_seeds(name):
    """configs[1]: examples/1h36 pocket -> pdb ingest -> sample_diffusion_ligand with prior-sampled sizes, seed 2021, every random number
    drawn from the CPU generators in the reference's order (rng='cpu'): sizes, atom types and positions must match what the
    unmodified reference driver produced on CPU."""
    case = LONG_CASES[name]
    g = _golden(name)
    pos, v, pos_traj, v_traj, v0_traj, vt_traj, _ = _run_driver(case)
    assert [len(p) for p in pos] == g['sizes'].tolist()                       # the prior drew the same ligand sizes
    got_pos_traj = torch.from_numpy(np.concatenate(pos_traj, axis=1)).float()
    got_v_traj = torch.from_numpy(np.concatenate(v_traj, axis=1))
    rep = chain_divergence(got_pos_traj, got_v_traj, g['pos_traj'], g['v_traj'].long())
    print(name + ':', json.dumps(rep))
    assert rep['first_type_mismatch_step'] is None, rep
    assert np.array_equal(np.concatenate(v), g['v'].numpy())
    torch.testing.assert_close(got_pos_traj, g['pos_traj'], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(torch.from_numpy(np.concatenate(pos)), g['pos'], rtol=1e-4, atol=1e-4)
    st = case['stride']
    torch.testing.assert_close(torch.from_numpy(np.concatenate(v0_traj, axis=1))[::st], g['v0_traj'], rtol=0, atol=1e-3)
    torch.testing.assert_close(torch.from_numpy(np.concatenate(vt_traj, axis=1))[::st], g['vt_traj'], rtol=0, atol=1e-3)


def test_1h36_forward_vs_oracle():
    """One network evaluation on the real pocket with three ragged ligands: edge_index bit-exact, outputs within tolerance."""
    from targetdiff_b200.pocket import pdb_to_pocket_data
    torch.set_num_threads(16)
    model, sd = _model(0)
    data = pdb_to_pocket_data(PDB_1H36)
    sizes = [25, 31, 18]
    n_prot = data.protein_pos.shape[0]
    g = torch.Generator().manual_seed(5)
    ppos = data.protein_pos.repeat(3, 1)
    pfeat = data.protein_atom_feature.float().repeat(3, 1)
    bp = torch.repeat_interleave(torch.arange(3), n_prot)
    bl = torch.repeat_interleave(torch.arange(3), torch.tensor(sizes))
    lpos = data.protein_pos.mean(0, keepdim=True) + torch.randn(sum(sizes), 3, generator=g)
    lv = torch.randint(0, 13, (sum(sizes),), generator=g)
    pp, lp, _ = restate.center_pos(ppos, lpos, bp, bl)
    tr = {}
    want = restate.forward(sd, None, pp, pfeat, bp, lp, lv, bl, trace=tr)
    out = model(pp.to(DEV), pfeat.to(DEV), bp.to(DEV), lp.to(DEV), lv.to(DEV), bl.to(DEV), return_edge_weight=True)
    assert torch.equal(out['edge_index'].cpu(), tr['edge_index'])
    torch.testing.assert_close(out['edge_weight'].cpu(), tr['e_w'], rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=1e-3)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=1e-4, atol=1e-4)


def test_edge_weight_vs_reference_golden():
    """The global edge gate e_w of the forward golden case (written by the reference itself), read back through tdiff_get_edge_weight."""
    from oracle.make_golden import CASES
    case = CASES['forward_small']
    g = _golden('forward_small')
    model, _ = _model(case['weight_seed'], case['cfg'])
    b = synth.make_batch(**case['batch'])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    out = model(pp.to(DEV), b['protein_v'].to(DEV), b['batch_protein'].to(DEV), lp.to(DEV), b['init_ligand_v'].to(DEV), b['batch_ligand'].to(DEV),
                return_edge_weight=True)
    assert torch.equal(out['edge_index'].cpu(), g['edge_index'])
    torch.testing.assert_close(out['edge_weight'].cpu(), g['e_w'], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize('pos_only,center', [(True, 'protein'), (False, 'none'), (True, 'none')])
def test_sampler_options_vs_oracle(pos_only, center):
    """pos_only=True keeps the atom types and records no v0 / vt trajectories (reference models/molopt_score_model.py:681-693);
    center_pos_mode='none' samples in the lab frame (:110-120)."""
    torch.set_num_threads(16)
    model, sd = _model(1)
    b = synth.make_batch(8, 2, n_protein=80, ligand_sizes=[11, 6])
    if center == 'none':                   # keep the lab-frame coordinates small: the network is not translation invariant without centring
        shift = b['protein_pos'].mean(0, keepdim=True)
        b['protein_pos'] = b['protein_pos'] - shift
        b['init_ligand_pos'] = b['init_ligand_pos'] - shift
    S = 6
    pn, vu = synth.make_tape(13, S, len(b['batch_ligand']))
    want = restate.sample_diffusion(sd, None, *_args(b, 'cpu'), pn, vu, num_steps=S, center_pos_mode=center, pos_only=pos_only)
    got = model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode=center, pos_only=pos_only, noise_tape=(pn, vu))
    assert torch.equal(torch.stack(got['v_traj']), torch.stack(want['v_traj']))
    torch.testing.assert_close(torch.stack(got['pos_traj']), torch.stack(want['pos_traj']), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(got['pos'].cpu(), want['pos'], rtol=1e-4, atol=1e-5)
    if pos_only:
        assert got['v0_traj'] == [] and got['vt_traj'] == [] and torch.equal(got['v'].cpu(), b['init_ligand_v'])
    else:
        torch.testing.assert_close(torch.stack(got['v0_traj']), torch.stack(want['v0_traj']), rtol=0, atol=1e-3)


def test_sample_host_odd_sizes_all_trajectories():
    """tdiff_sample_host with S * Nl odd and every trajectory buffer requested: the int64 trajectory must land on an aligned staging
    offset (round-1 advisor finding) and equal the device-buffer path."""
    import ctypes
    from targetdiff_b200 import _lib
    lib = _lib.load()
    model, _ = _model(0)
    b = synth.make_batch(3, 1, n_protein=40, ligand_sizes=[7])
    S, n_l, K = 3, 7, 13
    r = model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', seed=5, stack_traj=True)
    eng = model.engine(DEV)
    hp = {k: v.contiguous() for k, v in b.items()}
    out_pos, out_v = torch.empty(n_l, 3), torch.empty(n_l, dtype=torch.int64)
    pos_traj, v_traj = torch.empty(S, n_l, 3), torch.empty(S, n_l, dtype=torch.int64)
    v0_traj, vt_traj = torch.empty(S, n_l, K), torch.empty(S, n_l, K)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    _lib.check(lib.tdiff_sample_host(eng, 1, _lib.i32_array([40]), _lib.i32_array([7]), P(hp['protein_pos']), P(hp['protein_v']),
                                     P(hp['init_ligand_pos']), P(hp['init_ligand_v']), 1, S, None, None, ctypes.c_uint64(5), P(out_pos), P(out_v),
                                     P(pos_traj), P(v_traj), P(v0_traj), P(vt_traj), 0, st))
    assert torch.equal(pos_traj, r['pos_traj']) and torch.equal(v_traj, r['v_traj'])
    assert torch.equal(v0_traj, r['v0_traj']) and torch.equal(vt_traj, r['vt_traj'])
    assert torch.equal(out_pos, r['pos'].cpu()) and torch.equal(out_v, r['v'].cpu())


OPTION_CONFIGS = [{'num_blocks': 2}, {'ew_net_type': 'r'}, {'ew_net_type': 'm'}, {'ew_net_type': 'none'}, {'x2h_out_fc': True},
                  {'time_emb_dim': 1, 'time_emb_mode': 'simple'}, {'num_blocks': 2, 'ew_net_type': 'r', 'x2h_out_fc': True, 'time_emb_dim': 1}]


@pytest.mark.parametrize('cfgd', OPTION_CONFIGS, ids=lambda c: ','.join('%s=%s' % kv for kv in c.items()))
def test_backbone_options_vs_oracle(cfgd):
    """SURVEY 8(f) n2 on the engine: re-built k-NN graph per block (reference models/uni_transformer.py:306-307), per-sub-layer 'r' /
    value-driven 'm' / absent edge gates (:58-66,121-129), node_output MLP (:39-40,80-81), time embedding 'simple'
    (models/molopt_score_model.py:319-324): forward and a 6-step chain against the oracle (itself bit-exact against the reference,
    tests/test_oracle_vs_reference.py::test_backbone_options_restatement_bit_exact)."""
    torch.set_num_threads(16)
    model, sd = _model(2, cfgd)
    b = synth.make_batch(9, 3, n_protein=70, ligand_sizes=[12, 5, 9])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    t = torch.tensor([999, 500, 3])
    tr = {}
    want = restate.forward(sd, cfgd, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr, time_step=t)
    out = model(pp.to(DEV), b['protein_v'].to(DEV), b['batch_protein'].to(DEV), lp.to(DEV), b['init_ligand_v'].to(DEV), b['batch_ligand'].to(DEV),
                time_step=t.to(DEV))
    assert torch.equal(out['edge_index'].cpu(), tr['block_edge_index'][-1])          # graph of the last block
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=1e-3)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=1e-4, atol=1e-4)
    S = 6
    pn, vu = synth.make_tape(4, S, len(b['batch_ligand']))
    w = restate.sample_diffusion(sd, cfgd, *_args(b, 'cpu'), pn, vu, num_steps=S)
    got = model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', noise_tape=(pn, vu))
    assert torch.equal(torch.stack(got['v_traj']), torch.stack(w['v_traj']))
    torch.testing.assert_close(torch.stack(got['pos_traj']), torch.stack(w['pos_traj']), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(torch.stack(got['v0_traj']), torch.stack(w['v0_traj']), rtol=0, atol=1e-3)


def _sorted_edges(ei):
    """edge_index as a canonical [E,2] (dst, src) list: the hybrid graph of the reference is emitted per graph as [ligand-ligand |
    ligand<-protein | protein k-NN] (models/common.py:205-206), the engine's slot list is destination-sorted; the edge SET is what
    must agree bit for bit."""
    key = ei[1] * (int(ei.max()) + 1 if ei.numel() else 1) + ei[0]
    return ei[:, torch.argsort(key)]


HYBRID_CONFIGS = [{'cutoff_mode': 'hybrid'}, {'cutoff_mode': 'hybrid', 'knn': 8, 'num_blocks': 2},
                  {'cutoff_mode': 'hybrid', 'knn': 21, 'ew_net_type': 'r'}]


@pytest.mark.parametrize('cfgd', HYBRID_CONFIGS, ids=lambda c: ','.join('%s=%s' % kv for kv in c.items()))
def test_hybrid_cutoff_vs_oracle(cfgd):
    """SURVEY 8(f) n2, cutoff_mode='hybrid' (reference models/uni_transformer.py:281-283 -> models/common.py:165-212): every ligand atom
    is connected to all other ligand atoms of its graph and to its k nearest protein atoms, protein destinations keep the k-NN over all
    atoms.  Forward and a 6-step chain against the oracle (bit-exact against the unmodified reference for the same configurations,
    tests/test_oracle_vs_reference.py::test_backbone_options_restatement_bit_exact); slot rows = k + 12 - 1 (43 / 19 / 32: the last one
    also takes the fused-aggregation path of the edge kernel)."""
    torch.set_num_threads(16)
    model, sd = _model(2, cfgd)
    b = synth.make_batch(9, 3, n_protein=70, ligand_sizes=[12, 5, 9])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    want = restate.forward(sd, cfgd, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    out = model(pp.to(DEV), b['protein_v'].to(DEV), b['batch_protein'].to(DEV), lp.to(DEV), b['init_ligand_v'].to(DEV), b['batch_ligand'].to(DEV))
    got_ei, want_ei = out['edge_index'].cpu(), tr['block_edge_index'][-1]
    assert got_ei.shape == want_ei.shape
    assert torch.equal(_sorted_edges(got_ei), _sorted_edges(want_ei))
    k = cfgd.get('knn', 32)
    nodes = 70 * 3 + 26
    is_lig = torch.zeros(nodes, dtype=torch.bool)
    start = 0
    for n_l in (12, 5, 9):
        is_lig[start + 70:start + 70 + n_l] = True
        start += 70 + n_l
    deg = torch.bincount(got_ei[1], minlength=nodes)
    assert torch.equal(deg[~is_lig], torch.full((210,), k))                      # protein destinations: k-NN over all atoms
    assert sorted(set(deg[is_lig].tolist())) == sorted({k + 11, k + 4, k + 8})   # ligand destinations: n_l - 1 + k
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=1e-3)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=1e-4, atol=1e-4)
    S = 6
    pn, vu = synth.make_tape(4, S, len(b['batch_ligand']))
    w = restate.sample_diffusion(sd, cfgd, *_args(b, 'cpu'), pn, vu, num_steps=S)
    got = model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', noise_tape=(pn, vu))
    assert torch.equal(torch.stack(got['v_traj']), torch.stack(w['v_traj']))
    torch.testing.assert_close(torch.stack(got['pos_traj']), torch.stack(w['pos_traj']), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(torch.stack(got['v0_traj']), torch.stack(w['v0_traj']), rtol=0, atol=1e-3)


def test_hybrid_cutoff_rejects_what_does_not_fit():
    """k + n_ligand - 1 neighbour slots must fit the 64-slot rows, and every graph needs >= k protein atoms (torch.topk raises in the
    reference, models/common.py:176): both are refused at bind time with a message, never truncated silently."""
    from targetdiff_b200._lib import TdiffError
    model, _ = _model(2, {'cutoff_mode': 'hybrid'})
    b = synth.make_batch(9, 1, n_protein=70, ligand_sizes=[34])                  # 32 + 34 - 1 = 65 slots
    with pytest.raises(TdiffError, match='hybrid'):
        model(*_args(b))
    b = synth.make_batch(9, 1, n_protein=20, ligand_sizes=[5])                   # fewer protein atoms than k
    with pytest.raises(TdiffError, match='hybrid'):
        model(*_args(b))
    b = synth.make_batch(9, 1, n_protein=70, ligand_sizes=[33])                  # exactly 64 slots: accepted
    out = model(*_args(b))
    assert out['edge_index'].shape[1] == 70 * 32 + 33 * 64
