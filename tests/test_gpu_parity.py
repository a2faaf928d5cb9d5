"""CUDA path (through the C-ABI of libtdiff.so) vs the CPU oracle -- run on an H100 with `-m gpu`.

Tolerances (BASELINE.json north_star): edge_index bit-exact; positions within 1e-4 relative; logits within 1e-3."""
import os

import numpy as np
import pytest
import torch

from oracle import restate, synth
from oracle.make_golden import CASES, GOLDEN

pytestmark = pytest.mark.gpu

POS_RTOL, POS_ATOL = 1e-4, 1e-5      # positions: 1e-4 relative (atol for coordinates that happen to be ~0)
LOGIT_ATOL = 1e-3                    # atom-type logits / log-probabilities
H_RTOL, H_ATOL = 1e-4, 1e-4


def _dev():
    return torch.device('cuda:0')


def _model(weight_seed, cfg=None):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg))
    m.load_state_dict(sd, strict=True)
    return m.to(_dev()), sd


def _to(b, dev):
    return {k: v.to(dev) for k, v in b.items()}


def _golden(name):
    return {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLDEN, name + '.npz')).items()}


# ------------------------------------------------------------------------------------------------ operators
@pytest.mark.parametrize('k', [8, 32, 48])
def test_knn_graph_bit_exact(k):
    from targetdiff_b200 import ops
    b = synth.make_batch(11, 5, n_protein=90, ligand_sizes=[5, 9, 1, 20, 0])
    x = torch.cat([b['protein_pos'], b['init_ligand_pos']])
    batch = torch.cat([b['batch_protein'], b['batch_ligand']])
    order = torch.sort(batch, stable=True).indices
    x, batch = x[order], batch[order]
    want = restate.knn_graph_canonical(x, k, batch)
    got = ops.knn_graph(x.to(_dev()), k, batch.to(_dev())).cpu()
    assert got.dtype == torch.int64 and torch.equal(got, want)


def test_knn_graph_small_graphs_ties_duplicates():
    from targetdiff_b200 import ops
    g0 = torch.tensor([[0., 0, 0], [1, 0, 0], [-1, 0, 0], [0, 0, 0], [0, 1, 0]])        # < k+1 nodes, duplicate point, ties
    g1 = torch.stack(torch.meshgrid(torch.arange(5.), torch.arange(4.), torch.arange(2.), indexing='ij'), -1).reshape(-1, 3)
    g2 = torch.tensor([[3., 3, 3]])                                                        # single-node graph: no edges
    x = torch.cat([g0, g1, g2])
    batch = torch.cat([torch.zeros(5), torch.ones(40), torch.full((1,), 2)]).long()
    want = restate.knn_graph_canonical(x, 32, batch)
    got = ops.knn_graph(x.to(_dev()), 32, batch.to(_dev())).cpu()
    assert torch.equal(got, want)
    slots, ne = ops.knn_slots(x.to(_dev()), 32, batch.to(_dev()))
    assert ne == want.shape[1] and (slots[:5, 4:] == -1).all() and (slots[45] == -1).all()


def test_knn_large_pocket_k48():
    from targetdiff_b200 import ops
    b = synth.make_batch(21, 1, n_protein=1200, ligand_sizes=[40])
    x = torch.cat([b['protein_pos'], b['init_ligand_pos']])
    batch = torch.zeros(len(x), dtype=torch.long)
    want = restate.knn_graph_canonical(x, 48, batch)
    got = ops.knn_graph(x.to(_dev()), 48, batch.to(_dev())).cpu()
    assert torch.equal(got, want)


def _slot_problem(n, kk, seed, ragged=True):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (n, kk), generator=g, dtype=torch.int32)
    if ragged:                                  # absent edges are tail-padded with -1
        deg = torch.randint(0, kk + 1, (n,), generator=g)
        deg[0] = 0
        src[torch.arange(kk)[None, :] >= deg[:, None]] = -1
    k = torch.randn(n * kk, 128, generator=g)
    q = torch.randn(n, 128, generator=g)
    e_w = torch.rand(n * kk, generator=g)
    return src, k, q, e_w, g


def test_attn_aggregate_h_vs_scatter_oracle():
    from targetdiff_b200 import ops
    n, kk = 77, 32
    src, k, q, e_w, g = _slot_problem(n, kk, 5)
    v = torch.randn(n * kk, 128, generator=g)
    h = torch.randn(n, 128, generator=g)
    valid = (src.view(-1) >= 0)
    dst = torch.arange(n).repeat_interleave(kk)[valid]
    ke, ve, ew = k[valid].view(-1, 16, 8), v[valid], e_w[valid]
    alpha = restate.scatter_softmax_rows((q.view(-1, 16, 8)[dst] * ke / np.sqrt(8)).sum(-1), dst, n)
    want = restate.scatter_sum_rows(alpha.unsqueeze(-1) * (ve * ew[:, None]).view(-1, 16, 8), dst, n).view(n, 128) + h
    d = _dev()
    got = ops.attn_aggregate_h(k.to(d), v.to(d), e_w.to(d), src.to(d), q.to(d), h.to(d)).cpu()
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)


def test_attn_aggregate_x_vs_scatter_oracle():
    from targetdiff_b200 import ops
    n, kk = 53, 32
    src, k, q, e_w, g = _slot_problem(n, kk, 6)
    src[src == torch.arange(n, dtype=torch.int32)[:, None]] = 0
    v16 = torch.randn(n * kk, 16, generator=g)
    x = torch.randn(n, 3, generator=g) * 4
    mask = torch.rand(n, generator=g) < 0.4
    valid = (src.view(-1) >= 0)
    dst = torch.arange(n).repeat_interleave(kk)[valid]
    s = src.view(-1)[valid].long()
    ke = k[valid].view(-1, 16, 8)
    rel = x[dst] - x[s]
    alpha = restate.scatter_softmax_rows((q.view(-1, 16, 8)[dst] * ke / np.sqrt(8)).sum(-1), dst, n)
    m = alpha.unsqueeze(-1) * ((v16[valid] * e_w[valid][:, None]).unsqueeze(-1) * rel.unsqueeze(1))
    want = x + restate.scatter_sum_rows(m, dst, n).mean(1) * mask[:, None]
    d = _dev()
    got = ops.attn_aggregate_x(k.to(d), v16.to(d), e_w.to(d), src.to(d), q.to(d), x.to(d), mask.to(d)).cpu()
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)


def test_scatter_mean3_bit_exact():
    from targetdiff_b200 import ops
    b = synth.make_batch(3, 4, n_protein=123, ligand_sizes=[1, 1, 1, 1])
    _, _, want = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    got = ops.scatter_mean3(b['protein_pos'].to(_dev()), b['batch_protein'].to(_dev())).cpu()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ forward
def _check_forward(out, ref_out, trace):
    assert torch.equal(out['edge_index'].cpu(), trace['edge_index'])                        # bit-exact
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), ref_out['pred_ligand_pos'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), ref_out['pred_ligand_v'], rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(out['final_h'].cpu(), ref_out['final_h'], rtol=H_RTOL, atol=H_ATOL)
    torch.testing.assert_close(out['final_ligand_h'].cpu(), ref_out['final_ligand_h'], rtol=H_RTOL, atol=H_ATOL)


def test_forward_vs_oracle_and_golden():
    case = CASES['forward_small']
    model, sd = _model(case['weight_seed'])
    b = synth.make_batch(**case['batch'])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    want = restate.forward(sd, None, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    d = _dev()
    out = model(pp.to(d), b['protein_v'].to(d), b['batch_protein'].to(d), lp.to(d), b['init_ligand_v'].to(d), b['batch_ligand'].to(d))
    _check_forward(out, want, tr)
    g = _golden('forward_small')                      # produced by the reference itself
    assert torch.equal(out['edge_index'].cpu(), g['edge_index'])
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), g['pred_ligand_pos'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), g['pred_ligand_v'], rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(out['final_h'].cpu(), g['final_h'], rtol=H_RTOL, atol=H_ATOL)


@pytest.mark.parametrize('shape', [dict(n_graphs=1, n_protein=300, ligand_sizes=[20]),            # BASELINE config 1 shape
                                   dict(n_graphs=3, n_protein=200, ligand_sizes=[33, 1, 12]),
                                   dict(n_graphs=2, n_protein=20, ligand_sizes=[6, 40])])          # graphs with <= k nodes
def test_forward_shapes(shape):
    model, sd = _model(1)
    b = synth.make_batch(31, **shape)
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    want = restate.forward(sd, None, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    d = _dev()
    out = model(pp.to(d), b['protein_v'].to(d), b['batch_protein'].to(d), lp.to(d), b['init_ligand_v'].to(d), b['batch_ligand'].to(d))
    _check_forward(out, want, tr)


def test_forward_fix_x_and_k48():
    model, sd = _model(2, {'knn': 48})
    b = synth.make_batch(41, 1, n_protein=150, ligand_sizes=[25])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    d = _dev()
    args_d = (pp.to(d), b['protein_v'].to(d), b['batch_protein'].to(d), lp.to(d), b['init_ligand_v'].to(d), b['batch_ligand'].to(d))
    for fix_x in (False, True):
        tr = {}
        want = restate.forward(sd, {'knn': 48}, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'],
                               fix_x=fix_x, trace=tr)
        out = model(*args_d, fix_x=fix_x)
        _check_forward(out, want, tr)
        if fix_x:
            torch.testing.assert_close(out['pred_ligand_pos'].cpu(), lp, rtol=0, atol=0)


# ------------------------------------------------------------------------------------------------ sampling chains
@pytest.mark.parametrize('name', ['chain_trunc', 'chain_full_T20'])
def test_chain_vs_golden_and_oracle(name):
    """Free-running chain on one noise tape: CUDA path vs the reference's own output (golden) and the oracle."""
    case, g = CASES[name], _golden(name)
    model, sd = _model(case['weight_seed'], case['cfg'])
    b = synth.make_batch(**case['batch'])
    S = case['num_steps'] or sd['betas'].shape[0]
    pn, vu = synth.make_tape(case['tape_seed'], S, len(b['batch_ligand']))
    d = _dev()
    bd = _to(b, d)
    r = model.sample_diffusion(bd['protein_pos'], bd['protein_v'], bd['batch_protein'], bd['init_ligand_pos'], bd['init_ligand_v'],
                               bd['batch_ligand'], num_steps=case['num_steps'], center_pos_mode='protein', noise_tape=(pn, vu))
    assert torch.equal(r['v'].cpu(), g['v'])
    assert torch.equal(torch.stack(r['v_traj']), g['v_traj'])
    torch.testing.assert_close(r['pos'].cpu(), g['pos'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(torch.stack(r['pos_traj']), g['pos_traj'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(torch.stack(r['v0_traj']), g['v0_traj'], rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(torch.stack(r['vt_traj']), g['vt_traj'], rtol=0, atol=LOGIT_ATOL)


def test_chain_graph_replay_equals_eager(monkeypatch):
    """CUDA-graph replay and eager launches give identical results (same kernels, same order)."""
    model, sd = _model(5)
    b = _to(synth.make_batch(6, 2, n_protein=64, ligand_sizes=[7, 11]), _dev())
    S = 6
    pn, vu = synth.make_tape(3, S, len(b['batch_ligand']))
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    r1 = model.sample_diffusion(*args, num_steps=S, center_pos_mode='protein', noise_tape=(pn, vu))
    monkeypatch.setenv('TDIFF_NO_GRAPH', '1')
    r2 = model.sample_diffusion(*args, num_steps=S, center_pos_mode='protein', noise_tape=(pn, vu))
    assert torch.equal(r1['pos'], r2['pos']) and torch.equal(r1['v'], r2['v'])
    assert torch.equal(torch.stack(r1['vt_traj']), torch.stack(r2['vt_traj']))


def test_chain_philox_reproducible_and_sane():
    model, sd = _model(5)
    b = _to(synth.make_batch(8, 4, n_protein=100, ligand_sizes=[10, 20, 5, 15]), _dev())
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    r1 = model.sample_diffusion(*args, num_steps=12, center_pos_mode='protein', seed=123)
    r2 = model.sample_diffusion(*args, num_steps=12, center_pos_mode='protein', seed=123)
    r3 = model.sample_diffusion(*args, num_steps=12, center_pos_mode='protein', seed=124)
    assert torch.equal(r1['pos'], r2['pos']) and torch.equal(r1['v'], r2['v'])
    assert not torch.equal(r1['pos'], r3['pos'])
    assert torch.isfinite(r1['pos']).all() and int(r1['v'].min()) >= 0 and int(r1['v'].max()) < 13
    assert len(r1['pos_traj']) == 12 and r1['pos_traj'][0].shape == (50, 3)
    # device noise has the right moments: the one-step position noise is N(0, sigma_t^2)
    lp = torch.stack(r1['vt_traj'])
    torch.testing.assert_close(lp.exp().sum(-1), torch.ones(12, 50), rtol=0, atol=1e-4)


def test_errors_are_loud():
    from targetdiff_b200._lib import TdiffError
    model, sd = _model(0)
    b = _to(synth.make_batch(1, 1, n_protein=40, ligand_sizes=[5]), _dev())
    bad_v = torch.full_like(b['init_ligand_v'], 13)
    with pytest.raises(TdiffError):
        model(b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], bad_v, b['batch_ligand'])
    with pytest.raises(ValueError):
        model(b['protein_pos'], b['protein_v'], b['batch_protein'].flip(0) * 0 + torch.arange(40, device=_dev()).flip(0) // 20,
              b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])


def test_check_stability_vs_oracle():
    """SURVEY 8(f) n4: tdiff_check_stability against the CPU restatement of utils/evaluation/analyze.py:106-143 -- integer outputs,
    bit-exact; ragged molecule sizes incl. a single atom, both `hs` settings, and the per-atom bond counts."""
    import numpy as np
    from targetdiff_b200 import analyze
    rng = np.random.RandomState(1)
    sizes = [1, 2, 9, 25, 40, 33, 86, 17]
    pos, zs = [], []
    for n in sizes:
        pos.append(np.cumsum(rng.normal(scale=0.85, size=(n, 3)), axis=0).astype(np.float32).astype(np.float64) + rng.uniform(-30, 30, size=(1, 3)))
        zs.append(rng.choice([1, 6, 7, 8, 9, 15, 16, 17], size=n, p=[0.1, 0.5, 0.12, 0.15, 0.03, 0.02, 0.05, 0.03]))
    pos = [p.astype(np.float32).astype(np.float64) for p in pos]           # the sampler's positions are fp32 values widened to fp64
    for hs in (False, True):
        ms, ns, na, nb = analyze.check_stability_batch(pos, zs, hs=hs)
        off = 0
        for i, n in enumerate(sizes):
            w = restate.check_stability(pos[i], zs[i], hs=hs)
            assert (bool(ms[i]), int(ns[i]), int(na[i])) == (bool(w[0]), w[1], w[2])
            assert np.array_equal(nb[off:off + n], w[3])
            off += n
    one = analyze.check_stability(pos[3], zs[3], return_nr_bonds=True)
    w = restate.check_stability(pos[3], zs[3])
    assert one[:3] == (bool(w[0]), w[1], w[2]) and np.array_equal(one[3], w[3])
    with pytest.raises(Exception):
        analyze.check_stability(pos[1], np.array([6, 5]))                  # boron is not in the reference's table (KeyError there)
