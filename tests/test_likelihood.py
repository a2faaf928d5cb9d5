"""Likelihood scoring on the CPU (DESIGN.md section 1): the restated driver against the unmodified reference's pins, the oracle's terms
against restate.likelihood_estimation, the own-type prior, the host Philox restatement of the likelihood stream, and the refusals that
need no device."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import likelihood, restate, synth
from targetdiff_b200.likelihood import likelihood_time_steps

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
PINS = os.path.join(GOLDEN, 'reference_pins_likelihood_driver.pt')


def _pins():
    return torch.load(PINS, weights_only=False)


def _sd(case):
    return synth.make_state_dict(case['weight_seed'], case['cfg'], schedules=restate.make_schedules(case['cfg']), ligand_dim=case['K'])


# ------------------------------------------------------------------------------------------------ 1. the driver against the reference
@pytest.mark.parametrize('name', ['default_bs4', 'default_bs1', 'time_emb', 'K23', '1h36'])
def test_restated_driver_equals_reference_pins(name):
    torch.set_num_threads(1)
    case = _pins()[name]
    synth_seed = case['seed']
    from targetdiff_b200.sampling import seed_all
    seed_all(synth_seed)
    kp, kv, sp, sv = likelihood.data_likelihood_estimation(_sd(case), case['cfg'], case['data'], case['time_steps'], case['batch_size'])
    assert torch.equal(kp, case['kl_pos']) and torch.equal(kv, case['kl_v'])
    assert sp == case['sum_kl_pos'] and sv == case['sum_kl_v']
    assert kp.shape == (len(case['time_steps']) + 1,)


# ------------------------------------------------------------------------------------------------ 2. the oracle's terms
@pytest.mark.parametrize('cfgd,K', [({}, 13), ({'time_emb_dim': 1, 'time_emb_mode': 'simple'}, 13), ({}, 8), ({}, 23)])
def test_oracle_terms_equal_restated_likelihood_estimation(cfgd, K):
    sd = synth.make_state_dict(3, cfgd, schedules=restate.make_schedules(cfgd), ligand_dim=K)
    b = synth.make_batch(11, 4, n_protein=48, ligand_sizes=[7, 10, 5, 9], num_classes=K)
    ts = torch.tensor([0, 1, 417, 999])
    pn, vu = likelihood.likelihood_tape(5, ts, None, b['batch_ligand'], K)
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    got = likelihood.terms(sd, cfgd, *args, ts, pn, vu)
    want = restate.likelihood_estimation(sd, cfgd, *args, ts, pos_noise=pn, v_uniform=vu)
    assert torch.equal(got['kl_pos'], want[0]) and torch.equal(got['kl_v'], want[1])


# ------------------------------------------------------------------------------------------------ 3. the own-type prior
@pytest.mark.parametrize('K', [8, 13, 23])
def test_type_prior_is_class_symmetric(K):
    sd = restate.make_schedules()
    x0 = torch.zeros(K, 3)
    # the KL is a small difference of K terms of size about 1/K: rounding is bounded by the sum of their magnitudes S
    T = sd['alphas_cumprod'].shape[0]
    lq = restate.q_v_pred({k: v.double() for k, v in sd.items()}, torch.log(torch.eye(K, dtype=torch.float64)[:1].clamp(min=1e-30)),
                          torch.tensor([T - 1]), torch.tensor([0]), K)
    S = float((lq.exp() * (lq + np.log(K))).abs().sum())
    own = likelihood.prior_atom_terms(sd, x0, torch.arange(K), K, dtype=torch.float64)[1]
    assert float((own - own[0]).abs().max()) <= 4 * K * 2.0 ** -52 * S
    own32 = likelihood.prior_atom_terms(sd, x0, torch.arange(K), K)[1]
    graph_id = likelihood.prior_atom_terms(sd, x0, torch.zeros(K, dtype=torch.long), K)[1]      # the script's one-graph prior: class 0
    # fp32: the same K products, each rounded in its own way, summed in another order
    bound = 4 * K * 2.0 ** -23 * S
    assert float((own32 - graph_id).abs().max()) <= bound
    # the graph-id prior of the restated reference equals the own-type prior of class 0
    b = {'batch_ligand': torch.zeros(5, dtype=torch.long)}
    pos = torch.randn(5, 3)
    ref_prior = restate.likelihood_estimation({**sd, 'v_inference.2.weight': torch.zeros(K, 1)}, None, torch.zeros(3, 3),
                                              torch.zeros(3, 27), torch.zeros(3, dtype=torch.long), pos, torch.zeros(5, dtype=torch.long),
                                              b['batch_ligand'], torch.tensor([1000]))
    pp, pv = likelihood.prior_atom_terms(sd, pos - 0.0, torch.zeros(5, dtype=torch.long), K)
    assert torch.equal(ref_prior[0], pp.mean().reshape(1)) or torch.allclose(ref_prior[0], pp.mean().reshape(1), rtol=1e-6)
    assert torch.allclose(ref_prior[1], pv.mean().reshape(1), rtol=1e-6)


# ------------------------------------------------------------------------------------------------ 4. the host Philox restatement
def test_stream_does_not_depend_on_batch_layout():
    K = 13
    alone = likelihood.likelihood_tape(9, [417], [3], [0] * 6, K)
    # the same ligand (key 3, t 417) as graph 2 of a batch, among other graphs
    batch = [0] * 4 + [1] * 9 + [2] * 6 + [3] * 2
    pn, vu = likelihood.likelihood_tape(9, [5, 417, 417, 0], [0, 1, 3, 3], batch, K)
    assert torch.equal(pn[13:19], alone[0]) and torch.equal(vu[13:19], alone[1])
    # another key, another t or another seed changes the draw
    assert not torch.equal(pn[4:10], pn[13:19])
    assert not torch.equal(likelihood.likelihood_tape(9, [416], [3], [0] * 6, K)[0], alone[0])
    assert not torch.equal(likelihood.likelihood_tape(10, [417], [3], [0] * 6, K)[0], alone[0])


def test_domains_are_distinct():
    words = list(likelihood.DOMAINS.values())
    assert len(set(words)) == len(words) == 8
    assert likelihood.DOMAINS['likelihood_pos'] == int.from_bytes(b'lkps', 'big')
    assert likelihood.DOMAINS['likelihood_type'] == int.from_bytes(b'lktv', 'big')


def test_stream_moments():
    n = 20000
    batch = np.repeat(np.arange(40), n // 40)
    t = np.arange(40) * 24
    pn = likelihood.likelihood_normals(123, t, np.arange(40) + 7, batch).reshape(-1)
    vu = likelihood.likelihood_uniforms(123, t, np.arange(40) + 7, batch, 23).reshape(-1)
    assert stats.kstest(pn, 'norm').pvalue > 1e-3
    assert stats.kstest(vu, 'uniform').pvalue > 1e-3
    assert abs(pn.mean()) < 5 / np.sqrt(len(pn)) and abs(pn.var() - 1) < 0.02
    assert vu.min() >= 0 and vu.max() < 1


def test_stream_refuses_times_beyond_24_bits():
    with pytest.raises(ValueError, match='2\\^24'):
        likelihood.likelihood_tape(1, [1 << 24], None, [0], 13)


# ------------------------------------------------------------------------------------------------ 5. refusals and time steps
def test_likelihood_time_steps():
    assert likelihood_time_steps(1000) == list(range(0, 1000, 100))
    assert likelihood_time_steps(20, 20) == list(range(20))
    assert likelihood_time_steps(1000, 3) == [0, 333, 666]
    for n in (0, 21):
        with pytest.raises(ValueError):
            likelihood_time_steps(20, n)


def _cpu_model(cfg=None):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    return ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)


def test_python_refusals():
    from targetdiff_b200.likelihood import ligand_nll
    b = synth.make_batch(1, 2, n_protein=30, ligand_sizes=[4, 5])
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    m = _cpu_model()
    for ts in ([0, 1000], [-1, 3]):
        with pytest.raises(ValueError, match='0..T-1'):
            m.likelihood_terms(*args, ts)
    with pytest.raises(ValueError, match='C0'):
        _cpu_model({'model_mean_type': 'noise'}).likelihood_terms(*args, [1, 2])
    data = {'protein_pos': b['protein_pos'][:30], 'protein_atom_feature': b['protein_v'][:30]}
    lig = [(b['init_ligand_pos'][:4], b['init_ligand_v'][:4])]
    with pytest.raises(ValueError, match='time embedding'):
        ligand_nll(_cpu_model({'time_emb_dim': 1, 'time_emb_mode': 'simple'}), data, lig, embedding=True)
    with pytest.raises(ValueError, match='C0'):
        ligand_nll(_cpu_model({'model_mean_type': 'noise'}), data, lig)
    with pytest.raises(ValueError, match='0..T-1'):
        ligand_nll(m, data, lig, time_steps=[1000])
    with pytest.raises(ValueError, match='ligand 0'):
        ligand_nll(m, data, [(torch.zeros(3, 2), torch.zeros(3, dtype=torch.long))])
    with pytest.raises(RuntimeError, match='CUDA'):                                  # no CPU path
        m.likelihood_terms(*args, [1, 2])


def test_cli_refusals(tmp_path):
    from targetdiff_b200.cli import main
    np.savez(tmp_path / 'l.npz', pos=np.zeros((3, 3), np.float32), v=np.zeros(3, np.int64))
    with pytest.raises(ValueError, match='not both'):
        main(['score_ligands', 'x.yml', '--ligand', str(tmp_path / 'l.npz'), '--samples', 'sample.pt', '--pdb_path', 'p.pdb'])
    with pytest.raises(ValueError, match='not both'):
        main(['score_ligands', 'x.yml'])
    with pytest.raises(ValueError, match='--pdb_path'):
        main(['score_ligands', 'x.yml', '--ligand', str(tmp_path / 'l.npz')])
