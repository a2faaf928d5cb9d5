"""Resampled sampling on a time path (DESIGN.md section 1), CPU side: the float64 identities of the re-noising step, the unit upward
tables, the RePaint path builder, the oracle on decreasing paths, the rng='cpu' driver's draws and the refusals."""
import math

import numpy as np
import pytest
import torch
import yaml

from oracle import resample, respaced, restate, synth
from targetdiff_b200.config import Config, check_resampling, sampling_time_path
from targetdiff_b200.sampling import resampled_time_path, respaced_time_seq
from targetdiff_b200.score_model import PATH_MAX_PER_T, check_time_path

K13 = synth.LIGAND_NUM_CLASSES
PAIRS = [(0, 1), (5, 6), (3, 400), (100, 101), (250, 999), (998, 999), (0, 999), (600, 620)]


@pytest.fixture(scope='module')
def sd():
    return synth.make_state_dict(0, schedules=restate.make_schedules())


def _abar(sums, t):
    return math.exp(sums[0][t]), math.exp(sums[1][t])


def _q_types(abar_v, K):
    """[K, K] float64 transition matrix q(v_t = j | v0 = i) = abar onehot + (1 - abar) / K."""
    return abar_v * np.eye(K) + (1.0 - abar_v) / K


# ------------------------------------------------------------------------------------------------ float64 identities
@pytest.mark.parametrize('t,p', PAIRS)
def test_renoise_keeps_the_forward_marginal(sd, t, p):
    """x_t ~ q(x_t | x0) re-noised to p has the mean and variance of q(x_p | x0); the same for the types."""
    sums = respaced.prefix_sums(sd)
    c = resample.renoise_coefficients(sd, t, p, sums)
    (at, avt), (ap, avp) = _abar(sums, t), _abar(sums, p)
    assert abs(c['c'] * math.sqrt(at) - math.sqrt(ap)) <= 1e-14
    assert abs(c['c'] ** 2 * (1.0 - at) + c['d'] ** 2 - (1.0 - ap)) <= 1e-14
    up = math.exp(c['lam']) * np.eye(K13) + math.exp(c['l1ma']) / K13
    np.testing.assert_allclose(_q_types(avt, K13) @ up, _q_types(avp, K13), rtol=0, atol=1e-13)


@pytest.mark.parametrize('t,m,p', [(0, 1, 2), (3, 400, 999), (10, 11, 500), (100, 600, 601)])
def test_two_renoise_jumps_compose(sd, t, m, p):
    sums = respaced.prefix_sums(sd)
    a, b, ab = (resample.renoise_coefficients(sd, x, y, sums) for x, y in ((t, m), (m, p), (t, p)))
    assert abs(a['c'] * b['c'] - ab['c']) <= 1e-14
    assert abs(b['c'] ** 2 * a['d'] ** 2 + b['d'] ** 2 - ab['d'] ** 2) <= 1e-14
    assert abs(a['lam'] + b['lam'] - ab['lam']) <= 1e-12
    mat = lambda c: math.exp(c['lam']) * np.eye(K13) + math.exp(c['l1ma']) / K13
    np.testing.assert_allclose(mat(a) @ mat(b), mat(ab), rtol=0, atol=1e-13)


@pytest.mark.parametrize('p,t', [(0, 1), (10, 60), (500, 999), (998, 999)])
def test_jump_down_then_renoise_up_returns_the_forward_process(sd, p, t):
    """With x0_hat = x0: x_t ~ q(x_t | x0), the jump posterior down to p, then a re-noise back up to t is q(x_t | x0) again."""
    sums = respaced.prefix_sums(sd)
    j = respaced.jump_coefficients(sd, t, p, sums)
    r = resample.renoise_coefficients(sd, p, t, sums)
    (at, avt), (ap, avp) = _abar(sums, t), _abar(sums, p)
    mean_p = j['c0'] + j['ct'] * math.sqrt(at)                      # per unit x0
    var_p = j['ct'] ** 2 * (1.0 - at) + j['var']
    assert abs(mean_p - math.sqrt(ap)) <= 1e-13 and abs(var_p - (1.0 - ap)) <= 1e-13
    assert abs(r['c'] * mean_p - math.sqrt(at)) <= 1e-13
    assert abs(r['c'] ** 2 * var_p + r['d'] ** 2 - (1.0 - at)) <= 1e-13
    # types: q(v_p | v_t, v0) marginalised over v_t ~ q(v_t | v0), then q(v_t' | v_p)
    K = K13
    qt, qp = _q_types(avt, K), _q_types(avp, K)
    step = math.exp(j['lam']) * np.eye(K) + math.exp(j['l1ma']) / K           # q(v_t | v_p)
    for v0 in (0, 5):
        post = qp[v0][:, None] * step                                          # [v_p, v_t] unnormalised q(v_p | v0) q(v_t | v_p)
        post = post / post.sum(0, keepdims=True)
        marg = (post * qt[v0][None, :]).sum(1)
        np.testing.assert_allclose(marg, qp[v0], rtol=0, atol=1e-13)
        np.testing.assert_allclose(marg @ step, qt[v0], rtol=0, atol=1e-13)


# ------------------------------------------------------------------------------------------------ tables
def test_unit_upward_tables_are_q_v_pred_one_timestep(sd):
    path = [999, 500, 501, 200, 0, 1, 0]
    tab = resample.path_tables(sd, path)
    g = torch.Generator().manual_seed(3)
    vt = torch.randint(0, K13, (40,), generator=g)
    u = torch.rand(40, K13, generator=g)
    for s in (1, 4):
        t, p = int(tab['t'][s]), int(tab['p'][s])
        assert p == t + 1
        assert tab['la'][s] == sd['log_alphas_v'][p].item() and tab['l1ma'][s] == sd['log_one_minus_alphas_v'][p].item()
        want = restate.q_v_pred_one_timestep(sd, restate.index_to_log_onehot(vt, K13), torch.tensor([p]), torch.zeros(40, dtype=torch.long), K13)
        out = resample.renoise_step(sd, tab, s, torch.zeros(40, 3), vt, torch.zeros(40, 3), u, K13)
        assert torch.equal(out['v'], restate.log_sample_categorical_from_uniform(want, u))
        assert torch.equal(out['vt'], want - torch.logsumexp(want, -1, keepdim=True))
    # the other rows: denoising steps are respaced.jump_tables', re-noising jumps the float64 coefficients rounded once
    down = respaced.jump_tables(sd, [999, 500])
    for k in ('c0', 'ct', 'logvar', 'la', 'l1ma'):
        assert tab[k][0] == down[k][0]
    c = resample.renoise_coefficients(sd, 0, 1)
    assert tab["c0"][4] == np.float32(c["c"]) and tab["ct"][4] == np.float32(c["d"])
    c = resample.renoise_coefficients(sd, 200, 999)
    jump = resample.path_tables(sd, [999, 200, 999, 0])
    assert (jump['c0'][1], jump['ct'][1], jump['la'][1], jump['l1ma'][1]) == tuple(np.float32(c[k]) for k in ('c', 'd', 'lam', 'l1ma'))


def test_renoise_step_fp32_is_the_kernels_rounding(sd):
    tab = resample.path_tables(sd, [999, 200, 999, 0])
    g = torch.Generator().manual_seed(5)
    x, eps = torch.randn(30, 3, generator=g) * 4, torch.randn(30, 3, generator=g)
    out = resample.renoise_step(sd, tab, 1, x, torch.zeros(30, dtype=torch.long), eps, torch.rand(30, K13, generator=g), K13, pos_only=True)
    c, d = np.float32(tab['c0'][1]), np.float32(tab['ct'][1])
    want = (c * x.numpy().astype(np.float32)).astype(np.float32) + (d * eps.numpy().astype(np.float32)).astype(np.float32)
    assert np.array_equal(out['pos'].numpy(), want.astype(np.float32))
    ref = resample.renoise_step(sd, tab, 1, x, torch.zeros(30, dtype=torch.long), eps, torch.rand(30, K13, generator=g), K13, pos_only=True,
                                dtype=torch.float64)
    assert float(((out['pos'].double() - ref['pos']).abs() / ref['scale']).max()) < 4e-7


# ------------------------------------------------------------------------------------------------ the RePaint path
def test_resampled_time_path_hand_examples():
    assert resampled_time_path(range(5, -1, -1), 2, 2) == [5, 4, 3, 5, 4, 3, 2, 1, 3, 2, 1, 0, 1, 0]
    assert resampled_time_path([9, 6, 3, 0], 3, 1) == [9, 6, 9, 6, 9, 6, 3, 6, 3, 6, 3, 0, 3, 0, 3, 0]
    assert resampled_time_path([9, 6, 3, 0], 2, 5) == [9, 6, 3, 0, 9, 6, 3, 0]
    assert resampled_time_path([4], 3, 2) == [4]
    assert resampled_time_path(respaced_time_seq(1000, 100), 1, 7) == respaced_time_seq(1000, 100)
    assert resampled_time_path(range(5, -1, -1), 2, 2) == resample.resampled_time_path(range(5, -1, -1), 2, 2)


@pytest.mark.parametrize('base', [list(range(999, -1, -1)), respaced_time_seq(1000, 100), respaced_time_seq(1000, 37, start=400),
                                  list(range(300, -1, -1)), [999, 998, 500, 2, 1]])
@pytest.mark.parametrize('r,j', [(1, 1), (2, 1), (5, 10), (3, 7), (4, 1000)])
def test_resampled_time_path_counts(base, r, j):
    path = resampled_time_path(base, r, j)
    n = len(base)
    up = sum(1 for a, b in zip(path, path[1:]) if b > a)
    assert len(path) - up == r * (n - 1) + 1 and up == (r - 1) * math.ceil((n - 1) / j)
    assert path[0] == base[0] and path[-1] == base[-1]
    assert check_time_path(path, 1000, start=None if base[0] == 999 else base[0]) == path
    assert path == resample.resampled_time_path(base, r, j)
    if r == 1:
        assert path == base


def test_resampled_time_path_refusals():
    for base, r, j in (([], 2, 1), ([5, 5, 0], 2, 1), ([5, 6, 0], 2, 1), ([5, -1], 2, 1), ([5, 0], 0, 1), ([5, 0], 2, 0)):
        with pytest.raises(ValueError):
            resampled_time_path(base, r, j)


# ------------------------------------------------------------------------------------------------ the oracle
def test_oracle_on_a_decreasing_path_is_respaced(sd):
    b = synth.make_batch(21, 2, n_protein=30, ligand_sizes=[7, 5])
    n = len(b['batch_ligand'])
    seq = [999, 998, 600, 37, 0]
    pn, vu = synth.make_tape(22, len(seq), n)
    mask = torch.zeros(n, dtype=torch.bool)
    mask[[0, 1, 7]] = True
    g = torch.Generator().manual_seed(23)
    ft = (torch.randn(len(seq) + 1, n, 3, generator=g), torch.rand(len(seq) + 1, n, K13, generator=g))
    args = tuple(b[k] for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))
    for fx in ({}, dict(fixed_mask=mask, fixed_tape=ft)):
        want = respaced.sample_diffusion(sd, None, *args, pn, vu, seq, **fx)
        got = resample.sample_diffusion(sd, None, *args, pn, vu, seq, **fx)
        for k in ('pos', 'v'):
            assert torch.equal(got[k], want[k])
        for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
            assert all(torch.equal(x, y) for x, y in zip(got[k], want[k])) and len(got[k]) == len(want[k])


def test_oracle_renoise_trajectory_entries(sd):
    b = synth.make_batch(24, 1, n_protein=30, ligand_sizes=[6])
    path = [999, 500, 900, 100, 0]
    pn, vu = synth.make_tape(25, len(path), 6)
    args = tuple(b[k] for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))
    r = resample.sample_diffusion(sd, None, *args, pn, vu, path, center_pos_mode='none')
    assert torch.equal(r['v0_traj'][1], r['v0_traj'][0])
    tab = resample.path_tables(sd, path)
    o = resample.renoise_step(sd, tab, 1, r['pos_traj'][0], r['v_traj'][0], pn[1], vu[1], K13)
    assert torch.equal(r['pos_traj'][1], o['pos']) and torch.equal(r['v_traj'][1], o['v']) and torch.equal(r['vt_traj'][1], o['vt'])


def test_driver_draws_are_a_time_seq_of_s_steps(sd):
    """oracle.resample's rng='cpu' driver consumes the generator as oracle.respaced's driver on any S-step sequence: on a decreasing path
    the outputs are equal, and a resampled path of S steps leaves the generator where an S-step time sequence does."""
    ppos = synth.make_batch(26, 1, n_protein=30, ligand_sizes=[4])['protein_pos']
    pfeat = synth.make_batch(26, 1, n_protein=30, ligand_sizes=[4])['protein_v']
    frag = (ppos.mean(0) + torch.randn(2, 3, generator=torch.Generator().manual_seed(1)), torch.tensor([2, 4]))
    seq = [999, 700, 300, 0]
    kw = dict(batch_size=2, sample_num_atoms='range', fixed_ligand=frag)
    torch.manual_seed(5)
    want = respaced.sample_diffusion_ligand(sd, None, ppos, pfeat, 3, None, seq, **kw)
    state_seq = torch.get_rng_state()
    torch.manual_seed(5)
    got = resample.sample_diffusion_ligand(sd, None, ppos, pfeat, 3, None, seq, **kw)
    assert torch.equal(torch.get_rng_state(), state_seq)
    for a, c in zip(got[:6], want[:6]):
        assert all(np.array_equal(x, y) for x, y in zip(a, c))
    path = [999, 700, 999, 300, 0]
    seq5 = [999, 700, 500, 300, 0]
    torch.manual_seed(5)
    respaced.sample_diffusion_ligand(sd, None, ppos, pfeat, 3, None, seq5, **kw)
    state5 = torch.get_rng_state()
    torch.manual_seed(5)
    r = resample.sample_diffusion_ligand(sd, None, ppos, pfeat, 3, None, path, **kw)
    assert torch.equal(torch.get_rng_state(), state5)
    assert r[2][0].shape[0] == len(path)


# ------------------------------------------------------------------------------------------------ refusals
def test_check_time_path_refusals():
    T = 20
    assert check_time_path([19, 5, 10, 0, 3, 1], T) == [19, 5, 10, 0, 3, 1]
    assert check_time_path(torch.tensor([7, 3, 7]), T, start=7) == [7, 3, 7]
    assert check_time_path([19], T) == [19]
    cases = {'empty': ([], None), 'more than': ([19] + [18, 19] * (PATH_MAX_PER_T * T // 2), None), 'start at T - 1': ([18, 5], None),
             'start time 7': ([19, 5], 7), 'outside 0..T-1': ([19, 3, 20], None), 'outside': ([19, 3, -1], None),
             'repeats time 3': ([19, 3, 3, 0], None), 'goes up at its first step': ([7, 9, 0], 7), 'start time 25': ([19], 25)}
    for msg, (path, start) in cases.items():
        with pytest.raises(ValueError, match=msg):
            check_time_path(path, T, start=start)
    assert len(check_time_path([19] + [18, 19] * (PATH_MAX_PER_T * T // 2 - 1), T)) == PATH_MAX_PER_T * T - 1


def test_sample_diffusion_refusals():
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(num_diffusion_timesteps=20)
    model = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K13)
    b = synth.make_batch(1, 1, n_protein=30, ligand_sizes=[3])
    args = tuple(b[k] for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))
    with pytest.raises(ValueError, match='cannot be combined with time_seq'):
        model.sample_diffusion(*args, time_seq=[19, 0], time_path=[19, 0])
    with pytest.raises(ValueError, match='num_steps=3 disagrees'):
        model.sample_diffusion(*args, num_steps=3, time_path=[19, 0, 5, 0])
    with pytest.raises(ValueError, match='goes up'):
        model.sample_diffusion(*args, time_path=[10, 12], start_time=10)


def test_config_refusals():
    assert check_resampling(Config(), False) == (1, 1)
    assert sampling_time_path(Config(), 20, None, False) is None
    assert sampling_time_path(Config(resamplings=2, jump_length=2), 6, None, True) == [5, 4, 3, 5, 4, 3, 2, 1, 3, 2, 1, 0, 1, 0]
    assert sampling_time_path(Config(resamplings=2), 20, [19, 10, 0], True) == [19, 10, 19, 10, 0, 10, 0]
    with pytest.raises(ValueError, match='needs held atoms'):
        check_resampling(Config(resamplings=2), False)
    for bad in (dict(resamplings=0), dict(resamplings=1.5), dict(jump_length=0), dict(jump_length=True), dict(resamplings='2')):
        with pytest.raises(ValueError, match='integer >= 1'):
            check_resampling(Config(bad), True)


def _conf(tmp_path, **sample):
    conf = {'model': {'checkpoint': str(tmp_path / 'missing.pt')},
            'sample': dict({'seed': 1, 'num_samples': 2, 'num_steps': 20, 'pos_only': False, 'center_pos_mode': 'protein',
                            'sample_num_atoms': 'range'}, **sample)}
    path = tmp_path / 'sample.yml'
    with open(path, 'w') as f:
        yaml.safe_dump(conf, f)
    return str(path)


def test_cli_refusals(tmp_path):
    """Refused before any checkpoint is read or device touched: resamplings without held atoms, in sample_for_pocket and in
    sample_pockets; a start ligand without 'keep' holds nothing either."""
    from targetdiff_b200.cli import main
    pdb = str(tmp_path / 'p.pdb')
    open(pdb, 'w').close()
    with pytest.raises(ValueError, match='needs held atoms'):
        main(['sample_for_pocket', _conf(tmp_path, resamplings=3), '--pdb_path', pdb, '--result_path', str(tmp_path / 'o')])
    torch.save({'pos': torch.zeros(3, 3), 'v': torch.tensor([0, 1, 2])}, tmp_path / 'start.pt')
    with pytest.raises(ValueError, match='needs held atoms'):
        main(['sample_for_pocket', _conf(tmp_path, resamplings=3, start_time=5), '--pdb_path', pdb, '--start_ligand', str(tmp_path / 'start.pt')])
    with pytest.raises(ValueError, match='integer >= 1'):
        main(['sample_for_pocket', _conf(tmp_path, jump_length=0), '--pdb_path', pdb])
    (tmp_path / 'pockets').mkdir()
    with pytest.raises(ValueError, match='needs held atoms'):
        main(['sample_pockets', _conf(tmp_path, resamplings=2), '--pocket_dir', str(tmp_path / 'pockets')])
