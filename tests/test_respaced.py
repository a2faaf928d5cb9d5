"""Respaced sampling (DESIGN.md section 1) on the CPU: the jump posteriors against float64 identities of the forward process, the
jump tables against the checkpoint's one-step tables, the oracle's respaced chain against restate.sample_diffusion on unit sequences,
respaced_time_seq, the driver's draw order and the Python-side refusals.  The engine side is tests/test_gpu_respaced.py."""
import math

import numpy as np
import pytest
import torch

from oracle import fixed_atoms, respaced, restate, synth
from targetdiff_b200.config import Config, default_model_config, sampling_time_seq
from targetdiff_b200.sampling import respaced_time_seq
from targetdiff_b200.score_model import diffusion_tables

K13 = synth.LIGAND_NUM_CLASSES
T20 = {'num_diffusion_timesteps': 20}


def _tables(schedule, T=1000):
    return diffusion_tables(Config(default_model_config(), beta_schedule=schedule, pos_beta_s=0.01, num_diffusion_timesteps=T))


SEQS_1000 = [respaced_time_seq(1000, 100), respaced_time_seq(1000, 20), respaced_time_seq(1000, 2), [999, 998, 600, 37, 36, 2, 0],
             [999, 500, 120, 40]]


def _log_add_exp(a, b):
    m = np.maximum(a, b)
    return m + np.log(np.exp(a - m) + np.exp(b - m))


def _type_posterior(c, lca_p, l1mca_p, K):
    """float64 q(v_p | v_t, v0) [v0, v_t, v_p] by the formula of DESIGN.md section 1 (log space, then normalised over v_p)."""
    eye = np.where(np.eye(K, dtype=bool), 0.0, -np.inf)
    a = _log_add_exp(eye[:, None, :] + lca_p, np.full((K, 1, K), l1mca_p - math.log(K)))             # [v0, 1, v_p]
    b = _log_add_exp(eye[None, :, :] + c['lam'], np.full((1, K, K), c['l1ma'] - math.log(K)))         # [1, v_t, v_p]
    un = a + b
    un = un - un.max(-1, keepdims=True)
    q = np.exp(un)
    return q / q.sum(-1, keepdims=True)


def _q_v(log_ac, K):
    """float64 q(v | v0) [v0, v] = ac * onehot + (1 - ac) / K with ac = exp(log_ac)."""
    ac = math.exp(log_ac)
    return ac * np.eye(K) + (1.0 - ac) / K


# ------------------------------------------------------------------------------------------------ float64 identities
@pytest.mark.parametrize('schedule', ['sigmoid', 'cosine'])
@pytest.mark.parametrize('K', [8, 13, 23])
def test_jump_is_the_forward_process(schedule, K):
    """Every step of several sequences, in float64: if x_t ~ q(x_t | x0), the jump sample c0 x0 + ct x_t + sigma eps has the mean
    sqrt(abar_p) x0 and the variance 1 - abar_p of q(x_p | x0); sum_{v_t} q(v_p | v_t, v0) q(v_t | v0) = q(v_p | v0)."""
    sd = _tables(schedule)
    la, lv = respaced.prefix_sums(sd)
    worst = [0.0, 0.0, 0.0]
    for seq in SEQS_1000:
        for t, p in respaced.targets(seq):
            if p < 0:
                continue
            c = respaced.jump_coefficients(sd, t, p)
            mean = c['c0'] + c['ct'] * math.sqrt(c['ac_t'])
            var = c['ct'] ** 2 * c['om_t'] + c['var']
            worst[0] = max(worst[0], abs(mean - math.sqrt(c['ac_p'])) / math.sqrt(c['ac_p']))
            worst[1] = max(worst[1], abs(var - c['om_p']) / c['om_p'])
            lca_p = lv[p]
            post = _type_posterior(c, lca_p, math.log(1.0 - math.exp(lca_p) + 1e-40), K)
            marg = np.einsum('ij,ijk->ik', _q_v(lv[t], K), post)
            worst[2] = max(worst[2], float(np.abs(marg - _q_v(lv[p], K)).max()))
    assert max(worst) < 1e-14, worst


@pytest.mark.parametrize('schedule', ['sigmoid', 'cosine'])
def test_two_jumps_compose_to_one(schedule):
    """t -> m -> p is t -> p in distribution: the composed position coefficients and variance, and the composed type kernel
    sum_{v_m} q(v_p | v_m, v0) q(v_m | v_t, v0), equal the single jump's (float64)."""
    sd = _tables(schedule)
    lv = respaced.prefix_sums(sd)[1]
    K = 13
    for t, m, p in ((999, 600, 37), (999, 998, 0), (500, 120, 119), (40, 20, 1), (37, 36, 2)):
        a, b, d = respaced.jump_coefficients(sd, t, m), respaced.jump_coefficients(sd, m, p), respaced.jump_coefficients(sd, t, p)
        assert abs(b['c0'] + b['ct'] * a['c0'] - d['c0']) <= 1e-13 * abs(d['c0']) + 1e-300
        assert abs(b['ct'] * a['ct'] - d['ct']) <= 1e-13 * abs(d['ct'])
        assert abs(b['ct'] ** 2 * a['var'] + b['var'] - d['var']) <= 1e-12 * d['var']
        f = lambda c, q: _type_posterior(c, lv[q], math.log(1.0 - math.exp(lv[q]) + 1e-40), K)
        composed = np.einsum('itm,imp->itp', f(a, m), f(b, p))
        assert np.abs(composed - f(d, p)).max() < 1e-13


@pytest.mark.parametrize('schedule', ['sigmoid', 'cosine'])
def test_unit_jump_is_the_checkpoint_step(schedule):
    """jump_coefficients(t, t - 1) is the checkpoint's one-step tables at t up to their rounding, and jump_tables takes the
    checkpoint's entries themselves on unit steps.  c0 and ct agree within 3 fp32 ulp on the sigmoid schedule.  On the cosine schedule
    the last betas lie near 0.999, so 1 - beta taken from the fp32 betas keeps only about 5 digits: 1e-5 there.  The type tables agree
    within 2e-6 relative."""
    sd = _tables(schedule)
    T = sd['betas'].shape[0]
    sums = respaced.prefix_sums(sd)
    pos_tol = 3.6e-7 if schedule == 'sigmoid' else 1e-5
    for t in range(1, T):
        c = respaced.jump_coefficients(sd, t, t - 1, sums)
        for k, name, tol in (('c0', 'posterior_mean_c0_coef', pos_tol), ('ct', 'posterior_mean_ct_coef', pos_tol),
                             ('lam', 'log_alphas_v', 2e-6), ('l1ma', 'log_one_minus_alphas_v', 2e-6)):
            ref = float(sd[name][t])
            assert abs(c[k] - ref) <= tol * abs(ref) + 1e-30, (t, k, c[k], ref)
        if t >= 2:            # posterior_logvar[0] repeats entry 1 (the reference's clip), and entry 1 is log of an fp32 variance
            assert abs(c['logvar'] - float(sd['posterior_logvar'][t])) < 1e-5
    seq = list(range(T - 1, -1, -1))
    tab = respaced.jump_tables(sd, seq)
    for k, name in (('c0', 'posterior_mean_c0_coef'), ('ct', 'posterior_mean_ct_coef'), ('logvar', 'posterior_logvar'),
                    ('la', 'log_alphas_v'), ('l1ma', 'log_one_minus_alphas_v')):
        assert np.array_equal(tab[k], sd[name].numpy()[::-1]), k
    assert np.array_equal(tab['p'], tab['t'] - 1)


def test_jump_tables_rounding():
    """Jump entries are the float64 coefficients rounded to fp32 once; 1 - abar comes from the betas, not from fp32 alphas_cumprod."""
    sd = _tables('sigmoid')
    seq = [999, 998, 600, 37, 36, 2, 0]
    tab = respaced.jump_tables(sd, seq)
    assert tab['t'].tolist() == seq and tab['p'].tolist() == seq[1:] + [-1]
    for s, (t, p) in enumerate(respaced.targets(seq)):
        if p == t - 1:
            continue
        c = respaced.jump_coefficients(sd, t, p)
        for k, ck in (('c0', 'c0'), ('ct', 'ct'), ('logvar', 'logvar'), ('la', 'lam'), ('l1ma', 'l1ma')):
            assert tab[k][s] == np.float32(c[ck])
    # at p = 0, 1 - abar_0 = betas[0] (about 5e-6): the prefix sums keep it to full precision; from fp32 alphas_cumprod it is 0.4 % off
    c = respaced.jump_coefficients(sd, 37, 0)
    beta0 = float(sd['betas'][0])
    assert abs(c['om_p'] - beta0) < 1e-15 * beta0
    assert abs((1.0 - float(sd["alphas_cumprod"][0])) - beta0) > 1e-3 * beta0


# ------------------------------------------------------------------------------------------------ the oracle's chain
def _setup(S, cfg=T20, seed=5, sizes=(6, 9)):
    sd = synth.make_state_dict(seed, cfg, schedules=restate.make_schedules(cfg))
    b = synth.make_batch(seed + 1, len(sizes), n_protein=30, ligand_sizes=list(sizes))
    n = len(b['batch_ligand'])
    pn, vu = synth.make_tape(seed + 2, S, n)
    g = torch.Generator().manual_seed(seed + 3)
    ft = (torch.randn(S + 1, n, 3, generator=g), torch.rand(S + 1, n, K13, generator=g))
    mask = torch.zeros(n, dtype=torch.bool)
    mask[[0, 2, sizes[0] + 1]] = True
    return sd, b, pn, vu, ft, mask


def _args(sd, cfg, b, pn, vu):
    return (sd, cfg, b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'],
            pn, vu)


def _same(r1, r2):
    for k in ('pos', 'v'):
        assert torch.equal(r1[k], r2[k]), k
    for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
        assert len(r1[k]) == len(r2[k]) and all(torch.equal(x, y) for x, y in zip(r1[k], r2[k])), k


@pytest.mark.parametrize('cfg,pos_only', [(T20, False), (T20, True), (dict(T20, model_mean_type='noise'), False),
                                          (dict(T20, time_emb_dim=1), False)])
def test_oracle_unit_sequences_are_the_reference_chain(cfg, pos_only):
    """The respaced oracle on T-1..0 and on T-1..T-S is restate.sample_diffusion(num_steps) bit for bit (which is pinned to the
    reference), and with a fixed set fixed_atoms.sample_diffusion."""
    for S in (20, 5):
        sd, b, pn, vu, ft, mask = _setup(S, cfg)
        seq = list(range(19, 19 - S, -1))
        a = _args(sd, cfg, b, pn, vu)
        _same(respaced.sample_diffusion(*a, seq, pos_only=pos_only), restate.sample_diffusion(*a, num_steps=S, pos_only=pos_only))
        if S == 5:
            _same(respaced.sample_diffusion(*a, seq, pos_only=pos_only, fixed_mask=mask, fixed_tape=ft),
                  fixed_atoms.sample_diffusion(*a, mask, ft, num_steps=S, pos_only=pos_only))


@pytest.mark.parametrize('pos_only', [False, True])
def test_jump_step_is_the_oracle_chain_step(pos_only):
    """respaced.jump_step at fp32, on each step's input state and network outputs, is that step of respaced.sample_diffusion bit for
    bit (unit and jump steps, through t = 0); at float64 it agrees within stepwise.STEP_TOL."""
    from oracle import stepwise
    seq = [19, 12, 11, 4, 0]
    sd, b, pn, vu, _, _ = _setup(len(seq))
    tab = respaced.jump_tables(sd, seq)
    seen = []
    r = respaced.sample_diffusion(*_args(sd, None, b, pn, vu), seq, center_pos_mode='none', pos_only=pos_only,
                                  step_callback=lambda s, i, preds, pos, v: seen.append(preds))
    for s in range(len(seq)):
        xt = b['init_ligand_pos'] if s == 0 else r['pos_traj'][s - 1]
        vt = b['init_ligand_v'] if s == 0 else r['v_traj'][s - 1]
        a = (sd, None, tab, s, xt, vt, seen[s]['pred_ligand_pos'], seen[s]['pred_ligand_v'], pn[s], vu[s])
        got = respaced.jump_step(*a, pos_only=pos_only)
        assert torch.equal(got['pos'], r['pos_traj'][s]) and torch.equal(got['v'], r['v_traj'][s]), s
        if not pos_only:
            assert torch.equal(got['v0'], r['v0_traj'][s]) and torch.equal(got['vt'], r['vt_traj'][s]), s
        e = stepwise.errors(got['pos'], got['v'], got['v0'], got['vt'], respaced.jump_step(*a, pos_only=pos_only, dtype=torch.float64))
        assert e['v_diff'] == 0 and all(e[k] <= lim for k, lim in stepwise.STEP_TOL.items()), (s, e)


def test_oracle_jump_chain_fixed_rows():
    """On a jump sequence the fixed rows after step s are q(x_p | x0_f) from fixed-tape row s + 1 at p (float64 closed form within
    fp32 rounding), and x0_f / v0_f exactly after the step at 0."""
    seq = [19, 12, 11, 4, 0]
    S = len(seq)
    sd, b, pn, vu, ft, mask = _setup(S)
    r = respaced.sample_diffusion(*_args(sd, None, b, pn, vu), seq, fixed_mask=mask, fixed_tape=ft)
    _, x0c, off = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    off = off[b['batch_ligand']][mask].double()
    x0 = x0c[mask].double()
    for s, (t, p) in enumerate(respaced.targets(seq)):
        got = r['pos_traj'][s][mask].double()
        if p < 0:
            assert torch.equal(r['pos_traj'][s][mask], b['init_ligand_pos'][mask])
            assert torch.equal(r['v_traj'][s][mask], b['init_ligand_v'][mask])
            continue
        ac = float(sd['alphas_cumprod'][p])
        want = math.sqrt(ac) * x0 + math.sqrt(1.0 - ac) * ft[0][s + 1][mask].double() + off
        assert float((got - want).abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------------ time sequences and refusals
def test_respaced_time_seq():
    assert respaced_time_seq(1000, 2) == [999, 0]
    assert respaced_time_seq(1000, 1000) == list(range(999, -1, -1))
    assert respaced_time_seq(10, 4) == [9, 6, 3, 0]
    assert respaced_time_seq(1000, 4) == [999, 666, 333, 0]
    assert respaced_time_seq(1000, 3) == [999, 500, 0]          # 499.5 rounds half to even
    for T in (2, 3, 20, 1000):
        for n in range(2, T + 1):
            seq = respaced_time_seq(T, n)
            assert len(seq) == n and seq[0] == T - 1 and seq[-1] == 0 and all(b < a for a, b in zip(seq, seq[1:]))
            assert max(abs(x - (T - 1) * (n - 1 - i) / (n - 1)) for i, x in enumerate(seq)) <= 0.5
    for T, n in ((1000, 1), (1000, 0), (1000, 1001), (1, 1), (20, -3)):
        with pytest.raises(ValueError):
            respaced_time_seq(T, n)


class _Recorder:
    """Stands in for ScorePosNet3D in sample_diffusion_ligand: records what the driver hands to sample_diffusion."""
    num_classes, num_timesteps = K13, 20

    def __init__(self):
        self.calls = []

    def sample_diffusion(self, **kw):
        self.calls.append(kw)
        n, S = len(kw['batch_ligand']), len(kw['time_seq']) if kw.get('time_seq') is not None else kw['num_steps']
        return {'pos': kw['init_ligand_pos'].clone(), 'v': kw['init_ligand_v'].clone(), 'pos_traj': torch.zeros(S, n, 3),
                'v_traj': torch.zeros(S, n, dtype=torch.long), 'v0_traj': torch.zeros(S, n, K13), 'vt_traj': torch.zeros(S, n, K13)}


def _pocket(n=40):
    from targetdiff_b200.data import ProteinLigandData
    b = synth.make_batch(9, 1, n_protein=n, ligand_sizes=[1])
    return ProteinLigandData(protein_pos=b['protein_pos'], protein_atom_feature=b['protein_v'])


def test_driver_cpu_draw_order_with_a_fragment():
    """rng='cpu' with a time sequence of S steps: S interleaved steps of draws, then the fixed tape [S+1, ...]; the oracle's driver
    restatement consumes the generator the same way and hands the same tapes to its chain."""
    from targetdiff_b200.sampling import sample_diffusion_ligand
    data = _pocket()
    seq = [19, 11, 3, 0]
    S = len(seq)
    frag = (torch.randn(2, 3) + 10.0, torch.tensor([1, 4]))
    model = _Recorder()
    torch.manual_seed(21)
    sample_diffusion_ligand(model, data, 4, batch_size=4, device='cpu', sample_num_atoms='range', rng='cpu', fixed_ligand=frag,
                            time_seq=seq)
    kw = model.calls[0]
    assert kw['time_seq'] == seq and kw['num_steps'] is None
    n = len(kw['batch_ligand'])
    torch.manual_seed(21)
    torch.randn(n, 3), torch.rand(n, K13)
    pn, vu = torch.empty(S, n, 3), torch.empty(S, n, K13)
    for s in range(S):
        pn[s], vu[s] = torch.randn(n, 3), torch.rand(n, K13)
    fpn, fvu = torch.randn(S + 1, n, 3), torch.rand(S + 1, n, K13)
    assert torch.equal(kw['noise_tape'][0], pn) and torch.equal(kw['noise_tape'][1], vu)
    assert torch.equal(kw['fixed_noise_tape'][0], fpn) and torch.equal(kw['fixed_noise_tape'][1], fvu)
    seen = []
    real = respaced.sample_diffusion
    try:
        respaced.sample_diffusion = lambda *a, **k: seen.append((a, k)) or real(*a, **k)
        sd = synth.make_state_dict(0, T20, schedules=restate.make_schedules(T20))
        torch.manual_seed(21)
        respaced.sample_diffusion_ligand(sd, T20, data.protein_pos, data.protein_atom_feature, 4, None, seq, batch_size=4,
                                         sample_num_atoms='range', fixed_ligand=frag)
    finally:
        respaced.sample_diffusion = real
    a, k = seen[0]
    assert torch.equal(a[8], pn) and torch.equal(a[9], vu) and a[10] == seq
    assert torch.equal(k['fixed_mask'], kw['fixed_mask'])
    assert torch.equal(k['fixed_tape'][0], fpn) and torch.equal(k['fixed_tape'][1], fvu)
    assert torch.equal(a[6], kw['init_ligand_v'])


def test_driver_without_time_seq_is_unchanged():
    from targetdiff_b200.sampling import sample_diffusion_ligand
    model = _Recorder()
    sample_diffusion_ligand(model, _pocket(), 2, batch_size=2, device='cpu', num_steps=3, sample_num_atoms='range', rng='cpu')
    assert 'time_seq' not in model.calls[0] and model.calls[0]['num_steps'] == 3
    assert model.calls[0]['noise_tape'][0].shape[0] == 3


def test_python_refusals():
    """ScorePosNet3D.sample_diffusion and the driver refuse bad time sequences with ValueError before they touch a device."""
    from targetdiff_b200.sampling import sample_diffusion_ligand
    from targetdiff_b200.score_model import ScorePosNet3D
    model = ScorePosNet3D(default_model_config(), synth.PROTEIN_FEATURE_DIM, K13)
    T = model.num_timesteps
    b = synth.make_batch(1, 1, n_protein=20, ligand_sizes=[4])
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    bad = lambda T: {'empty': [], 'more than T': list(range(T, -1, -1)) + [-1], 'start at T - 1': [T - 2, 0],
                     'strictly decreasing': [T - 1, 5, 5, 0], 'negative': [T - 1, 3, -1]}
    for msg, seq in bad(T).items():
        with pytest.raises(ValueError, match=msg):
            model.sample_diffusion(*args, time_seq=seq)
    for msg, seq in bad(_Recorder.num_timesteps).items():
        with pytest.raises(ValueError, match=msg):
            sample_diffusion_ligand(_Recorder(), _pocket(), 1, device='cpu', sample_num_atoms='range', time_seq=seq)
    with pytest.raises(ValueError, match='disagrees'):
        model.sample_diffusion(*args, num_steps=3, time_seq=[T - 1, 0])
    with pytest.raises(ValueError, match='disagrees'):
        sample_diffusion_ligand(_Recorder(), _pocket(), 1, device='cpu', sample_num_atoms='range', num_steps=20, time_seq=[19, 0])


def test_config_respaced_steps():
    """sample.respaced_steps = n gives respaced_time_seq(T, n); None is the default chain; it is refused with num_steps != T."""
    T = 1000
    assert sampling_time_seq(Config(num_steps=1000), T) is None
    assert sampling_time_seq(Config(num_steps=1000, respaced_steps=None), T) is None
    assert sampling_time_seq(Config(num_steps=1000, respaced_steps=100), T) == respaced_time_seq(T, 100)
    assert sampling_time_seq(Config(respaced_steps=50), T) == respaced_time_seq(T, 50)
    with pytest.raises(ValueError, match='num_steps'):
        sampling_time_seq(Config(num_steps=500, respaced_steps=100), T)
    with pytest.raises(ValueError):
        sampling_time_seq(Config(num_steps=1000, respaced_steps=1), T)
