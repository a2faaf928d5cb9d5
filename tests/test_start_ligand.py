"""Start-ligand sampling (DESIGN.md section 1) on the CPU: the host start stream's statistics in float64, its Philox domains, the time
sequences from a start time, the oracle chain's decoder step, and the refusals of the driver, the config and the CLI."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import fixed_atoms, philox, restate, start_ligand, synth
from targetdiff_b200.config import Config, sampling_start, sampling_time_seq
from targetdiff_b200.sampling import respaced_time_seq
from targetdiff_b200.score_model import check_time_seq

K13 = synth.LIGAND_NUM_CLASSES
T = 1000


@pytest.fixture(scope='module')
def sched():
    return restate.make_schedules()


# ------------------------------------------------------------------------------------------------ the start stream
@pytest.mark.parametrize('t0', [0, 1, 37, 500, T - 1])
def test_start_positions_are_the_forward_process(sched, t0):
    """(x - sqrt(abar) x0) / sqrt(1 - abar) of float64 start draws is N(0,1) (KS), on 20000 atoms with spread-out x0."""
    n = 20000
    rng = np.random.default_rng(t0)
    x0 = rng.normal(0.0, 5.0, (n, 3))
    eps = start_ligand.start_position_normals(2 ** 33 + t0, np.arange(n, dtype=np.uint32))
    ab = float(sched['alphas_cumprod'][t0])
    x = math.sqrt(ab) * x0 + math.sqrt(1.0 - ab) * eps
    z = ((x - math.sqrt(ab) * x0) / math.sqrt(1.0 - ab)).reshape(-1)
    assert stats.kstest(z, 'norm').pvalue > 1e-3
    assert abs(z.mean()) < 0.02 and abs(z.std() - 1.0) < 0.02


@pytest.mark.parametrize('t0', [0, 1, 300, T - 1])
def test_start_types_are_the_forward_process(sched, t0):
    """Gumbel-max over log q(v_t0 | v0) with the start stream's uniforms: class frequencies match q (chi-square, sparse classes
    pooled)."""
    n = 40000
    v0 = np.arange(n) % K13
    u = start_ligand.start_type_uniforms(7 + t0, np.arange(n, dtype=np.uint32), K13)
    lq = restate.q_v_pred({k: sched[k].double() for k in sched}, restate.index_to_log_onehot(torch.from_numpy(v0), K13).double(),
                          torch.full((1,), t0), torch.zeros(n, dtype=torch.long), K13).numpy()
    q = np.exp(lq - lq.max(1, keepdims=True))
    q /= q.sum(1, keepdims=True)
    draw = np.argmax(-np.log(-np.log(u + 1e-30) + 1e-30) + lq, 1)
    for c in range(K13):                      # each start class separately: q(v_t0 | v0 = c)
        rows = v0 == c
        obs = np.bincount(draw[rows], minlength=K13).astype(np.float64)
        exp = q[rows][0] * rows.sum()
        big = exp >= 5
        o = np.append(obs[big], obs[~big].sum())
        e = np.append(exp[big], exp[~big].sum())
        if e[-1] < 5:                         # fold a pooled remainder below 5 into the largest class
            j = int(np.argmax(e[:-1]))
            o[j] += o[-1]; e[j] += e[-1]
            o, e = o[:-1], e[:-1]
        if len(e) < 2:                        # q is nearly one-hot: the number of draws away from c is binomial
            assert stats.binomtest(int(rows.sum() - obs[c]), int(rows.sum()), float(1.0 - q[rows][0][c])).pvalue > 1e-4, (t0, c)
            continue
        assert stats.chisquare(o, e).pvalue > 1e-4, (t0, c)


def test_start_domains_are_distinct():
    words = {'pst\0': 0x70737400, 'vuni': 0x76756E69, 'fxps': fixed_atoms.FIX_POS_DOMAIN, 'fxtv': fixed_atoms.FIX_TYPE_DOMAIN,
             'stps': start_ligand.START_POS_DOMAIN, 'sttv': start_ligand.START_TYPE_DOMAIN}
    for name, w in words.items():
        assert int.from_bytes(name.encode(), 'big') == w
    assert len(set(words.values())) == 6


def test_start_tape_layout():
    """start_tape row a is atom a's counter (a, 0, ., domain); it differs from the fixed stream's draw 0 and the sampler's step 0."""
    pn, vu = start_ligand.start_tape(123, 9, K13)
    assert pn.shape == (9, 3) and vu.shape == (9, K13) and pn.dtype == torch.float32
    a = np.arange(9, dtype=np.uint32)
    assert torch.equal(pn, torch.from_numpy(start_ligand.start_position_normals(123, a).astype(np.float32)))
    fpn, _ = fixed_atoms.fixed_tape(123, 9, 0, K13)
    spn, _ = philox.engine_tape(123, 9, 1, K13)
    assert not torch.equal(pn, fpn[0]) and not torch.equal(pn, spn[0])
    assert torch.equal(start_ligand.start_tape(123, 9, K13, pos_only=True)[1], torch.zeros(9, K13))


# ------------------------------------------------------------------------------------------------ time sequences
@pytest.mark.parametrize('start,n', [(500, 50), (500, 501), (999, 100), (1, 2), (7, 3), (0, 1), (40, 2)])
def test_respaced_time_seq_from_start(start, n):
    seq = respaced_time_seq(T, n, start=start)
    assert len(seq) == n and seq[0] == start and seq[-1] == 0 and all(b < a for a, b in zip(seq, seq[1:]))
    assert check_time_seq(seq, T, start=start) == seq


def test_respaced_time_seq_without_start_is_unchanged():
    for TT, n in ((1000, 100), (1000, 20), (20, 6), (20, 20), (7, 2)):
        assert respaced_time_seq(TT, n) == respaced_time_seq(TT, n, start=None) == \
            [int(x) for x in np.rint(np.linspace(TT - 1, 0, n))]
    assert respaced_time_seq(T, n=T - 0, start=T - 1) == respaced_time_seq(T, T)
    with pytest.raises(ValueError, match='2..T'):
        respaced_time_seq(T, 1)


@pytest.mark.parametrize('start,n', [(500, 502), (500, 1), (0, 2), (-1, 2), (T, 2)])
def test_respaced_time_seq_from_start_refusals(start, n):
    with pytest.raises(ValueError):
        respaced_time_seq(T, n, start=start)


def test_check_time_seq_with_and_without_start():
    assert check_time_seq([999, 500, 0], T) == [999, 500, 0]
    with pytest.raises(ValueError, match='T - 1'):
        check_time_seq([500, 0], T)
    assert check_time_seq([500, 0], T, start=500) == [500, 0]
    assert check_time_seq(list(range(500, -1, -1)), T, start=500)[-1] == 0
    assert check_time_seq([0], T, start=0) == [0]
    for seq, start, msg in (([999, 0], 500, 'start time 500'), ([500, 500, 0], 500, 'strictly'), ([500, -1], 500, 'negative'),
                            ([5, 0], -1, 'outside'), ([5, 0], T, 'outside'), ([], 5, 'empty')):
        with pytest.raises(ValueError, match=msg):
            check_time_seq(seq, T, start=start)


# ------------------------------------------------------------------------------------------------ the oracle chain
def test_oracle_decoder_step_ends_on_the_network_x0():
    """A chain from t0 = 0 is one decoder step: sigma = 0 and c0 = 1, ct = 0, so it ends on the network's x0 for the start state."""
    sd = synth.make_state_dict(0, schedules=restate.make_schedules())
    b = synth.make_batch(3, 2, n_protein=30, ligand_sizes=[6, 4])
    n = len(b['batch_ligand'])
    pn, vu = synth.make_tape(4, 1, n)
    st = start_ligand.start_tape(5, n, K13)
    r = start_ligand.sample_diffusion(sd, None, *[b[k] for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos',
                                                                 'init_ligand_v', 'batch_ligand')], pn, vu, 0, st)
    pp, x0, off = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    xs, vs = start_ligand.start_state(sd, x0, b['init_ligand_v'], b['batch_ligand'], 0, st, K13)
    out = restate.forward(sd, None, pp, b['protein_v'], b['batch_protein'], xs, vs, b['batch_ligand'],
                          time_step=torch.zeros(2, dtype=torch.long))
    assert len(r['pos_traj']) == 1
    assert torch.equal(r['pos'], out['pred_ligand_pos'] + off[b['batch_ligand']])


def test_oracle_kept_rows_end_on_the_start_ligand():
    sd = synth.make_state_dict(1, schedules=restate.make_schedules())
    b = synth.make_batch(8, 1, n_protein=30, ligand_sizes=[7])
    n = len(b['batch_ligand'])
    seq = [40, 20, 3, 0]
    mask = torch.tensor([True, False, True, False, False, False, False])
    pn, vu = synth.make_tape(9, len(seq), n)
    ft = fixed_atoms.fixed_tape(10, n, len(seq), K13)
    r = start_ligand.sample_diffusion(sd, None, *[b[k] for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos',
                                                                 'init_ligand_v', 'batch_ligand')], pn, vu, 40,
                                      start_ligand.start_tape(11, n, K13), seq, fixed_mask=mask, fixed_tape=ft)
    assert len(r['pos_traj']) == 4
    torch.testing.assert_close(r['pos'][mask], b['init_ligand_pos'][mask], rtol=2 ** -22, atol=0)
    assert torch.equal(r['v'][mask], b['init_ligand_v'][mask])


# ------------------------------------------------------------------------------------------------ refusals
def _model():
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    return ScorePosNet3D(default_model_config(), synth.PROTEIN_FEATURE_DIM, K13)


@pytest.mark.parametrize('kw,msg', [
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4])), fixed_ligand=(torch.zeros(1, 3), torch.tensor([1])),
          start_time=10), 'keep_atoms'),
    (dict(start_time=10), 'start_ligand'),
    (dict(keep_atoms=[0]), 'start_ligand'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4]))), 'start_time'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, K13])), start_time=10), 'classes'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1., 2., 3., 4.])), start_time=10), 'integer'),
    (dict(start_ligand=(torch.zeros(4, 2), torch.tensor([1, 2, 3, 4])), start_time=10), r'\[n,3\]'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4])), start_time=T), 'outside'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4])), start_time=10, keep_atoms=[4]), '0..3'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4])), start_time=10, keep_atoms=[-1]), '0..3'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4])), start_time=10, keep_atoms=[1, 1]), 'unique'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4])), start_time=10, keep_atoms=[0, 1, 2, 3]), 'free'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4])), start_time=10, time_seq=[999, 0]), 'start time 10'),
    (dict(start_ligand=(torch.zeros(4, 3), torch.tensor([1, 2, 3, 4])), start_time=10, num_steps=1000), 'num_steps'),
])
def test_driver_refusals(kw, msg):
    from targetdiff_b200.sampling import sample_diffusion_ligand
    data = Config(protein_pos=torch.zeros(5, 3), protein_atom_feature=torch.zeros(5, 27))
    with pytest.raises(ValueError, match=msg):
        sample_diffusion_ligand(_model(), data, 2, device='cpu', **kw)


def test_config_start():
    s = Config(num_steps=1000, start_time=500)
    assert sampling_start(s, T, True) == (500, list(range(500, -1, -1)))
    s = Config(num_steps=1000, start_time=500, respaced_steps=50)
    t0, seq = sampling_start(s, T, True)
    assert t0 == 500 and seq == respaced_time_seq(T, 50, start=500) and len(seq) == 50
    assert sampling_start(Config(num_steps=1000), T, False) == (None, None)
    assert sampling_time_seq(Config(num_steps=1000, respaced_steps=50), T) == respaced_time_seq(T, 50)
    for sample, have, msg in ((Config(num_steps=1000), True, 'needs sample.start_time'),
                              (Config(num_steps=1000, start_time=5), False, 'needs a start ligand'),
                              (Config(num_steps=100, start_time=5), True, 'num_steps'),
                              (Config(num_steps=1000, start_time=T), True, 'outside'),
                              (Config(num_steps=1000, start_time=5, respaced_steps=7), True, '2..6')):
        with pytest.raises(ValueError, match=msg):
            sampling_start(sample, T, have)


@pytest.mark.parametrize('fmt', ['pt', 'npz'])
def test_load_start_ligand(tmp_path, fmt):
    from targetdiff_b200.cli import load_start_ligand
    pos, v = np.arange(12, dtype=np.float32).reshape(4, 3), np.array([1, 2, 3, 4])

    def write(name, **d):
        p = str(tmp_path / ('%s.%s' % (name, fmt)))
        if fmt == 'pt':
            torch.save({k: torch.as_tensor(x) for k, x in d.items()}, p)
        else:
            np.savez(p, **d)
        return p

    p_, v_, k_ = load_start_ligand(write('plain', pos=pos, v=v))
    assert torch.equal(p_, torch.from_numpy(pos)) and v_.tolist() == [1, 2, 3, 4] and k_ is None
    _, _, k_ = load_start_ligand(write('keep', pos=pos, v=v, keep=np.array([0, 2], np.int32)))
    assert k_.dtype == torch.int64 and k_.tolist() == [0, 2]
    for name, d, msg in (('fkeep', dict(pos=pos, v=v, keep=np.array([0.0, 2.0])), 'keep'),
                         ('k2d', dict(pos=pos, v=v, keep=np.array([[0, 1]])), 'keep'),
                         ('nov', dict(pos=pos), "'pos'"),
                         ('fv', dict(pos=pos, v=v.astype(np.float32)), 'integer')):
        with pytest.raises(ValueError, match=msg):
            load_start_ligand(write(name, **d))
    with pytest.raises(ValueError, match='.pt or .npz'):
        load_start_ligand(str(tmp_path / 'x.sdf'))


def test_cli_refuses_fragment_with_start_ligand(tmp_path):
    from targetdiff_b200.cli import main
    with pytest.raises(ValueError, match='--fragment cannot be combined with --start_ligand'):
        main(['sample_for_pocket', str(tmp_path / 'none.yml'), '--pdb_path', 'x.pdb', '--fragment', 'a.pt', '--start_ligand', 'b.pt'])


def test_cli_sample_pockets_refuses_start_time(tmp_path):
    import yaml
    from targetdiff_b200.cli import main
    with open(tmp_path / 's.yml', 'w') as f:
        yaml.safe_dump({'model': {'checkpoint': 'none.pt'}, 'sample': {'seed': 1, 'num_samples': 1, 'num_steps': 1000,
                                                                       'start_time': 5}}, f)
    with pytest.raises(ValueError, match='start ligand'):
        main(['sample_pockets', str(tmp_path / 's.yml'), '--pocket_dir', str(tmp_path)])
