"""Resampled sampling on a time path (DESIGN.md section 1) on the engine (run with -m gpu; `pytest -s` prints the errors).

A. A strictly decreasing path through tdiff_sample_path is tdiff_sample_seq's chain bit for bit; launches per step.
B. Resampled chains (fragment; start ligand with kept atoms) against oracle.resample on noise tapes: the whole chain within the respaced
   tests' tolerances, every re-noising step bit for bit (positions and types) from the engine's own state, fixed rows on the closed
   form at p, and the trajectory contents.
C. Every re-noising step against float64.
D. The seeded stream equals philox.engine_tape; graph replay equals TDIFF_NO_GRAPH=1; the incremental caches' switches change nothing.
E. The rng='cpu' driver on the 1h36 pocket against oracle.resample's driver; the CLI with sample.resamplings and --fragment.
F. Refusals through the C-ABI."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import fixed_atoms, philox, resample, restate, stepwise, synth
from targetdiff_b200.sampling import resampled_time_path, respaced_time_seq

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K13 = synth.LIGAND_NUM_CLASSES
EPS32 = 2.0 ** -23
POS_RTOL, POS_ATOL, LOGIT_ATOL = 1e-4, 1e-5, 1e-3
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')
PATH = resampled_time_path(respaced_time_seq(1000, 10), resamplings=3, jump_length=3)       # 28 denoising, 6 re-noising steps
PDB_1H36 = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', '1h36_pocket10.pdb')


def _model(cfg=None, weight_seed=0):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K13)
    sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg))
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ARGS)


def _mask(b, lead=3):
    bl = b['batch_ligand']
    m = torch.zeros(len(bl), dtype=torch.bool)
    start = 0
    for n in torch.bincount(bl).tolist():
        m[start:start + min(lead, n - 1)] = True
        start += n
    return m


def _fixed_tape(seed, S, n):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(S + 1, n, 3, generator=g), torch.rand(S + 1, n, K13, generator=g)


def _sample(model, b, seq=None, path=None, mask=None, ft=None, tape=None, mode='protein', **kw):
    r = model.sample_diffusion(*_args(b), time_seq=seq, time_path=path, center_pos_mode=mode, noise_tape=tape, stack_traj=True,
                               fixed_mask=None if mask is None else mask.to(DEV), fixed_noise_tape=ft, **kw)
    return {k: (r[k].cpu() if torch.is_tensor(r[k]) else r[k]) for k in TRAJ}


def _differing(a, c):
    return [k for k in TRAJ if not (a[k] is None and c[k] is None) and not torch.equal(a[k], c[k])]


def _origin_batch(seed, sizes, n_protein=40):
    b = synth.make_batch(seed, len(sizes), n_protein=n_protein, ligand_sizes=sizes, distinct_pockets=1)
    shift = b['protein_pos'].mean(0, keepdim=True)
    b['protein_pos'], b['init_ligand_pos'] = b['protein_pos'] - shift, b['init_ligand_pos'] - shift
    return b


# ------------------------------------------------------------------------------------------------ A. decreasing paths, launches
@pytest.mark.parametrize('noise,fixed,pos_only', [('tape', False, False), ('seed', True, False), ('tape', True, False),
                                                  ('seed', False, True), ('tape', True, True)])
def test_decreasing_path_is_the_respaced_chain(noise, fixed, pos_only):
    model, _ = _model()
    b = synth.make_batch(11, 3, n_protein=50, ligand_sizes=[9, 14, 5])
    n = len(b['batch_ligand'])
    seq = [999, 998, 600, 37, 36, 2, 0]
    kw = dict(tape=synth.make_tape(12, len(seq), n)) if noise == 'tape' else dict(seed=2 ** 40 + 3)
    if fixed:
        kw.update(mask=_mask(b), ft=_fixed_tape(13, len(seq), n) if noise == 'tape' else None)
    assert not _differing(_sample(model, b, seq=seq, pos_only=pos_only, **kw), _sample(model, b, path=seq, pos_only=pos_only, **kw))


@pytest.mark.parametrize('fixed', [False, True])
def test_launches_per_step(fixed):
    """Each denoising step of a path issues the respaced chain's launches, each re-noising step 2."""
    from targetdiff_b200 import _lib
    lib = _lib.load()
    b = synth.make_batch(6, 2, n_protein=150, ligand_sizes=[20, 7])
    mask = _mask(b) if fixed else None
    counts = {}
    for name, kw in (('seq', dict(seq=[999, 500, 200, 0])), ('path', dict(path=[999, 500, 700, 200, 0])),
                     ('path3', dict(path=[999, 500, 700, 200, 400, 100, 0]))):
        model, _ = _model(weight_seed=3)
        model.sample_diffusion(*_args(b), time_seq=kw.get('seq'), time_path=kw.get('path'), center_pos_mode='protein', return_traj=False,
                               fixed_mask=None if mask is None else mask.to(DEV))
        counts[name] = lib.tdiff_launch_count(model.engine(DEV))
        model._drop_engine()
    model, _ = _model(weight_seed=3)
    model.sample_diffusion(*_args(b), time_seq=[999, 500, 200, 100, 0], center_pos_mode='protein', return_traj=False,
                           fixed_mask=None if mask is None else mask.to(DEV))
    counts['seq5'] = lib.tdiff_launch_count(model.engine(DEV))
    model._drop_engine()
    print('launches:', counts)
    assert counts['path'] == counts['seq'] + 2
    assert counts['path3'] == counts['seq5'] + 4


# ------------------------------------------------------------------------------------------------ B. against the oracle
def _chain_case(case):
    """(model, sd, batch, path, tape, oracle kwargs, engine kwargs) of a resampled chain with held atoms, pockets at the origin."""
    model, sd = _model()
    b = _origin_batch(61, [9, 14, 6])
    n = len(b['batch_ligand'])
    if case == 'fragment':
        path = PATH
        mask = _mask(b, lead=4)
        ft = _fixed_tape(63, len(path), n)
        return model, sd, b, path, dict(fixed_mask=mask, fixed_tape=ft), dict(mask=mask, ft=ft)
    t0 = 400
    path = resampled_time_path(respaced_time_seq(1000, 12, start=t0), resamplings=2, jump_length=4)
    mask = _mask(b, lead=3)
    ft = _fixed_tape(64, len(path), n)
    st = (torch.randn(n, 3, generator=torch.Generator().manual_seed(65)), torch.rand(n, K13, generator=torch.Generator().manual_seed(66)))
    return (model, sd, b, path, dict(fixed_mask=mask, fixed_tape=ft, start_time=t0, start_tape=st),
            dict(mask=mask, ft=ft, start_time=t0, start_noise_tape=st))


@pytest.mark.parametrize('case', ['fragment', 'start_keep'])
def test_resampled_chain_vs_oracle(case):
    torch.set_num_threads(16)
    model, sd, b, path, ofx, efx = _chain_case(case)
    n, S = len(b['batch_ligand']), len(path)
    pn, vu = synth.make_tape(62, S, n)
    got = _sample(model, b, path=path, tape=(pn, vu), mode='none', **efx)
    want = resample.sample_diffusion(sd, None, *_args(b, 'cpu'), pn, vu, path, center_pos_mode='none', **ofx)
    first_bad = (got['v_traj'] != torch.stack(want['v_traj'])).any(1).nonzero()
    assert len(first_bad) == 0, 'atom types diverge from the oracle at step %d' % int(first_bad[0])
    torch.testing.assert_close(got['pos_traj'], torch.stack(want['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['v0_traj'], torch.stack(want['v0_traj']), rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(got['vt_traj'], torch.stack(want['vt_traj']), rtol=0, atol=LOGIT_ATOL)

    # every re-noising step from the engine's own state: bit for bit, fixed rows on the closed form at p
    tab = resample.path_tables(sd, path)
    mask = ofx['fixed_mask']
    x0 = b['init_ligand_pos']
    n_up, worst_fixed, vt_err = 0, 0.0, 0.0
    for s in range(1, S):
        t, p = int(tab['t'][s]), int(tab['p'][s])
        if p < t:
            continue
        n_up += 1
        xt, vt = got['pos_traj'][s - 1], got['v_traj'][s - 1]
        o = resample.renoise_step(sd, tab, s, xt, vt, pn[s], vu[s], K13)
        free = ~mask
        assert torch.equal(got['pos_traj'][s][free], o['pos'][free]), 're-noising step %d: positions differ' % s
        assert torch.equal(got['v_traj'][s][free], o['v'][free]), 're-noising step %d: types differ' % s
        vt_err = max(vt_err, float((got['vt_traj'][s] - o['vt']).abs().max()))
        # trajectory contents: v0 repeats the latest prediction, vt is a normalised distribution
        assert torch.equal(got['v0_traj'][s], got['v0_traj'][s - 1])
        assert float(torch.logsumexp(got['vt_traj'][s].double(), -1).abs().max()) < 1e-5
        # fixed rows: q(x_p | x0_f), q(v_p | v0_f) from fixed draw s + 1, the fp32 closed form
        fp, fv = fixed_atoms.forward_sample(sd, x0[mask], b['init_ligand_v'][mask], b['batch_ligand'][mask], p, ofx['fixed_tape'][0][s + 1][mask],
                                            ofx['fixed_tape'][1][s + 1][mask], K13)
        worst_fixed = max(worst_fixed, float(((got['pos_traj'][s][mask] - fp).abs() / (EPS32 * fp.abs().clamp(min=1.0))).max()))
        assert torch.equal(got['v_traj'][s][mask], fv), 're-noising step %d: fixed types differ' % s
    print('%s: %d steps (%d re-noising), max |pos - oracle| %.2e, re-noised vt %.2e, fixed rows %.2f ulp'
          % (case, S, n_up, float((got['pos_traj'] - torch.stack(want['pos_traj'])).abs().max()), vt_err, worst_fixed))
    assert n_up > 0 and vt_err <= 2e-6 and worst_fixed <= 4.0
    assert torch.equal(got['v'][mask], b['init_ligand_v'][mask])


# ------------------------------------------------------------------------------------------------ C. re-noising steps in float64
@pytest.mark.parametrize('pos_only', [False, True])
def test_every_renoise_step_vs_float64(pos_only):
    model, sd = _model()
    b = _origin_batch(41, [9, 14])
    path = [999, 900, 950, 500, 501, 100, 600, 2, 1, 0, 300, 0]
    S = len(path)
    pn, vu = synth.make_tape(41, S, len(b['batch_ligand']))
    r = _sample(model, b, path=path, tape=(pn, vu), mode='none', pos_only=pos_only)
    tab = resample.path_tables(sd, path)
    worst = {'pos': 0.0, 'vt': 0.0}
    exempt = 0
    for s in range(1, S):
        if tab['p'][s] < tab['t'][s]:
            continue
        xt, vt = r['pos_traj'][s - 1], r['v_traj'][s - 1]
        ref = resample.renoise_step(sd, tab, s, xt, vt, pn[s], vu[s], K13, pos_only=pos_only, dtype=torch.float64)
        e = float(((r['pos_traj'][s].double() - ref['pos']).abs() / ref['scale'].clamp(min=1e-30)).max())
        worst['pos'] = max(worst['pos'], e)
        if not pos_only:
            close = ref['margin'] <= stepwise.MARGIN
            exempt += int(close.sum())
            assert torch.equal(r['v_traj'][s][~close], ref['v'][~close]), s
            worst['vt'] = max(worst['vt'], float((r['vt_traj'][s].double() - ref['vt']).abs().max()))
        else:
            assert torch.equal(r['v_traj'][s], vt)
        print('s=%2d t=%4d p=%4d  pos %.2e  vt %.2e' % (s, tab['t'][s], tab['p'][s], e, worst['vt']))
    assert worst['pos'] <= stepwise.STEP_TOL['pos'] and worst['vt'] <= stepwise.STEP_TOL['vt'] and exempt <= stepwise.MAX_EXEMPT


# ------------------------------------------------------------------------------------------------ D. stream, graph, switches
def test_seeded_path_is_engine_tape():
    model, sd = _model()
    b = synth.make_batch(31, 4, n_protein=50, ligand_sizes=[60, 45, 33, 37])         # 175 atoms: two blocks of the kernels
    n, S = len(b['batch_ligand']), len(PATH)
    mask = _mask(b, lead=5)
    seed = 2 ** 32 + 7
    dev = _sample(model, b, path=PATH, mask=mask, seed=seed)
    pn, vu = philox.engine_tape(seed, n, S, K13)
    tape = _sample(model, b, path=PATH, mask=mask, ft=fixed_atoms.fixed_tape(seed, n, S, K13), tape=(pn, vu))
    assert torch.equal(dev['v_traj'], tape['v_traj'])
    sigma0 = float(np.exp(0.5 * float(resample.path_tables(sd, PATH)['logvar'][0])))
    ulps, later = philox.stream_errors(dev['pos_traj'][:, ~mask], tape['pos_traj'][:, ~mask], pn[0][~mask], sigma0)
    print('seeded path S=%d: %.2f ulp first step, %.2e later' % (S, ulps, later))
    assert ulps <= philox.STREAM_ULPS and later <= philox.STREAM_LATER_REL


@pytest.mark.parametrize('env', ['TDIFF_NO_GRAPH', 'TDIFF_NO_RESTRICT', 'TDIFF_KNN_FULL', 'TDIFF_NO_SLOT_KEEP', 'TDIFF_FREE_DEPTH'])
def test_switches_change_nothing(monkeypatch, env):
    """Graph replay equals eager steps, and the ligand-free cache, the incremental k-NN, the edge-gate slot keep and the backward cone
    stay exact when re-noising steps move the ligand between forwards."""
    b = synth.make_batch(33, 3, n_protein=120, ligand_sizes=[12, 20, 7])
    mask = _mask(b)
    model, _ = _model()
    base = _sample(model, b, path=PATH, mask=mask, seed=77)
    model._drop_engine()
    monkeypatch.setenv(env, '0' if env == 'TDIFF_FREE_DEPTH' else '1')
    other = _sample(model, b, path=PATH, mask=mask, seed=77)
    model._drop_engine()
    assert not _differing(base, other)


# ------------------------------------------------------------------------------------------------ E. driver and CLI
def test_1h36_driver_cpu_rng_vs_oracle():
    from targetdiff_b200 import atom_num
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand, seed_all
    torch.set_num_threads(16)
    model, sd = _model()
    data = pdb_to_pocket_data(PDB_1H36)
    path = resampled_time_path(respaced_time_seq(1000, 8), resamplings=2, jump_length=2)
    ctr = data.protein_pos.float().mean(0)
    frag = (ctr + torch.randn(3, 3, generator=torch.Generator().manual_seed(4)), torch.tensor([1, 3, 0]))
    seed_all(2021)
    got = sample_diffusion_ligand(model, data, 2, batch_size=2, device=DEV, sample_num_atoms='prior', rng='cpu', time_path=path,
                                  fixed_ligand=frag)
    seed_all(2021)
    want = resample.sample_diffusion_ligand(sd, None, data.protein_pos, data.protein_atom_feature, 2, atom_num._table(), path, batch_size=2,
                                            fixed_ligand=frag)
    assert [len(p) for p in got[0]] == [len(p) for p in want[0]]
    assert np.array_equal(np.concatenate(got[1]), np.concatenate(want[1]))
    assert np.array_equal(np.concatenate(got[3], axis=1), np.concatenate(want[3], axis=1))
    np.testing.assert_allclose(np.concatenate(got[2], axis=1), np.concatenate(want[2], axis=1), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(np.concatenate(got[0]), np.concatenate(want[0]), rtol=1e-4, atol=1e-4)
    assert got[2][0].shape[0] == len(path)


def test_cli_resamplings_with_fragment(tmp_path):
    import yaml
    from targetdiff_b200.cli import main
    from targetdiff_b200.config import Config, default_model_config
    cfg = dict(num_diffusion_timesteps=20)
    _, sd = _model(cfg)
    mc = default_model_config()
    mc.update(cfg)
    torch.save({'config': Config(model=mc, data={'transform': {'ligand_atom_mode': 'add_aromatic'}}), 'model': sd}, tmp_path / 'ckpt.pt')
    conf = {'model': {'checkpoint': str(tmp_path / 'ckpt.pt')},
            'sample': {'seed': 1, 'num_samples': 3, 'num_steps': 20, 'pos_only': False, 'center_pos_mode': 'protein',
                       'sample_num_atoms': 'range', 'respaced_steps': 6, 'resamplings': 2, 'jump_length': 2}}
    with open(tmp_path / 'sample.yml', 'w') as f:
        yaml.safe_dump(conf, f)
    from targetdiff_b200.pocket import pdb_to_pocket_data
    ctr = pdb_to_pocket_data(PDB_1H36).protein_pos.float().mean(0)
    frag = {'pos': ctr + torch.randn(2, 3, generator=torch.Generator().manual_seed(4)), 'v': torch.tensor([1, 3])}
    torch.save(frag, tmp_path / 'frag.pt')
    main(['sample_for_pocket', str(tmp_path / 'sample.yml'), '--pdb_path', PDB_1H36, '--result_path', str(tmp_path / 'out'),
          '--device', DEV, '--fragment', str(tmp_path / 'frag.pt')])
    r = torch.load(tmp_path / 'out' / 'sample.pt', weights_only=False)
    assert r['time_seq'] == [19, 15, 11, 8, 4, 0]
    assert r['time_path'] == [19, 15, 11, 19, 15, 11, 8, 4, 11, 8, 4, 0, 4, 0]
    for pos, v, ptraj, vtraj in zip(r['pred_ligand_pos'], r['pred_ligand_v'], r['pred_ligand_pos_traj'], r['pred_ligand_v_traj']):
        assert ptraj.shape == (14, len(pos), 3) and vtraj.shape == (14, len(pos))
        assert torch.allclose(torch.from_numpy(pos[:2]).float(), frag['pos'], rtol=EPS32, atol=0)
        assert v[:2].tolist() == [1, 3]


# ------------------------------------------------------------------------------------------------ F. refusals
def test_cabi_refusals():
    from targetdiff_b200 import _lib
    from targetdiff_b200.score_model import PATH_MAX_PER_T
    model, sd = _model(dict(num_diffusion_timesteps=20))
    T = sd['betas'].shape[0]
    lib = _lib.load()
    eng = model.engine(DEV)
    st = model._stream(torch.device(DEV))
    b = synth.make_batch(95, 2, n_protein=60, ligand_sizes=[8, 5])
    a = _args(b)
    model._bind(eng, a[0], a[1], a[2], a[5], 1)
    lpos, lv = a[3].float().contiguous(), a[4].long().contiguous()
    _lib.check(lib.tdiff_set_ligand(eng, ctypes.c_void_p(lpos.data_ptr()), ctypes.c_void_p(lv.data_ptr()), 1, st))

    def run(path, S=None, arr=True):
        S = len(path) if S is None else S
        return lib.tdiff_sample_path(eng, _lib.i32_array(path) if arr else None, S, None, None, ctypes.c_uint64(1), None, None, None, None, 0,
                                     st)

    too_long = [T - 1] + [T - 2, T - 1] * (PATH_MAX_PER_T * T // 2)
    cases = {'null pointer': ([T - 1], None, False), 'empty': ([T - 1], 0, True), 'not at T - 1': ([T - 2, 5, 0], None, True),
             'equal times': ([T - 1, 5, 5, 0], None, True), 'outside 0..T-1': ([T - 1, 3, T, 0], None, True),
             'more than': (too_long, None, True)}
    for msg, (path, S, arr) in cases.items():
        assert run(path, S, arr) == _lib.TDIFF_EINVAL, msg
        assert msg in lib.tdiff_last_error().decode(), (msg, lib.tdiff_last_error())
    assert run([T - 1, 3, -2]) == _lib.TDIFF_EINVAL and 'outside 0..T-1' in lib.tdiff_last_error().decode()
    _lib.check(lib.tdiff_set_start(eng, 5, None, None))            # an upward first step needs tau_0 below T - 1
    assert run([5, 7, 0]) == _lib.TDIFF_EINVAL and 'first step goes up' in lib.tdiff_last_error().decode()
    assert run([T - 1, 7, 0]) == _lib.TDIFF_EINVAL and 'start time' in lib.tdiff_last_error().decode()
    _lib.check(lib.tdiff_set_start(eng, -1, None, None))
    assert run([T - 1, 10, 15, 3, 0]) == _lib.TDIFF_OK                # the engine is still usable
    # tdiff_sample_seq keeps refusing a path that goes up
    assert lib.tdiff_sample_seq(eng, _lib.i32_array([T - 1, 3, 8, 0]), 4, None, None, ctypes.c_uint64(1), None, None, None, None, 0,
                                st) == _lib.TDIFF_EINVAL
    torch.cuda.synchronize()
