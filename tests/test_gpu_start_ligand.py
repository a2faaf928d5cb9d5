"""Start-ligand sampling (DESIGN.md section 1) on the engine (run with -m gpu; `pytest -s` prints the errors).

A. The seeded start draw is the host restatement of its Philox stream (oracle.start_ligand.start_tape): a seeded start chain equals the
   same chain on start_tape + philox.engine_tape (+ fixed_atoms.fixed_tape), with and without kept atoms and with pos_only.
B. Tape-driven start chains against the CPU oracle (oracle.start_ligand.sample_diffusion) at the tolerances of test_gpu_respaced.py.
C. Every step of a start chain against float64 (respaced.jump_step), the first one on the host's start state; from t0 = 0 the
   chain is one decoder step and ends on the network's x0.
D. Launches: the default chain's per step plus one init launch per chain; graph replay equals TDIFF_NO_GRAPH=1.
E. The rng='cpu' driver on the 1h36 pocket against the oracle's driver, with the reference's first 1h36 molecule as start ligand.
F. The CLI with --start_ligand, sample.respaced_steps and 'keep'.
G. Refusals through the C-ABI."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import fixed_atoms, philox, respaced, restate, start_ligand, stepwise, synth
from targetdiff_b200.sampling import respaced_time_seq

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K13 = synth.LIGAND_NUM_CLASSES
EPS32 = 2.0 ** -23
POS_RTOL, POS_ATOL, LOGIT_ATOL = 1e-4, 1e-5, 1e-3
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
PDB_1H36 = os.path.join(GOLDEN, '1h36_pocket10.pdb')
JUMPS = [600, 450, 200, 37, 36, 2, 0]


def _model(cfg=None, weight_seed=0, K=K13):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K)
    sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg), ligand_dim=K)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ARGS)


def _mask(b, lead=3):
    """The first `lead` atoms of every graph (leaving at least one free atom)."""
    m = torch.zeros(len(b['batch_ligand']), dtype=torch.bool)
    start = 0
    for n in torch.bincount(b['batch_ligand']).tolist():
        m[start:start + min(lead, n - 1)] = True
        start += n
    return m


def _sample(model, b, t0, time_seq=None, mask=None, ft=None, tape=None, st=None, mode='protein', **kw):
    r = model.sample_diffusion(*_args(b), time_seq=time_seq, center_pos_mode=mode, noise_tape=tape, stack_traj=True, start_time=t0,
                               start_noise_tape=st, fixed_mask=None if mask is None else mask.to(DEV), fixed_noise_tape=ft, **kw)
    return {k: (r[k].cpu() if torch.is_tensor(r[k]) else r[k]) for k in TRAJ}


def _differing(a, c):
    return [k for k in TRAJ if not (a[k] is None and c[k] is None) and not torch.equal(a[k], c[k])]


# ------------------------------------------------------------------------------------------------ A. the seeded start stream
@pytest.mark.parametrize('t0,seq,kept,pos_only', [(0, None, False, False), (1, None, True, False), (500, [500, 300, 40, 0], False, False),
                                                  (500, [500, 499, 100, 0], True, False), (999, [999, 600, 0], True, False),
                                                  (999, [999, 600, 0], False, True), (1, None, True, True)])
def test_seeded_start_draw_is_the_host_stream(t0, seq, kept, pos_only):
    model, _ = _model()
    b = synth.make_batch(31, 4, n_protein=50, ligand_sizes=[60, 45, 33, 37])         # 175 atoms: two blocks of the init launch
    n = len(b['batch_ligand'])
    S = t0 + 1 if seq is None else len(seq)
    seed = 2 ** 32 + 19 + t0
    mask = _mask(b, lead=5) if kept else None
    dev = _sample(model, b, t0, seq, mask, seed=seed, pos_only=pos_only)
    tape = philox.engine_tape(seed, n, S, K13, pos_only=pos_only)
    st = start_ligand.start_tape(seed, n, K13, pos_only=pos_only)
    ft = fixed_atoms.fixed_tape(seed, n, S, K13, pos_only=pos_only) if kept else None
    host = _sample(model, b, t0, seq, mask, ft, tape, st, pos_only=pos_only)
    assert torch.equal(dev['v_traj'], host['v_traj'])
    err = float((dev['pos_traj'] - host['pos_traj']).abs().max())
    print('seeded start chain t0=%d S=%d kept=%s pos_only=%s: max |seeded - host stream| %.2e' % (t0, S, kept, pos_only, err))
    torch.testing.assert_close(dev['pos_traj'], host['pos_traj'], rtol=POS_RTOL, atol=POS_ATOL)


# ------------------------------------------------------------------------------------------------ B. against the oracle
PARITY_CASES = {
    'unit_t30': ({}, 30, None, [9, 14, 5], False, False),
    'jumps_t600': ({}, 600, JUMPS, [9, 14, 5], False, False),
    'respaced_t500': ({}, 500, respaced_time_seq(1000, 12, start=500), [9, 6], False, False),
    'kept_jumps': ({}, 600, JUMPS, [9, 14, 5], True, False),
    'kept_unit_t20': ({}, 20, None, [9, 6], True, False),
    'time_emb_simple': (dict(time_emb_dim=1, time_emb_mode='simple'), 600, JUMPS, [9, 6], False, False),
    'noise_mean': (dict(model_mean_type='noise'), 600, JUMPS, [9, 6], False, False),
    'pos_only_kept': ({}, 600, JUMPS, [9, 6], True, True),
    'end_above_0': ({}, 700, [700, 300, 120], [9, 6], False, False),
}


@pytest.mark.parametrize('name', list(PARITY_CASES))
def test_start_chain_vs_oracle(name):
    torch.set_num_threads(16)
    cfg, t0, seq, sizes, kept, pos_only = PARITY_CASES[name]
    model, sd = _model(cfg)
    b = synth.make_batch(61, len(sizes), n_protein=40, ligand_sizes=sizes)
    n = len(b['batch_ligand'])
    S = t0 + 1 if seq is None else len(seq)
    pn, vu = synth.make_tape(62, S, n)
    g = torch.Generator().manual_seed(63)
    st = (torch.randn(n, 3, generator=g), torch.rand(n, K13, generator=g))
    fx = dict(fixed_mask=_mask(b), fixed_tape=(torch.randn(S + 1, n, 3, generator=g), torch.rand(S + 1, n, K13, generator=g))) if kept else {}
    want = start_ligand.sample_diffusion(sd, cfg, *_args(b, 'cpu'), pn, vu, t0, st, seq, pos_only=pos_only, **fx)
    got = _sample(model, b, t0, seq, fx.get('fixed_mask'), fx.get('fixed_tape'), (pn, vu), st, pos_only=pos_only)
    first_bad = (got['v_traj'] != torch.stack(want['v_traj'])).any(1).nonzero()
    assert len(first_bad) == 0, 'atom types diverge from the oracle at step %d' % int(first_bad[0])
    torch.testing.assert_close(got['pos_traj'], torch.stack(want['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['pos'], want['pos'], rtol=POS_RTOL, atol=POS_ATOL)
    if not pos_only:
        torch.testing.assert_close(got['v0_traj'], torch.stack(want['v0_traj']), rtol=0, atol=LOGIT_ATOL)
        torch.testing.assert_close(got['vt_traj'], torch.stack(want['vt_traj']), rtol=0, atol=LOGIT_ATOL)
    print('%s: %d steps, max |pos - oracle| %.2e' % (name, S, float((got['pos_traj'] - torch.stack(want['pos_traj'])).abs().max())))


# ------------------------------------------------------------------------------------------------ C. every step in float64
@pytest.mark.parametrize('label,cfg,t0,seq,pos_only', [('jumps', {}, 600, JUMPS, False), ('unit_t5', {}, 5, None, False),
                                                       ('noise_mean', dict(model_mean_type='noise'), 600, JUMPS, False),
                                                       ('pos_only', {}, 300, [300, 100, 1], True), ('decoder_t0', {}, 0, None, False)])
def test_every_start_step_vs_float64(label, cfg, t0, seq, pos_only):
    """Each step against respaced.jump_step in float64 on the engine's input state and network outputs; step 0's input is the host's
    start state (oracle.start_ligand.start_state on the same start tape)."""
    model, sd = _model(cfg)
    b = synth.make_batch(41, 2, n_protein=40, ligand_sizes=[9, 14], distinct_pockets=1)
    shift = b['protein_pos'].mean(0, keepdim=True)
    b['protein_pos'], b['init_ligand_pos'] = b['protein_pos'] - shift, b['init_ligand_pos'] - shift
    seq = list(range(t0, -1, -1)) if seq is None else seq
    S, n = len(seq), len(b['batch_ligand'])
    pn, vu = synth.make_tape(41, S, n)
    st = start_ligand.start_tape(42, n, K13, pos_only=pos_only)
    tab = respaced.jump_tables(sd, seq)
    r = _sample(model, b, t0, seq, tape=(pn, vu), st=st, mode='none', pos_only=pos_only)
    xs, vs = start_ligand.start_state(sd, b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'], t0, st, K13, pos_only)
    B = int(b['batch_protein'].max()) + 1
    time_emb = cfg.get('time_emb_dim', 0) > 0
    rows = []
    for s in range(S):
        t = int(tab['t'][s])
        xt = xs if s == 0 else r['pos_traj'][s - 1]
        vt = vs if s == 0 else r['v_traj'][s - 1]
        kw = {'time_step': torch.full((B,), t, dtype=torch.long, device=DEV)} if time_emb else {}
        a = _args(b)
        out = model(a[0], a[1], a[2], xt.to(DEV), vt.to(DEV), a[5], **kw)
        x0, logits = out['pred_ligand_pos'].cpu(), out['pred_ligand_v'].cpu()
        step_args = (sd, cfg, tab, s, xt, vt, x0, logits, pn[s], vu[s])
        ref = respaced.jump_step(*step_args, pos_only=pos_only, dtype=torch.float64)
        f32 = respaced.jump_step(*step_args, pos_only=pos_only)
        e = stepwise.errors(r['pos_traj'][s], r['v_traj'][s], None if pos_only else r['v0_traj'][s], None if pos_only else r['vt_traj'][s],
                            ref, stepwise.MARGIN)
        o = stepwise.errors(f32['pos'], f32['v'], f32['v0'], f32['vt'], ref, stepwise.MARGIN)
        rows.append((s, t, e, o))
        print('%-12s s=%3d t=%4d p=%4d  pos %.2e  v0 %.2e  vt %.2e  exempt %d   fp32 oracle: pos %.2e  v0 %.2e  vt %.2e' %
              (label, s, t, int(tab['p'][s]), e['pos'], e['v0'], e['vt'], e['exempt'], o['pos'], o['v0'], o['vt']))
        if t == 0 and cfg.get('model_mean_type', 'C0') == 'C0':      # the decoder step: sigma = 0, c0 = 1, ct = 0 -- the state becomes the network's x0
            d = float(((r['pos_traj'][s].double() - x0.double()).abs() / (EPS32 * x0.double().abs().clamp(min=1e-3))).max())
            print('%-12s decoder step: %.2f ulp of the network x0' % (label, d))
            assert d <= 4.0
    stepwise.check_steps(label, rows)


# ------------------------------------------------------------------------------------------------ D. launches, graph replay
def test_launches_are_the_default_chains_plus_one():
    from targetdiff_b200 import _lib
    lib = _lib.load()
    b = synth.make_batch(6, 2, n_protein=150, ligand_sizes=[20, 7])
    counts = {}
    for arm in ('respaced', 'start', 'fixed', 'start_fixed'):
        for seq in ([999, 500, 0], [999, 998, 500, 20, 0]):
            model, _ = _model(weight_seed=3)
            kw = dict(time_seq=seq, center_pos_mode='protein', return_traj=False)
            if arm.startswith('start'):                                          # the same number of steps from t0 = tau_0 - 100
                kw.update(start_time=seq[0] - 100, time_seq=[seq[0] - 100, seq[1] - 100] + seq[2:])
            if arm.endswith('fixed'):
                kw.update(fixed_mask=_mask(b).to(DEV))
            model.sample_diffusion(*_args(b), **kw)
            counts[arm, len(seq)] = lib.tdiff_launch_count(model.engine(DEV))
            model._drop_engine()
    print('launches: %s' % counts)
    for S in (3, 5):
        assert counts['start', S] == counts['respaced', S] + 1
        assert counts['start_fixed', S] == counts['fixed', S]                  # the start launch replaces the fixed set's
    assert counts['start', 5] - counts['start', 3] == counts['respaced', 5] - counts['respaced', 3]


def test_graph_replay_is_eager(monkeypatch):
    b = synth.make_batch(33, 3, n_protein=60, ligand_sizes=[12, 20, 7])
    seq = respaced_time_seq(1000, 10, start=400)
    mask = _mask(b)
    model, _ = _model()
    graph = _sample(model, b, 400, seq, mask, seed=77)
    model._drop_engine()
    monkeypatch.setenv('TDIFF_NO_GRAPH', '1')
    eager = _sample(model, b, 400, seq, mask, seed=77)
    model._drop_engine()
    assert not _differing(graph, eager)


def test_chain_without_start_is_unchanged_after_one():
    """An engine that ran a start chain runs the default chain bit for bit as a fresh one (bind clears the start)."""
    b = synth.make_batch(34, 2, n_protein=50, ligand_sizes=[10, 8])
    model, _ = _model()
    fresh = _sample(model, b, None, None, seed=5, num_steps=6)
    _sample(model, b, 300, [300, 10, 0], seed=5)
    again = _sample(model, b, None, None, seed=5, num_steps=6)
    assert not _differing(fresh, again)


# ------------------------------------------------------------------------------------------------ E. driver, F. CLI
def _1h36_ligand():
    z = np.load(os.path.join(GOLDEN, 'pocket_1h36_full.npz'))
    n = int(z['sizes'][0])
    return torch.from_numpy(z['pos'][:n]).float(), torch.from_numpy(z['v'][:n]).long()


@pytest.mark.parametrize('t0,n_steps,keep,pos_only', [(300, 10, None, False), (12, None, [0, 3, 5], False), (200, 6, [1, 2], True)])
def test_1h36_driver_cpu_rng_vs_oracle(t0, n_steps, keep, pos_only):
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand, seed_all
    torch.set_num_threads(16)
    model, sd = _model()
    data = pdb_to_pocket_data(PDB_1H36)
    lig = _1h36_ligand()
    seq = None if n_steps is None else respaced_time_seq(1000, n_steps, start=t0)
    seed_all(2021)
    got = sample_diffusion_ligand(model, data, 3, batch_size=2, device=DEV, rng='cpu', time_seq=seq, start_ligand=lig, start_time=t0,
                                  keep_atoms=keep, pos_only=pos_only)
    seed_all(2021)
    want = start_ligand.sample_diffusion_ligand(sd, None, data.protein_pos, data.protein_atom_feature, 3, lig, t0, seq, keep_atoms=keep,
                                                batch_size=2, pos_only=pos_only)
    assert [len(p) for p in got[0]] == [len(lig[1])] * 3 == [len(p) for p in want[0]]
    assert np.array_equal(np.concatenate(got[1]), np.concatenate(want[1]))
    assert np.array_equal(np.concatenate(got[3], axis=1), np.concatenate(want[3], axis=1))
    np.testing.assert_allclose(np.concatenate(got[2], axis=1), np.concatenate(want[2], axis=1), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(np.concatenate(got[0]), np.concatenate(want[0]), rtol=1e-4, atol=1e-4)
    assert got[2][0].shape[0] == (t0 + 1 if seq is None else len(seq))
    if pos_only:
        assert all(np.array_equal(v, lig[1].numpy()) for v in got[1])
    if keep is not None and not pos_only:
        for pos, v in zip(got[0], got[1]):
            assert np.array_equal(v[keep], lig[1].numpy()[keep])
            np.testing.assert_allclose(pos[keep], lig[0].numpy()[keep], rtol=2 * EPS32, atol=0)


def test_cli_start_ligand_with_respaced_steps_and_keep(tmp_path):
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
                       'sample_num_atoms': 'prior', 'respaced_steps': 5, 'start_time': 12}}
    with open(tmp_path / 'sample.yml', 'w') as f:
        yaml.safe_dump(conf, f)
    pos, v = _1h36_ligand()
    np.savez(tmp_path / 'start.npz', pos=pos.numpy(), v=v.numpy(), keep=np.array([0, 2]))
    main(['sample_for_pocket', str(tmp_path / 'sample.yml'), '--pdb_path', PDB_1H36, '--result_path', str(tmp_path / 'out'),
          '--device', DEV, '--start_ligand', str(tmp_path / 'start.npz')])
    r = torch.load(tmp_path / 'out' / 'sample.pt', weights_only=False)
    assert r['time_seq'] == respaced_time_seq(20, 5, start=12) == [12, 9, 6, 3, 0]
    assert r['start_time'] == 12 and r['kept_atoms'] == [0, 2]
    assert torch.equal(r['start_ligand'][0], pos) and torch.equal(r['start_ligand'][1], v)
    assert len(r['pred_ligand_pos']) == 3
    for p, vv, ptraj, vtraj in zip(r['pred_ligand_pos'], r['pred_ligand_v'], r['pred_ligand_pos_traj'], r['pred_ligand_v_traj']):
        assert p.shape == (len(v), 3) and ptraj.shape == (5, len(v), 3) and vtraj.shape == (5, len(v))
        assert vv[[0, 2]].tolist() == v[[0, 2]].tolist()
        assert torch.allclose(torch.from_numpy(p[[0, 2]]).float(), pos[[0, 2]], rtol=2 * EPS32, atol=0)
    conf['sample'].pop('start_time')
    with open(tmp_path / 'bad.yml', 'w') as f:
        yaml.safe_dump(conf, f)
    with pytest.raises(ValueError, match='start_time'):
        main(['sample_for_pocket', str(tmp_path / 'bad.yml'), '--pdb_path', PDB_1H36, '--result_path', str(tmp_path / 'bad'),
              '--device', DEV, '--start_ligand', str(tmp_path / 'start.npz')])


# ------------------------------------------------------------------------------------------------ G. refusals
def test_cabi_refusals():
    from targetdiff_b200 import _lib
    model, sd = _model()
    T = sd['betas'].shape[0]
    lib = _lib.load()
    eng = model.engine(DEV)
    st = model._stream(torch.device(DEV))
    b = synth.make_batch(95, 2, n_protein=60, ligand_sizes=[8, 5])
    a = _args(b)
    n = len(b['batch_ligand'])
    vp = lambda t: ctypes.c_void_p(t.data_ptr())                                    # noqa: E731
    tape = [torch.zeros(4, n, 3, device=DEV), torch.zeros(4, n, K13, device=DEV)]
    stape = [torch.zeros(n, 3, device=DEV), torch.zeros(n, K13, device=DEV)]
    assert lib.tdiff_set_start(None, 5, None, None) == _lib.TDIFF_ESTATE
    model._bind(eng, a[0], a[1], a[2], a[5], 1)
    lpos, lv = a[3].float().contiguous(), a[4].long().contiguous()
    _lib.check(lib.tdiff_set_ligand(eng, vp(lpos), vp(lv), 1, st))

    def seq_run(seq, pn=None, vu=None):
        return lib.tdiff_sample_seq(eng, _lib.i32_array(seq), len(seq), pn, vu, ctypes.c_uint64(1), None, None, None, None, 0, st)

    for t in (-2, T, T + 5):
        assert lib.tdiff_set_start(eng, t, None, None) == _lib.TDIFF_EINVAL and b'outside -1..' in lib.tdiff_last_error()
    _lib.check(lib.tdiff_set_start(eng, 300, None, None))
    assert seq_run([T - 1, 100, 0]) == _lib.TDIFF_EINVAL and b'not at the start time t_start = 300' in lib.tdiff_last_error()
    rc = lib.tdiff_sample(eng, 3, None, None, ctypes.c_uint64(1), None, None, None, None, 0, st)
    assert rc == _lib.TDIFF_EINVAL and b'tdiff_sample_seq' in lib.tdiff_last_error()
    # mixed tape sources: a step tape without a start tape, and a start tape without a step tape
    assert seq_run([300, 100, 20, 0], vp(tape[0]), vp(tape[1])) == _lib.TDIFF_EINVAL and b'needs a start tape' in lib.tdiff_last_error()
    _lib.check(lib.tdiff_set_start(eng, 300, vp(stape[0]), vp(stape[1])))
    assert seq_run([300, 100, 20, 0]) == _lib.TDIFF_EINVAL and b'start tape is set' in lib.tdiff_last_error()
    _lib.check(lib.tdiff_set_start(eng, 300, vp(stape[0]), None))
    assert seq_run([300, 100, 20, 0], vp(tape[0]), vp(tape[1])) == _lib.TDIFF_EINVAL and b'needs v_uniform' in lib.tdiff_last_error()
    _lib.check(lib.tdiff_set_start(eng, 300, vp(stape[0]), vp(stape[1])))
    assert seq_run([300, 100, 20, 0], vp(tape[0]), vp(tape[1])) == _lib.TDIFF_OK
    _lib.check(lib.tdiff_set_start(eng, -1, None, None))                             # clearing: the default rules again
    assert seq_run([300, 0]) == _lib.TDIFF_EINVAL and b'not at T - 1' in lib.tdiff_last_error()
    _lib.check(lib.tdiff_set_start(eng, 300, None, None))
    model._bind(eng, a[0], a[1], a[2], a[5], 1)                                      # bind clears the start
    _lib.check(lib.tdiff_set_ligand(eng, vp(lpos), vp(lv), 1, st))
    assert lib.tdiff_sample(eng, 3, None, None, ctypes.c_uint64(1), None, None, None, None, 0, st) == _lib.TDIFF_OK
    assert seq_run([300, 0]) == _lib.TDIFF_EINVAL
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match='start_noise_tape'):
        model.sample_diffusion(*a, start_time=10, noise_tape=synth.make_tape(1, 11, n))
    with pytest.raises(ValueError, match='start_time'):
        model.sample_diffusion(*a, start_noise_tape=(stape[0], stape[1]))
