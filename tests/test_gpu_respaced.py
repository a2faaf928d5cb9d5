"""Respaced sampling (DESIGN.md section 1) on the engine (run with -m gpu; `pytest -s` prints the errors).

A. Default path unchanged: tdiff_sample_seq on T-1..0 and T-1..T-S is tdiff_sample(T) / tdiff_sample(S) bit for bit, on a tape and
   seeded, with and without a fixed set, with pos_only and a time embedding; the same launches per step.
B. Against the CPU oracle (oracle.respaced.sample_diffusion) on noise tapes, with the chain tolerances of the other GPU tests.
C. Every jump step against float64 (oracle.respaced.jump_step) within stepwise.STEP_TOL.
D. A seeded respaced chain equals the same chain on philox.engine_tape (+ fixed_atoms.fixed_tape); graph replay equals
   TDIFF_NO_GRAPH=1 bit for bit.
E. Fixed rows follow the fp32 closed form of q(x_p | x0_f) and end exactly on x0_f / v0_f.
F. The rng='cpu' driver against oracle.respaced's restatement on the 1h36 pocket; the CLI with sample.respaced_steps.
G. Refusals through the C-ABI."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import fixed_atoms, philox, respaced, restate, stepwise, synth
from targetdiff_b200.sampling import respaced_time_seq

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K13 = synth.LIGAND_NUM_CLASSES
EPS32 = 2.0 ** -23
POS_RTOL, POS_ATOL, LOGIT_ATOL = 1e-4, 1e-5, 1e-3
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')
IRREGULAR = [999, 998, 600, 37, 36, 2, 0]
PDB_1H36 = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', '1h36_pocket10.pdb')


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
    bl = b['batch_ligand']
    m = torch.zeros(len(bl), dtype=torch.bool)
    start = 0
    for n in torch.bincount(bl).tolist():
        m[start:start + min(lead, n - 1)] = True
        start += n
    return m


def _fixed_tape(seed, S, n, K=K13):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(S + 1, n, 3, generator=g), torch.rand(S + 1, n, K, generator=g)


def _sample(model, b, S=None, time_seq=None, mask=None, ft=None, tape=None, mode='protein', **kw):
    r = model.sample_diffusion(*_args(b), num_steps=S, time_seq=time_seq, center_pos_mode=mode, noise_tape=tape, stack_traj=True,
                               fixed_mask=None if mask is None else mask.to(DEV), fixed_noise_tape=ft, **kw)
    return {k: (r[k].cpu() if torch.is_tensor(r[k]) else r[k]) for k in TRAJ}


def _differing(a, c):
    return [k for k in TRAJ if not (a[k] is None and c[k] is None) and not torch.equal(a[k], c[k])]


# ------------------------------------------------------------------------------------------------ A. default path unchanged
@pytest.mark.parametrize('noise,fixed,pos_only,full', [('tape', False, False, True), ('seed', True, False, True),
                                                       ('tape', True, False, False), ('seed', False, False, False),
                                                       ('tape', False, True, False), ('seed', True, True, False)])
def test_unit_sequences_are_the_default_chain(noise, fixed, pos_only, full):
    """T-1..0 is tdiff_sample(T) and T-1..T-7 is tdiff_sample(7), bit for bit."""
    model, sd = _model()
    T = sd['betas'].shape[0]
    b = synth.make_batch(11, 3, n_protein=50, ligand_sizes=[9, 14, 5])
    n = len(b['batch_ligand'])
    S = T if full else 7
    kw = dict(tape=synth.make_tape(12, S, n)) if noise == 'tape' else dict(seed=2 ** 40 + 3)
    if fixed:
        kw.update(mask=_mask(b), ft=_fixed_tape(13, S, n) if noise == 'tape' else None)
    plain = _sample(model, b, S, pos_only=pos_only, **kw)
    seq = _sample(model, b, None, list(range(T - 1, T - 1 - S, -1)), pos_only=pos_only, **kw)
    assert not _differing(plain, seq)


def test_unit_sequence_with_time_embedding():
    cfg = dict(num_diffusion_timesteps=20, time_emb_dim=1, time_emb_mode='simple')
    model, _ = _model(cfg)
    b = synth.make_batch(14, 2, n_protein=40, ligand_sizes=[9, 6])
    tape = synth.make_tape(15, 20, len(b['batch_ligand']))
    assert not _differing(_sample(model, b, 20, tape=tape), _sample(model, b, None, list(range(19, -1, -1)), tape=tape))


def test_launches_per_step_are_the_default_chains():
    """On test_default_form_launches_per_step's batch, a respaced chain issues what the default chain of the same length does."""
    from targetdiff_b200 import _lib
    lib = _lib.load()
    b = synth.make_batch(6, 2, n_protein=150, ligand_sizes=[20, 7])
    counts = {}
    for respace in (False, True):
        for S in (3, 5):
            model, _ = _model(weight_seed=3)
            seq = {3: [999, 500, 0], 5: [999, 998, 500, 20, 0]}[S] if respace else None
            model.sample_diffusion(*_args(b), num_steps=None if respace else S, time_seq=seq, center_pos_mode='protein', return_traj=False)
            counts[respace, S] = lib.tdiff_launch_count(model.engine(DEV))
            model._drop_engine()
    print('launches: default chain %s, respaced %s' % ((counts[False, 3], counts[False, 5]), (counts[True, 3], counts[True, 5])))
    assert counts[True, 3] == counts[False, 3] and counts[True, 5] == counts[False, 5]


# ------------------------------------------------------------------------------------------------ B. against the oracle
PARITY_CASES = {
    'stride10': ({}, respaced_time_seq(1000, 100), [7, 11], 40, False, K13, False),
    'stride50': ({}, respaced_time_seq(1000, 20), [7, 11], 40, False, K13, False),
    'irregular': ({}, IRREGULAR, [9, 14, 5], 40, False, K13, False),
    'ends_above_0': ({}, [999, 700, 400, 120], [9, 6], 40, False, K13, False),
    'noise_mean': (dict(model_mean_type='noise'), IRREGULAR, [9, 6], 40, False, K13, False),
    'pos_only': ({}, IRREGULAR, [9, 6], 40, True, K13, False),
    'time_emb_simple': (dict(time_emb_dim=1, time_emb_mode='simple'), IRREGULAR, [9, 6], 40, False, K13, False),
    'hybrid': (dict(cutoff_mode='hybrid'), IRREGULAR, [9, 6], 40, False, K13, False),
    'num_blocks_2': (dict(num_blocks=2), IRREGULAR, [9, 6], 40, False, K13, False),
    'k48': (dict(knn=48), IRREGULAR, [9, 6], 60, False, K13, False),
    'K8': ({}, IRREGULAR, [9, 6], 40, False, 8, False),
    'K23': ({}, respaced_time_seq(1000, 20), [9, 6], 40, False, 23, False),
    'ragged': ({}, [999, 900, 899, 450, 10, 0], [1, 14, 3, 6], (35, 50, 42, 61), False, K13, False),
    'fixed_atoms': ({}, respaced_time_seq(1000, 20), [9, 14, 5], 40, False, K13, True),
}


@pytest.mark.parametrize('name', list(PARITY_CASES))
def test_respaced_chain_vs_oracle(name):
    torch.set_num_threads(16)
    cfg, seq, sizes, n_protein, pos_only, K, fixed = PARITY_CASES[name]
    model, sd = _model(cfg, K=K)
    if isinstance(n_protein, tuple):
        b = synth.make_ragged_batch(61, list(n_protein), sizes, num_classes=K)
    else:
        b = synth.make_batch(61, len(sizes), n_protein=n_protein, ligand_sizes=sizes, num_classes=K)
    n, S = len(b['batch_ligand']), len(seq)
    pn, vu = synth.make_tape(62, S, n, num_classes=K)
    fx = dict(fixed_mask=_mask(b), fixed_tape=_fixed_tape(63, S, n, K)) if fixed else {}
    want = respaced.sample_diffusion(sd, cfg, *_args(b, 'cpu'), pn, vu, seq, pos_only=pos_only, **fx)
    got = _sample(model, b, None, seq, fx.get('fixed_mask'), fx.get('fixed_tape'), (pn, vu), pos_only=pos_only)
    first_bad = (got['v_traj'] != torch.stack(want['v_traj'])).any(1).nonzero()
    assert len(first_bad) == 0, 'atom types diverge from the oracle at step %d' % int(first_bad[0])
    torch.testing.assert_close(got['pos_traj'], torch.stack(want['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['pos'], want['pos'], rtol=POS_RTOL, atol=POS_ATOL)
    if not pos_only:
        torch.testing.assert_close(got['v0_traj'], torch.stack(want['v0_traj']), rtol=0, atol=LOGIT_ATOL)
        torch.testing.assert_close(got['vt_traj'], torch.stack(want['vt_traj']), rtol=0, atol=LOGIT_ATOL)
    print('%s: %d steps, max |pos - oracle| %.2e' % (name, S, float((got['pos_traj'] - torch.stack(want['pos_traj'])).abs().max())))


# ------------------------------------------------------------------------------------------------ C. every jump step in float64
@pytest.mark.parametrize('label,cfg,seq,pos_only', [('irregular', {}, IRREGULAR, False), ('stride50', {}, respaced_time_seq(1000, 20), False),
                                                    ('noise_mean', dict(model_mean_type='noise'), IRREGULAR, False),
                                                    ('pos_only', {}, [999, 600, 100, 1], True)])
def test_every_jump_step_vs_float64(label, cfg, seq, pos_only):
    """Each step of the engine's respaced chain against respaced.jump_step in float64 on the same input state and network outputs."""
    model, sd = _model(cfg)
    b = synth.make_batch(41, 2, n_protein=40, ligand_sizes=[9, 14], distinct_pockets=1)
    shift = b['protein_pos'].mean(0, keepdim=True)
    b['protein_pos'], b['init_ligand_pos'] = b['protein_pos'] - shift, b['init_ligand_pos'] - shift
    S = len(seq)
    pn, vu = synth.make_tape(41, S, len(b['batch_ligand']))
    tab = respaced.jump_tables(sd, seq)
    r = _sample(model, b, None, seq, tape=(pn, vu), mode='none', pos_only=pos_only)
    B = int(b['batch_protein'].max()) + 1
    time_emb = cfg.get('time_emb_dim', 0) > 0
    rows = []
    for s in range(S):
        t = int(tab['t'][s])
        xt = b['init_ligand_pos'] if s == 0 else r['pos_traj'][s - 1]
        vt = b['init_ligand_v'] if s == 0 else r['v_traj'][s - 1]
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
    stepwise.check_steps(label, rows)


# ------------------------------------------------------------------------------------------------ D. seeded stream, graph replay
@pytest.mark.parametrize('seed,seq,fixed', [(123, [999, 600, 37, 2, 0], False), (2 ** 32 + 7, respaced_time_seq(1000, 20), True)])
def test_seeded_respaced_chain_is_engine_tape(seed, seq, fixed):
    model, sd = _model()
    b = synth.make_batch(31, 4, n_protein=50, ligand_sizes=[60, 45, 33, 37])         # 175 atoms: two blocks of the epilogue
    n, S = len(b['batch_ligand']), len(seq)
    mask = _mask(b, lead=5) if fixed else None
    dev = _sample(model, b, None, seq, mask, seed=seed)
    pn, vu = philox.engine_tape(seed, n, S, K13)
    ft = fixed_atoms.fixed_tape(seed, n, S, K13) if fixed else None
    tape = _sample(model, b, None, seq, mask, ft, (pn, vu))
    assert torch.equal(dev['v_traj'], tape['v_traj'])
    free = ~mask if fixed else torch.ones(n, dtype=torch.bool)
    sigma0 = math.exp(0.5 * float(respaced.jump_tables(sd, seq)['logvar'][0]))
    ulps, later = philox.stream_errors(dev['pos_traj'][:, free], tape['pos_traj'][:, free], pn[0][free], sigma0)
    print('seeded respaced chain seed=%d S=%d: %.2f ulp first step, %.2e later' % (seed, S, ulps, later))
    assert ulps <= philox.STREAM_ULPS and later <= philox.STREAM_LATER_REL


def test_graph_replay_is_eager(monkeypatch):
    b = synth.make_batch(33, 3, n_protein=60, ligand_sizes=[12, 20, 7])
    seq = respaced_time_seq(1000, 10)
    mask = _mask(b)
    model, _ = _model()
    graph = _sample(model, b, None, seq, mask, seed=77)
    model._drop_engine()
    monkeypatch.setenv('TDIFF_NO_GRAPH', '1')
    eager = _sample(model, b, None, seq, mask, seed=77)
    model._drop_engine()
    assert not _differing(graph, eager)


# ------------------------------------------------------------------------------------------------ E. fixed rows
def test_fixed_rows_follow_the_closed_form_at_p():
    model, sd = _model()
    b = synth.make_batch(71, 3, n_protein=50, ligand_sizes=[10, 21, 8])
    n = len(b['batch_ligand'])
    seq = respaced_time_seq(1000, 100)
    S = len(seq)
    pn, vu = synth.make_tape(72, S, n)
    ft = _fixed_tape(73, S, n)
    mask = _mask(b, lead=4)
    got = _sample(model, b, None, seq, mask, ft, (pn, vu))
    _, x0c, off = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    x0c, off, v0 = x0c[mask], off[b['batch_ligand'][mask]], b['init_ligand_v'][mask]
    worst, exempt, flips = 0.0, 0, 0
    for s, (t, p) in enumerate(respaced.targets(seq)[:-1]):
        eps, u = ft[0][s + 1][mask], ft[1][s + 1][mask]
        ac = sd['alphas_cumprod'][p]
        x = ac.sqrt() * x0c + (1.0 - ac).sqrt() * eps + off                                 # fp32, as the kernel
        scale = x.double().abs() + off.double().abs() + eps.double().abs()
        worst = max(worst, float(((got['pos_traj'][s][mask].double() - x.double()).abs() / (EPS32 * scale)).max()))
        lq = restate.q_v_pred(sd, restate.index_to_log_onehot(v0, K13).double(), torch.full((3,), p), b['batch_ligand'][mask], K13)
        sc = -torch.log(-torch.log(u.double() + 1e-30) + 1e-30) + lq
        top = sc.topk(2, dim=1).values
        ok = (top[:, 0] - top[:, 1]) > 1e-4
        exempt += int((~ok).sum())
        flips += int((got['v_traj'][s][mask][ok] != sc.argmax(1)[ok]).sum())
    final = got['pos'][mask].double()
    x0f = b['init_ligand_pos'][mask].double()
    final_ulps = float(((final - x0f).abs() / (EPS32 * x0f.abs())).max())
    print('fixed rows over %d respaced steps: %.2f ulp of the fp32 closed form; %d type flips (%d exempt); final %.2f ulp of x0_f'
          % (S, worst, flips, exempt, final_ulps))
    assert worst <= 4.0 and flips == 0 and exempt <= 2
    assert final_ulps <= 1.0
    assert torch.equal(got['v'][mask], v0) and torch.equal(got['v_traj'][-1][mask], v0)


# ------------------------------------------------------------------------------------------------ F. driver and CLI
def test_1h36_driver_cpu_rng_vs_oracle():
    """rng='cpu' with a 20-step respaced sequence on the 1h36 pocket, prior sizes, seed 2021: oracle.respaced's driver restatement
    draws the same sizes and noise; types equal, positions within the chain tolerances."""
    from targetdiff_b200 import atom_num
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand, seed_all
    torch.set_num_threads(16)
    model, sd = _model()
    data = pdb_to_pocket_data(PDB_1H36)
    seq = respaced_time_seq(1000, 20)
    seed_all(2021)
    got = sample_diffusion_ligand(model, data, 2, batch_size=2, device=DEV, sample_num_atoms='prior', rng='cpu', time_seq=seq)
    seed_all(2021)
    want = respaced.sample_diffusion_ligand(sd, None, data.protein_pos, data.protein_atom_feature, 2, atom_num._table(), seq, batch_size=2)
    assert [len(p) for p in got[0]] == [len(p) for p in want[0]]
    assert np.array_equal(np.concatenate(got[1]), np.concatenate(want[1]))
    assert np.array_equal(np.concatenate(got[3], axis=1), np.concatenate(want[3], axis=1))
    np.testing.assert_allclose(np.concatenate(got[2], axis=1), np.concatenate(want[2], axis=1), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(np.concatenate(got[0]), np.concatenate(want[0]), rtol=1e-4, atol=1e-4)
    assert got[2][0].shape[0] == len(seq)


def test_cli_respaced_steps_with_fragment(tmp_path):
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
                       'sample_num_atoms': 'range', 'respaced_steps': 6}}
    with open(tmp_path / 'sample.yml', 'w') as f:
        yaml.safe_dump(conf, f)
    from targetdiff_b200.pocket import pdb_to_pocket_data
    ctr = pdb_to_pocket_data(PDB_1H36).protein_pos.float().mean(0)
    frag = {'pos': ctr + torch.randn(2, 3, generator=torch.Generator().manual_seed(4)), 'v': torch.tensor([1, 3])}
    torch.save(frag, tmp_path / 'frag.pt')
    main(['sample_for_pocket', str(tmp_path / 'sample.yml'), '--pdb_path', PDB_1H36, '--result_path', str(tmp_path / 'out'),
          '--device', DEV, '--fragment', str(tmp_path / 'frag.pt')])
    r = torch.load(tmp_path / 'out' / 'sample.pt', weights_only=False)
    assert r['time_seq'] == respaced_time_seq(20, 6) == [19, 15, 11, 8, 4, 0]
    assert r['fixed_ligand_atoms'] == 2
    for pos, v, ptraj, vtraj in zip(r['pred_ligand_pos'], r['pred_ligand_v'], r['pred_ligand_pos_traj'], r['pred_ligand_v_traj']):
        assert ptraj.shape == (6, len(pos), 3) and vtraj.shape == (6, len(pos))
        assert torch.allclose(torch.from_numpy(pos[:2]).float(), frag['pos'], rtol=EPS32, atol=0)
        assert v[:2].tolist() == [1, 3]
    conf['sample']['num_steps'] = 10
    with open(tmp_path / 'bad.yml', 'w') as f:
        yaml.safe_dump(conf, f)
    with pytest.raises(ValueError, match='num_steps'):
        main(['sample_for_pocket', str(tmp_path / 'bad.yml'), '--pdb_path', PDB_1H36, '--result_path', str(tmp_path / 'bad'), '--device', DEV])


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
    model._bind(eng, a[0], a[1], a[2], a[5], 1)
    lpos, lv = a[3].float().contiguous(), a[4].long().contiguous()
    _lib.check(lib.tdiff_set_ligand(eng, ctypes.c_void_p(lpos.data_ptr()), ctypes.c_void_p(lv.data_ptr()), 1, st))

    def run(seq, S=None, arr=True):
        S = len(seq) if S is None else S
        return lib.tdiff_sample_seq(eng, _lib.i32_array(seq) if arr else None, S, None, None, ctypes.c_uint64(1), None, None, None, None, 0, st)

    cases = {'null pointer': ([T - 1], None, False), 'empty': ([T - 1], 0, True), 'outside': (list(range(T - 1, -1, -1)) + [0], None, True),
             'not at T - 1': ([T - 2, 5, 0], None, True), 'not strictly decreasing': ([T - 1, 5, 5, 0], None, True),
             'negative': ([T - 1, 3, -2], None, True)}
    for msg, (seq, S, arr) in cases.items():
        assert run(seq, S, arr) == _lib.TDIFF_EINVAL, msg
        assert msg in lib.tdiff_last_error().decode(), (msg, lib.tdiff_last_error())
    assert run([T - 1, 400, 0]) == _lib.TDIFF_OK                # the engine is still usable
    torch.cuda.synchronize()
