"""Element constraints on the CPU (DESIGN.md section 1): the class tables against the reference's maps, the constrained oracle chain
with the full set against the unconstrained one, the conditioned posterior against a float64 closed form, an adversarial tape, the
config / driver / CLI refusals and the result field."""
import json
import math
import os

import numpy as np
import pytest
import torch
import yaml

from oracle import clash_guidance as cg
from oracle import resample, restate, synth
from oracle import type_constraints as tc
from targetdiff_b200 import pocket
from targetdiff_b200.config import Config, sample_allowed_classes

ROOT = os.path.dirname(os.path.abspath(__file__))
K13 = synth.LIGAND_NUM_CLASSES
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj')


# ------------------------------------------------------------------------------------------------ class tables
def test_class_tables_are_the_reference_maps():
    """tests/golden/reference_ligand_class_maps.json: the reference's MAP_ATOM_TYPE_{ONLY,AROMATIC,FULL}_TO_INDEX (oracle/make_class_map_pins.py)."""
    with open(os.path.join(ROOT, 'golden', 'reference_ligand_class_maps.json')) as f:
        pins = json.load(f)
    ours = {'basic': [[z] for z in pocket.LIGAND_CLASS_TO_ATOM_BASIC], 'add_aromatic': [list(a) for a in pocket.LIGAND_CLASS_TO_ATOM],
            'full': [list(a) for a in pocket.LIGAND_CLASS_TO_ATOM_FULL]}
    assert sorted(pins) == sorted(ours) == sorted(pocket.LIGAND_CLASS_ELEMENTS)
    for mode, pairs in pins.items():
        assert [i for _, i in pairs] == list(range(len(pairs))), mode
        assert [k for k, _ in pairs] == ours[mode], mode
        zs = [k[0] for k, _ in pairs]
        assert list(pocket.LIGAND_CLASS_ELEMENTS[mode]) == zs
        for z in sorted(set(zs)):                        # every class of an element, no other
            sym = pocket.ELEMENT_SYMBOL[z]
            assert pocket.element_classes([sym], mode) == [i for i, y in enumerate(zs) if y == z], (mode, sym)
    assert pocket.element_classes(['C', 'N', 'O'], 'add_aromatic') == [1, 2, 3, 4, 5, 6]
    assert pocket.element_classes(['C', 'N', 'O'], 'basic') == [1, 2, 3]
    assert pocket.element_classes(['o', 'Cl'], 'full') == [9, 10, 11, 22]


def test_element_helper_refusals():
    with pytest.raises(ValueError, match='H, C, N, O, F, P, S, Cl'):
        pocket.element_classes(['C', 'Br'], 'add_aromatic')
    with pytest.raises(ValueError, match='not a ligand class'):
        pocket.element_classes(['Se'], 'full')
    with pytest.raises(ValueError, match='at least one element'):
        pocket.element_classes([], 'basic')
    with pytest.raises(ValueError, match='ligand_atom_mode'):
        pocket.element_classes(['C'], 'other')


def test_type_violations():
    from targetdiff_b200.analyze import type_violations
    v = np.array([0, 1, 2, 5, 12])
    assert type_violations(v, [1, 2, 5]) == 2
    m = torch.zeros(K13, dtype=torch.bool)
    m[[0, 12]] = True
    assert type_violations(torch.from_numpy(v), m) == 3
    per = torch.ones(5, K13, dtype=torch.bool)
    per[3, 5] = False
    assert type_violations([v[:2], v[2:]], per) == 1
    assert type_violations([], [1]) == 0


# ------------------------------------------------------------------------------------------------ the oracle with the full set
@pytest.fixture(scope='module')
def sd():
    return synth.make_state_dict(0, schedules=restate.make_schedules())


def _chain_cases(sd):
    T = sd['betas'].shape[0]
    b = synth.make_batch(11, 2, n_protein=40, ligand_sizes=[6, 9])
    nl = len(b['batch_ligand'])
    seq = [T - 1, T // 2, T // 4, 3, 0]
    path = [T - 1, T - 2, T - 1, T // 2, 40, 300, 2, 0]
    fm = torch.zeros(nl, dtype=torch.bool)
    fm[[0, 1, 7]] = True
    g = torch.Generator().manual_seed(4)
    ftape = lambda S: (torch.randn(S + 1, nl, 3, generator=g), torch.rand(S + 1, nl, K13, generator=g))
    stape = (torch.randn(nl, 3, generator=g), torch.rand(nl, K13, generator=g))
    yield 'default', b, cg.unit_path(T, 4), {}
    yield 'respaced', b, seq, {}
    yield 'fragment', b, seq, dict(fixed_mask=fm, fixed_tape=ftape(len(seq)))
    yield 'start', b, [9, 6, 3, 0], dict(start_time=9, start_tape=stape, fixed_mask=fm, fixed_tape=ftape(4))
    yield 'path', b, path, dict(fixed_mask=fm, fixed_tape=ftape(len(path)))


def _same(a, b):
    return torch.equal(a['pos'], b['pos']) and torch.equal(a['v'], b['v']) and \
        all(len(a[k]) == len(b[k]) and all(torch.equal(x, y) for x, y in zip(a[k], b[k])) for k in TRAJ)


@pytest.mark.parametrize('mean_type', ['C0', 'noise'])
def test_full_set_is_the_unconstrained_oracle_chain(sd, mean_type):
    """allowed=None is clash_guidance.sample_diffusion itself; the full mask runs the masked loop and gives its bits, with and without
    clash guidance; a constraint changes the chains that end at t = 0."""
    cfg = {'model_mean_type': mean_type}
    for label, b, path, kw in _chain_cases(sd):
        nl = len(b['batch_ligand'])
        pn, vu = synth.make_tape(2, len(path), nl)
        args = (sd, cfg, b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'],
                b['batch_ligand'], pn, vu, path)
        want = resample.sample_diffusion(*args, **kw)
        full = torch.ones(nl, K13, dtype=torch.bool)
        assert _same(tc.sample_diffusion(*args, **kw), want), label
        assert _same(tc.sample_diffusion(*args, allowed=full, **kw), want), label
        hook = cg.hook(3.0, 0.5)
        assert _same(tc.sample_diffusion(*args, allowed=full, guidance=hook, **kw), cg.sample_diffusion(*args, guidance=hook, **kw)), label
        few = torch.zeros(nl, K13, dtype=torch.bool)
        few[:, [1, 3]] = True
        on = tc.sample_diffusion(*args, allowed=few, **kw)
        assert not torch.equal(torch.stack(on['v0_traj']), torch.stack(want['v0_traj'])), label
        assert all(torch.isfinite(x).any(1).all() and not torch.isnan(x).any() for k in ('v0_traj', 'vt_traj') for x in on[k]), label
        if path[-1] == 0:
            free = ~kw['fixed_mask'] if 'fixed_mask' in kw else torch.ones(nl, dtype=torch.bool)
            assert bool(few[free, on['v'][free]].all()), label


def test_full_set_driver_is_the_unconstrained_driver(sd):
    """The rng='cpu' driver with the full set makes the same draws and gives the bits of clash_guidance's driver."""
    b = synth.make_batch(12, 1, n_protein=40, ligand_sizes=[5])
    path = [999, 600, 700, 300, 0]
    frag = (b['protein_pos'].mean(0) + torch.randn(2, 3, generator=torch.Generator().manual_seed(1)), torch.tensor([1, 3]))
    outs = []
    for fn, kw in ((cg.sample_diffusion_ligand, {}), (tc.sample_diffusion_ligand, {'allowed': torch.ones(K13, dtype=torch.bool)})):
        torch.manual_seed(5)
        outs.append(fn(sd, None, b['protein_pos'], b['protein_v'], 3, None, path, batch_size=2, sample_num_atoms='range',
                       fixed_ligand=frag, **kw) + (torch.rand(1),))
    for x, y in zip(outs[0][:6], outs[1][:6]):
        assert all(np.array_equal(p, q) for p, q in zip(x, y))
    assert torch.equal(outs[0][-1], outs[1][-1])
    torch.manual_seed(5)
    allowed = torch.zeros(K13, dtype=torch.bool)
    allowed[[2, 5]] = True
    r = tc.sample_diffusion_ligand(sd, None, b['protein_pos'], b['protein_v'], 3, None, path, batch_size=2, sample_num_atoms='range',
                                   fixed_ligand=frag, allowed=allowed)
    for v in r[1]:                                          # the fragment rows keep their classes, the grown atoms are 2 or 5
        assert v[:2].tolist() == [1, 3] and set(v[2:].tolist()) <= {2, 5}


# ------------------------------------------------------------------------------------------------ float64 closed form
def test_conditioned_posterior_closed_form(sd):
    """The step's type outputs at float64 against the posterior written out in probability space: v0_hat = softmax over A (0
    elsewhere), q(v_p | v_t, v0_hat) proportional to (abar_p v0_hat + (1 - abar_p) / K) (a v_t + (1 - a) / K), and on the decoder step
    restricted to A and renormalised."""
    g = torch.Generator().manual_seed(9)
    n = 7
    seq = [999, 620, 300, 41, 1, 0]
    tab = resample.path_tables(sd, seq)
    xt = torch.randn(n, 3, generator=g)
    x0 = torch.randn(n, 3, generator=g)
    logits = torch.randn(n, K13, generator=g) * 3
    vt = torch.randint(0, K13, (n,), generator=g)
    allowed = torch.rand(n, K13, generator=g) < 0.4
    allowed[torch.arange(n), vt] = allowed[torch.arange(n), vt] & (torch.arange(n) % 2 == 0)     # v_t itself sometimes forbidden
    allowed[0] = False
    allowed[0, 4] = True                                    # a single-class row
    allowed[1] = True
    pn, vu = torch.randn(n, 3, generator=g), torch.rand(n, K13, generator=g)
    L = logits.double().numpy()
    A = allowed.numpy()
    for s in range(len(seq)):
        p = int(tab['p'][s])
        out = tc.conditioned_step(sd, None, tab, s, xt, vt, x0, logits, pn, vu, allowed, dtype=torch.float64)
        e = np.where(A, np.exp(L - L.max(1, keepdims=True)), 0.0)
        v0hat = e / e.sum(1, keepdims=True)
        pm = max(p, 0)
        abar = math.exp(float(sd['log_alphas_cumprod_v'][pm]))
        om_abar = math.exp(float(sd['log_one_minus_alphas_cumprod_v'][pm]))
        a, om_a = math.exp(float(tab['la'][s])), math.exp(float(tab['l1ma'][s]))
        onehot = np.full((n, K13), 1e-30)
        onehot[np.arange(n), vt.numpy()] = 1.0
        un = (abar * v0hat + om_abar / K13) * (a * onehot + om_a / K13)
        if p < 0:
            un = np.where(A, un, 0.0)
        post = un / un.sum(1, keepdims=True)
        with np.errstate(divide='ignore'):
            want_v0, want_vt = np.log(v0hat), np.log(post)
        got_v0, got_vt = out['v0'].numpy(), out['vt'].numpy()
        assert np.array_equal(np.isneginf(got_v0), ~A) and np.array_equal(np.isneginf(got_vt), np.isneginf(want_vt)), s
        assert np.isneginf(want_vt).any() == (p < 0)
        fin = np.isfinite(want_v0)
        assert np.abs(got_v0[fin] - want_v0[fin]).max() <= 1e-12, s
        fin = np.isfinite(want_vt)
        assert np.abs(got_vt[fin] - want_vt[fin]).max() <= 1e-9, s
        if p < 0:
            assert bool(allowed[torch.arange(n), out['v']].all())
            assert float(out['vt'][0, 4]) == 0.0 and float(out['v0'][0, 4]) == 0.0 and int(out['v'][0]) == 4


# ------------------------------------------------------------------------------------------------ adversarial tape
def test_adversarial_tape_draws_the_forbidden_class_only_before_the_decoder_step(sd):
    """Uniforms of 1 - 2^-24 on a forbidden class c and 1e-6 elsewhere give c a Gumbel lead of about 19 at every step: the intermediate
    states take it, the decoder step cannot."""
    b = synth.make_batch(13, 2, n_protein=40, ligand_sizes=[5, 7])
    nl = len(b['batch_ligand'])
    seq = [999, 500, 100, 20, 5, 0]
    pn, _ = synth.make_tape(3, len(seq), nl)
    c = 7
    vu = torch.full((len(seq), nl, K13), 1e-6)
    vu[:, :, c] = float(np.float32(1.0 - 2.0 ** -24))
    allowed = torch.ones(nl, K13, dtype=torch.bool)
    allowed[:, c] = False
    args = (sd, None, b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'],
            pn, vu, seq)
    r = tc.sample_diffusion(*args, allowed=allowed)
    plain = resample.sample_diffusion(*args)
    assert bool((plain['v'] == c).all())                                  # without the constraint every atom ends in c
    assert bool((r['v_traj'][-2] == c).all())                             # the step before the decoder step drew c everywhere
    assert int((r['v'] == c).sum()) == 0
    assert bool(torch.isneginf(r['vt_traj'][-1][:, c]).all()) and bool(torch.isneginf(r['v0_traj'][-1][:, c]).all())


# ------------------------------------------------------------------------------------------------ config, driver, CLI
def test_config_keys():
    assert sample_allowed_classes(Config(), 'add_aromatic') is None
    assert sample_allowed_classes(Config(allowed_elements=['C', 'N', 'O']), 'add_aromatic') == [1, 2, 3, 4, 5, 6]
    assert sample_allowed_classes(Config(allowed_elements=['C', 'N', 'O']), 'basic') == [1, 2, 3]
    assert sample_allowed_classes(Config(allowed_classes=[5, 1, 5]), 'add_aromatic') == [1, 5]
    for bad, mode, msg in ((dict(allowed_elements=['C'], allowed_classes=[1]), 'basic', 'not both'),
                           (dict(allowed_elements=['C', 'Br']), 'basic', 'H, C, N, O, F, P, S, Cl'),
                           (dict(allowed_elements='C'), 'basic', 'list of element symbols'),
                           (dict(allowed_elements=[]), 'basic', 'at least one element'),
                           (dict(allowed_classes=[]), 'basic', 'non-empty list'),
                           (dict(allowed_classes=[8]), 'basic', r'0\.\.7'), (dict(allowed_classes=[-1]), 'full', r'0\.\.22'),
                           (dict(allowed_classes=[True]), 'full', 'not a class index'), (dict(allowed_classes=[1.0]), 'full', 'not a class')):
        with pytest.raises(ValueError, match=msg):
            sample_allowed_classes(Config(**bad), mode)


def test_python_entry_points_refuse_before_touching_the_engine():
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand
    from targetdiff_b200.score_model import ScorePosNet3D
    m = ScorePosNet3D(default_model_config(), 27, K13)
    z = torch.zeros
    with pytest.raises(ValueError, match='pos_only'):
        m.sample_diffusion(z(3, 3), z(3, 27), z(3, dtype=torch.long), z(1, 3), z(1, dtype=torch.long), z(1, dtype=torch.long), num_steps=2,
                           pos_only=True, allowed_types=torch.ones(1, K13, dtype=torch.bool))
    data = pdb_to_pocket_data(os.path.join(ROOT, 'golden', '1h36_pocket10.pdb'))
    start = (torch.zeros(4, 3), torch.tensor([1, 3, 5, 1]))
    few = torch.zeros(K13, dtype=torch.bool)
    for kw, msg in ((dict(allowed_types=[]), 'empty'), (dict(allowed_types=[1, 13]), r'0\.\.12'), (dict(allowed_types=[-1]), r'0\.\.12'),
                    (dict(allowed_types=few), 'allows no class'), (dict(allowed_types=torch.ones(5, dtype=torch.bool)), r'\[K\]'),
                    (dict(allowed_types=[1.5]), 'class indices'), (dict(allowed_types=[1], pos_only=True), 'pos_only'),
                    (dict(allowed_types=torch.ones(4, K13, dtype=torch.bool)), 'needs a start_ligand'),
                    (dict(allowed_types=torch.ones(3, K13, dtype=torch.bool), start_ligand=start, start_time=10), r'\[n, K\] = \(4, 13\)'),
                    (dict(allowed_types=torch.eye(K13, dtype=torch.bool)[[0, 1, 2, 4]] & torch.tensor([True] * 3 + [False] * 10),
                          start_ligand=start, start_time=10), r'start atom\(s\) \[3\]')):
        with pytest.raises(ValueError, match=msg):
            sample_diffusion_ligand(m, data, 1, device='cpu', **kw)


def _ckpt(tmp_path, mode='add_aromatic'):
    from targetdiff_b200.cli import LIGAND_ATOM_MODE_CLASSES
    from targetdiff_b200.config import default_model_config
    cfg = dict(num_diffusion_timesteps=20)
    sd = synth.make_state_dict(0, cfg, schedules=restate.make_schedules(cfg), ligand_dim=LIGAND_ATOM_MODE_CLASSES[mode])
    mc = default_model_config()
    mc.update(cfg)
    torch.save({'config': Config(model=mc, data={'transform': {'ligand_atom_mode': mode}}), 'model': sd}, tmp_path / 'ckpt.pt')


def _conf(tmp_path, **sample):
    conf = {'model': {'checkpoint': str(tmp_path / 'ckpt.pt')},
            'sample': dict({'seed': 1, 'num_samples': 2, 'num_steps': 20, 'pos_only': False, 'center_pos_mode': 'protein',
                            'sample_num_atoms': 'range'}, **sample)}
    path = tmp_path / 'sample.yml'
    with open(path, 'w') as f:
        yaml.safe_dump(conf, f)
    return str(path)


def _commands(tmp_path):
    import shutil
    pdb = os.path.join(ROOT, 'golden', '1h36_pocket10.pdb')
    (tmp_path / 'pockets').mkdir(exist_ok=True)
    shutil.copyfile(pdb, tmp_path / 'pockets' / 'p.pdb')
    return {'sample_for_pocket': ['sample_for_pocket', None, '--pdb_path', pdb, '--device', 'cpu', '--result_path', str(tmp_path / 'a')],
            'sample_pockets': ['sample_pockets', None, '--pocket_dir', str(tmp_path / 'pockets'), '--device', 'cpu', '--result_path',
                               str(tmp_path / 'b')]}


def test_cli_refusals(tmp_path):
    """Refused in the checkpoint's atom mode, before anything is sampled, in both commands."""
    from targetdiff_b200.cli import main
    _ckpt(tmp_path, 'basic')
    for cmd in _commands(tmp_path).values():
        for bad, msg in ((dict(allowed_elements=['C'], allowed_classes=[1]), 'not both'),
                         (dict(allowed_elements=['C', 'Br']), 'basic mode .*H, C, N, O, F, P, S, Cl'),
                         (dict(allowed_classes=[8]), r'0\.\.7')):
            cmd[1] = _conf(tmp_path, **bad)
            with pytest.raises(ValueError, match=msg):
                main(cmd)


@pytest.mark.parametrize('command', ['sample_for_pocket', 'sample_pockets'])
def test_cli_passes_the_set_and_writes_the_field(tmp_path, monkeypatch, command):
    """The CLI's wiring with the sampler replaced: the config's set reaches sample_diffusion_ligand as class indices of the checkpoint's
    mode, and the result file holds 'allowed_classes' only with a constraint."""
    from targetdiff_b200 import cli
    calls = []

    def fake_sampler(model, data, num_samples, **kw):
        calls.append(kw.get('allowed_types'))
        pos = [np.zeros((3, 3)) for _ in range(num_samples)]
        return pos, [np.zeros(3, dtype=np.int64)] * num_samples, pos, pos, pos, pos, [0.5]

    monkeypatch.setattr(cli, 'sample_diffusion_ligand', fake_sampler)
    _ckpt(tmp_path, 'full')
    cmd = _commands(tmp_path)[command]
    out = tmp_path / ('a' if command == 'sample_for_pocket' else 'b') / ('sample.pt' if command == 'sample_for_pocket' else 'result_0.pt')
    for sample, want in ((dict(allowed_elements=['N', 'O']), [5, 6, 7, 8, 9, 10, 11]), (dict(allowed_classes=[0, 22]), [0, 22]), ({}, None)):
        cmd[1] = _conf(tmp_path, **sample)
        cli.main(cmd)
        assert calls[-1] == want
        r = torch.load(out, weights_only=False)
        if want is None:
            assert 'allowed_classes' not in r
        else:
            assert r['allowed_classes'] == want
