"""Clash guidance on the CPU (DESIGN.md section 1): the rule's closed forms in float64, the guided oracle chain at strength 0 against
the unguided one, the config / Python refusals and the result field."""
import math

import numpy as np

import pytest
import torch
import yaml

from oracle import clash_guidance as cg
from oracle import resample, restate, synth
from targetdiff_b200.cli import add_clash_guidance
from targetdiff_b200.config import Config, check_clash_guidance, sample_clash_guidance

D = torch.float64


def _one(y, prot, radius, strength):
    y = torch.tensor(y, dtype=D).reshape(-1, 3)
    prot = torch.tensor(prot, dtype=D).reshape(-1, 3)
    return cg.guide(y, prot, torch.zeros(len(y), dtype=torch.long), torch.zeros(len(prot), dtype=torch.long), radius, strength)


def test_isolated_contact_lands_at_the_radius():
    for y, p, rho in (([0.3, -0.2, 0.5], [0.0, 0.0, 0.0], 2.0), ([1.0, 2.0, 3.0], [1.7, 1.1, 2.4], 3.5), ([5.0, 5.0, 5.0], [4.999, 5.0, 5.0], 1.0)):
        out = _one(y, p, rho, 1.0)
        d = float(torch.linalg.norm(out[0] - torch.tensor(p, dtype=D)))
        assert abs(d - rho) <= 1e-12 * rho, (y, p, rho, d)
        # lambda = 0.5 moves it half way
        half = _one(y, p, rho, 0.5)
        d0 = float(torch.linalg.norm(torch.tensor(y, dtype=D) - torch.tensor(p, dtype=D)))
        assert abs(float(torch.linalg.norm(half[0] - torch.tensor(p, dtype=D))) - 0.5 * (d0 + rho)) <= 1e-12 * rho


def test_pairs_at_the_radius_and_coincident_pairs_do_not_contribute():
    y = [1.0, 2.0, 3.0]
    assert torch.equal(_one(y, [3.0, 2.0, 3.0], 2.0, 1.0)[0], torch.tensor(y, dtype=D))        # d = rho exactly
    out = _one(y, [1.0, 2.0, 3.0], 2.0, 1.0)                                                     # d = 0
    assert torch.isfinite(out).all() and torch.equal(out[0], torch.tensor(y, dtype=D))
    # a coincident pair next to a contributing one: only the contributing one acts
    out = _one(y, [[1.0, 2.0, 3.0], [1.5, 2.0, 3.0]], 2.0, 1.0)
    assert torch.isfinite(out).all()
    assert torch.allclose(out[0], torch.tensor([-0.5, 2.0, 3.0], dtype=D), rtol=0, atol=1e-15)


def test_symmetric_contacts_cancel():
    y = [0.25, -1.0, 2.0]
    out = _one(y, [[0.25 - 0.75, -1.0, 2.0], [0.25 + 0.75, -1.0, 2.0]], 1.5, 1.0)
    assert torch.allclose(out[0], torch.tensor(y, dtype=D), rtol=0, atol=1e-15)


def test_atoms_without_contacts_are_returned_bit_for_bit():
    g = torch.Generator().manual_seed(3)
    y = torch.randn(40, 3, generator=g, dtype=D) * 4
    prot = torch.randn(300, 3, generator=g, dtype=D) * 6
    bl, bp = torch.arange(40) % 3, torch.arange(300) % 3
    for dt in (torch.float64, torch.float32):
        out = cg.guide(y.to(dt), prot.to(dt), bl, bp, 1.2, 0.7, dtype=dt)
        d = torch.cdist(y, prot, compute_mode='donot_use_mm_for_euclid_dist')
        d[bl[:, None] != bp[None, :]] = float('inf')
        far = (d.min(1).values >= 1.2)
        assert int(far.sum()) > 5 and int((~far).sum()) > 2
        assert torch.equal(out[far], y.to(dt)[far])
        assert not torch.equal(out[~far], y.to(dt)[~far])
    assert torch.equal(cg.guide(y, prot, bl, bp, 1.2, 0.0), y)


def test_the_update_is_minus_half_lambda_times_the_energy_gradient():
    g = torch.Generator().manual_seed(5)
    prot = torch.randn(60, 3, generator=g, dtype=D) * 2.5
    y = torch.randn(12, 3, generator=g, dtype=D) * 2.0
    bl, bp = torch.zeros(12, dtype=torch.long), torch.zeros(60, dtype=torch.long)
    rho, lam, h = 1.7, 0.8, 1e-6
    step = cg.guide(y, prot, bl, bp, rho, lam) - y
    grad = torch.zeros_like(y)
    for i in range(y.shape[0]):
        for k in range(3):
            yp, ym = y.clone(), y.clone()
            yp[i, k] += h
            ym[i, k] -= h
            grad[i, k] = (cg.energy(yp, prot, bl, bp, rho) - cg.energy(ym, prot, bl, bp, rho)) / (2 * h)
    assert float(grad.abs().max()) > 0.1
    assert torch.allclose(step, -0.5 * lam * grad, rtol=0, atol=1e-7)


@pytest.fixture(scope='module')
def sd():
    return synth.make_state_dict(0, schedules=restate.make_schedules())


def _chain_cases(sd):
    T = sd['betas'].shape[0]
    b = synth.make_batch(11, 2, n_protein=40, ligand_sizes=[6, 9])
    nl = len(b['batch_ligand'])
    seq = [T - 1, T // 2, T // 4, 3, 0]
    path = [T - 1, T - 2, T - 1, T - 3, T - 5, T - 4, T - 6]
    fm = torch.zeros(nl, dtype=torch.bool)
    fm[[0, 1, 7]] = True
    g = torch.Generator().manual_seed(4)
    ftape = lambda S: (torch.randn(S + 1, nl, 3, generator=g), torch.rand(S + 1, nl, synth.LIGAND_NUM_CLASSES, generator=g))
    stape = (torch.randn(nl, 3, generator=g), torch.rand(nl, synth.LIGAND_NUM_CLASSES, generator=g))
    yield 'default', b, cg.unit_path(T, 4), {}
    yield 'respaced', b, seq, {}
    yield 'fragment', b, seq, dict(fixed_mask=fm, fixed_tape=ftape(len(seq)))
    yield 'start', b, [9, 6, 3, 0], dict(start_time=9, start_tape=stape, fixed_mask=fm, fixed_tape=ftape(4))
    yield 'path', b, path, dict(fixed_mask=fm, fixed_tape=ftape(len(path)))


@pytest.mark.parametrize('mean_type', ['C0', 'noise'])
def test_oracle_chains_without_guidance_are_the_unguided_chains(sd, mean_type):
    """guidance=None is resample.sample_diffusion itself; the restated loop with a strength-0 hook gives the same bits."""
    cfg = {'model_mean_type': mean_type}
    for label, b, path, kw in _chain_cases(sd):
        pn, vu = synth.make_tape(2, len(path), len(b['batch_ligand']))
        args = (sd, cfg, b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'],
                b['batch_ligand'], pn, vu, path)
        want = resample.sample_diffusion(*args, **kw)
        for guidance in (None, cg.hook(2.0, 0.0)):
            got = cg.sample_diffusion(*args, guidance=guidance, **kw)
            assert torch.equal(got['pos'], want['pos']) and torch.equal(got['v'], want['v']), (label, guidance)
            for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
                assert all(torch.equal(x, y) for x, y in zip(got[k], want[k])), (label, k)
        # and guidance on moves something
        on = cg.sample_diffusion(*args, guidance=cg.hook(4.0, 1.0), **kw)
        assert not torch.equal(on['pos'], want['pos']), label


def test_config_and_python_refusals():
    assert check_clash_guidance(None, 0.0) == (None, 0.0)
    assert check_clash_guidance(3.0, 0) == (None, 0.0)                 # radius ignored when off
    assert check_clash_guidance(2, 1) == (2.0, 1.0)
    assert sample_clash_guidance(Config()) == (None, 0.0)
    assert sample_clash_guidance(Config(clash_radius=2.5, clash_strength=0.5)) == (2.5, 0.5)
    for r, s, msg in ((2.0, -1.0, 'finite and >= 0'), (2.0, float('nan'), 'finite and >= 0'), (2.0, float('inf'), 'finite and >= 0'),
                      (None, 1.0, 'needs a clash_radius'), (0.0, 1.0, 'finite number > 0'), (-1.0, 1.0, 'finite number > 0'),
                      (float('inf'), 1.0, 'finite number > 0'), (float('nan'), 1.0, 'finite number > 0'), (2.0, True, 'must be a number'),
                      (2.0, '1', 'must be a number')):
        with pytest.raises(ValueError, match=msg):
            check_clash_guidance(r, s)
        with pytest.raises(ValueError, match=msg):
            sample_clash_guidance(Config(clash_radius=r, clash_strength=s))


def test_python_entry_points_refuse_before_touching_the_engine():
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.sampling import sample_diffusion_ligand
    from targetdiff_b200.score_model import ScorePosNet3D
    m = ScorePosNet3D(default_model_config(), 27, 13)
    z = torch.zeros
    with pytest.raises(ValueError, match='needs a clash_radius'):
        m.sample_diffusion(z(3, 3), z(3, 27), z(3, dtype=torch.long), z(1, 3), z(1, dtype=torch.long), z(1, dtype=torch.long), num_steps=2,
                           clash_strength=1.0)
    with pytest.raises(ValueError, match='finite and >= 0'):
        sample_diffusion_ligand(m, None, 1, clash_radius=2.0, clash_strength=-0.5)


def _conf(tmp_path, **sample):
    conf = {'model': {'checkpoint': str(tmp_path / 'missing.pt')},
            'sample': dict({'seed': 1, 'num_samples': 2, 'num_steps': 20, 'pos_only': False, 'center_pos_mode': 'protein',
                            'sample_num_atoms': 'range'}, **sample)}
    path = tmp_path / 'sample.yml'
    with open(path, 'w') as f:
        yaml.safe_dump(conf, f)
    return str(path)


def test_cli_refusals(tmp_path):
    """Refused before any checkpoint is read or device touched, in both commands."""
    from targetdiff_b200.cli import main
    pdb = str(tmp_path / 'p.pdb')
    open(pdb, 'w').close()
    (tmp_path / 'pockets').mkdir()
    for cmd in (['sample_for_pocket', None, '--pdb_path', pdb], ['sample_pockets', None, '--pocket_dir', str(tmp_path / 'pockets')]):
        for bad, msg in ((dict(clash_strength=1.0), 'needs a clash_radius'), (dict(clash_strength=-1.0, clash_radius=2.0), '>= 0'),
                         (dict(clash_strength=1.0, clash_radius=0.0), 'finite number > 0')):
            cmd[1] = _conf(tmp_path, **bad)
            with pytest.raises(ValueError, match=msg):
                main(cmd)


def test_result_field_only_when_guidance_is_on():
    assert add_clash_guidance({'a': 1}, None, 0.0) == {'a': 1}
    assert add_clash_guidance({'a': 1}, 2.0, 0.5) == {'a': 1, 'clash_guidance': {'radius': 2.0, 'strength': 0.5}}
    assert math.isclose(add_clash_guidance({}, 1.5, 1.0)['clash_guidance']['radius'], 1.5)


def test_oracle_driver_without_guidance_is_the_unguided_driver(sd):
    """The hooked rng='cpu' driver at strength 0 makes the draws and gives the bits of oracle.resample's driver."""
    b = synth.make_batch(12, 1, n_protein=40, ligand_sizes=[5])
    path = [999, 600, 700, 300, 0]
    frag = (b['protein_pos'].mean(0) + torch.randn(2, 3, generator=torch.Generator().manual_seed(1)), torch.tensor([1, 3]))
    outs = []
    for fn, kw in ((resample.sample_diffusion_ligand, {}), (cg.sample_diffusion_ligand, {'guidance': cg.hook(2.0, 0.0)})):
        torch.manual_seed(5)
        outs.append(fn(sd, None, b['protein_pos'], b['protein_v'], 3, None, path, batch_size=2, sample_num_atoms='range',
                       fixed_ligand=frag, **kw) + (torch.rand(1),))
    for x, y in zip(outs[0][:6], outs[1][:6]):
        assert all(np.array_equal(p, q) for p, q in zip(x, y))
    assert torch.equal(outs[0][-1], outs[1][-1])                 # the same number of draws
