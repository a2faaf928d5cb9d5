"""Connectivity guidance on the CPU (DESIGN.md section 1): the rule's closed forms in float64, the guided oracle chains and driver at
strength 0 against the unguided ones, the config / Python / CLI refusals and the result field."""
import numpy as np

import pytest
import torch
import yaml

from oracle import clash_guidance as cg
from oracle import connect_guidance as kg
from oracle import resample, restate, synth
from targetdiff_b200.analyze import ligand_components
from targetdiff_b200.cli import add_connect_guidance
from targetdiff_b200.config import Config, check_connect_guidance, sample_connect_guidance

D = torch.float64


def _one(y, radius, length, strength, held=None, info=None):
    y = torch.tensor(y, dtype=D).reshape(-1, 3)
    hm = None if held is None else torch.tensor(held, dtype=torch.bool)
    return kg.guide(y, torch.zeros(len(y), dtype=torch.long), radius, length, strength, held=hm, targets=y, info=info)


def _dist(a, b):
    return float(torch.linalg.norm(a - b))


def test_two_free_components_end_their_closest_pair_at_the_bond_length():
    # piece A = rows 0, 1 (bonded), piece B = rows 2, 3; the closest pair is (1, 2)
    y = [[0.0, 0.0, 0.0], [1.2, 0.3, -0.1], [4.0, 1.0, 0.5], [5.1, 1.4, 0.2]]
    for lam in (1.0, 0.5):
        out = _one(y, 2.0, 1.5, lam)
        t = torch.tensor(y, dtype=D)
        d0 = _dist(t[1], t[2])
        assert abs(_dist(out[1], out[2]) - (d0 - lam * (d0 - 1.5))) <= 1e-12
        # rigid moves: each piece keeps its shape, and the two move by opposite halves
        assert abs(_dist(out[0], out[1]) - _dist(t[0], t[1])) <= 1e-12 and abs(_dist(out[2], out[3]) - _dist(t[2], t[3])) <= 1e-12
        assert torch.allclose((out[:2] - t[:2]).sum(0) / 2, -(out[2:] - t[2:]).sum(0) / 2, rtol=0, atol=1e-12)


def test_a_held_component_stays_and_its_partner_takes_the_full_step():
    y = [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [4.5, 2.0, 0.0], [5.5, 2.5, 0.0]]
    t = torch.tensor(y, dtype=D)
    out = _one(y, 2.0, 1.4, 1.0, held=[True, False, False, False])
    assert torch.equal(out[:2], t[:2])
    assert abs(_dist(out[1], out[2]) - 1.4) <= 1e-12
    # the held row enters the graph at its target, not at its prediction
    targets = t.clone()
    targets[0] = torch.tensor([3.5, 2.0, 0.0], dtype=D)            # target next to piece B: rows 0, 2, 3 bonded, row 1 alone
    out = kg.guide(t, torch.zeros(4, dtype=torch.long), 2.0, 1.4, 1.0, held=torch.tensor([True, False, False, False]), targets=targets)
    assert torch.equal(out[[0, 2, 3]], t[[0, 2, 3]])
    q1 = t[1]
    d = min(_dist(q1, targets[0]), _dist(q1, t[2]), _dist(q1, t[3]))
    assert abs(d - _dist(q1, targets[0])) == 0
    assert abs(_dist(out[1], targets[0]) - 1.4) <= 1e-12


def test_three_components():
    # single atoms at x = 0, 5, 12: A and B pair up, C pairs with B; every shift from the unshifted positions
    y = [[0.0, 0.0, 0.0], [5.0, 0.0, 0.0], [12.0, 0.0, 0.0]]
    out = _one(y, 2.0, 1.5, 1.0)
    want = torch.tensor([[1.75, 0.0, 0.0], [3.25, 0.0, 0.0], [9.25, 0.0, 0.0]], dtype=D)
    assert torch.allclose(out, want, rtol=0, atol=1e-12)
    info = []
    _one(y, 2.0, 1.5, 1.0, info=info)
    assert info[0]['n_comp'] == 3 and sorted(info[0]['pairs'].values()) == [(0, 1), (1, 0), (2, 1)]


def test_ties_pick_the_lowest_pair():
    # row 0 alone; rows 1 and 2 bonded and at the same distance from row 0
    y = [[0.0, 0.0, 0.0], [3.0, 0.5, 0.0], [3.0, -0.5, 0.0]]
    info = []
    out = _one(y, 2.0, 1.0, 1.0, info=info)
    assert sorted(info[0]['pairs'].values()) == [(0, 1), (1, 0)]
    t = torch.tensor(y, dtype=D)
    d = _dist(t[0], t[1])
    u = (t[1] - t[0]) / d
    assert torch.allclose(out[0], t[0] + 0.5 * (d - 1.0) * u, rtol=0, atol=1e-12)
    assert torch.allclose(out[1:], t[1:] - 0.5 * (d - 1.0) * u, rtol=0, atol=1e-12)


def test_pairs_at_exactly_the_radius_are_not_bonded():
    for dt in (torch.float64, torch.float32):
        y = torch.tensor([[1.0, 2.0, 3.0], [3.0, 2.0, 3.0]], dtype=dt)          # d = 2 exactly
        out = kg.guide(y, torch.zeros(2, dtype=torch.long), 2.0, 1.0, 1.0, dtype=dt)
        assert abs(_dist(out[0].double(), out[1].double()) - 1.0) <= 1e-6
        inside = torch.tensor([[1.0, 2.0, 3.0], [2.9990234375, 2.0, 3.0]], dtype=dt)
        assert torch.equal(kg.guide(inside, torch.zeros(2, dtype=torch.long), 2.0, 1.0, 1.0, dtype=dt), inside)


def test_a_connected_graph_is_returned_bit_for_bit():
    g = torch.Generator().manual_seed(3)
    steps = torch.randn(30, 3, generator=g, dtype=D)
    y = torch.cumsum(steps / torch.linalg.norm(steps, dim=1, keepdim=True) * 1.3, 0)       # a random walk of 1.3 A steps
    bl = torch.zeros(30, dtype=torch.long)
    for dt in (torch.float64, torch.float32):
        assert torch.equal(kg.guide(y.to(dt), bl, 1.5, 1.0, 1.0, dtype=dt), y.to(dt))
    assert int(ligand_components(y, bl, 1.5)[0]) == 1
    assert torch.equal(kg.guide(y, bl, 0.5, 0.2, 0.0), y)                      # strength 0: off


def test_graphs_are_independent_and_components_match_the_tool():
    g = torch.Generator().manual_seed(8)
    y = torch.randn(60, 3, generator=g, dtype=D) * 3
    bl = torch.arange(60) % 4
    out = kg.guide(y, bl, 1.6, 1.2, 0.7)
    info = []
    kg.guide(y, bl, 1.6, 1.2, 0.7, info=info)
    assert [r['n_comp'] for r in info] == ligand_components(y, bl, 1.6).tolist()
    for k in range(4):
        rows = (bl == k).nonzero().reshape(-1)
        alone = kg.guide(y[rows], torch.zeros(len(rows), dtype=torch.long), 1.6, 1.2, 0.7)
        assert torch.equal(alone, out[rows])


def test_the_shift_is_minus_a_quarter_lambda_times_the_pair_energy_gradient():
    g = torch.Generator().manual_seed(5)
    a = torch.randn(5, 3, generator=g, dtype=D) * 0.5
    b = torch.randn(4, 3, generator=g, dtype=D) * 0.5 + torch.tensor([6.0, 1.0, -2.0], dtype=D)
    y = torch.cat([a, b])
    rho, bl, lam, h = 2.5, 1.5, 0.8, 1e-6
    info = []
    out = kg.guide(y, torch.zeros(9, dtype=torch.long), rho, bl, lam, info=info)
    rec = info[0]
    assert rec['n_comp'] == 2
    for c, (i, j) in rec['pairs'].items():
        members = torch.from_numpy(rec['labels'] == c)
        shift = out[members] - y[members]
        assert torch.allclose(shift, shift[0].expand_as(shift), rtol=0, atol=1e-14)       # rigid
        grad = torch.zeros(3, dtype=D)
        for k in range(3):
            e = torch.zeros(3, dtype=D)
            e[k] = h
            grad[k] = (kg.pair_energy(y[i], y[j], bl, e) - kg.pair_energy(y[i], y[j], bl, -e)) / (2 * h)
        assert float(grad.abs().max()) > 0.1
        assert torch.allclose(shift[0], -0.25 * lam * grad, rtol=0, atol=1e-7)


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
def test_oracle_chains_at_strength_zero_are_the_unguided_chains(sd, mean_type):
    cfg = {'model_mean_type': mean_type}
    for label, b, path, kw in _chain_cases(sd):
        pn, vu = synth.make_tape(2, len(path), len(b['batch_ligand']))
        args = (sd, cfg, b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'],
                b['batch_ligand'], pn, vu, path)
        want = resample.sample_diffusion(*args, **kw)
        held, targets = kw.get('fixed_mask'), b['init_ligand_pos']
        for hook in (kg.hook(2.0, 1.5, 0.0, held=held, targets=targets), kg.hook(2.0, 1.5, 0.0, clash=cg.hook(2.0, 0.0))):
            got = cg.sample_diffusion(*args, guidance=hook, **kw)
            assert torch.equal(got['pos'], want['pos']) and torch.equal(got['v'], want['v']), label
            for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
                assert all(torch.equal(x, y) for x, y in zip(got[k], want[k])), (label, k)
        on = cg.sample_diffusion(*args, guidance=kg.hook(0.5, 0.3, 1.0, held=held, targets=targets), **kw)
        assert not torch.equal(on['pos'], want['pos']), label


def test_oracle_driver_at_strength_zero_is_the_unguided_driver(sd):
    b = synth.make_batch(12, 1, n_protein=40, ligand_sizes=[5])
    path = [999, 600, 700, 300, 0]
    outs = []
    for fn, kw in ((resample.sample_diffusion_ligand, {}), (cg.sample_diffusion_ligand, {'guidance': kg.hook(2.0, 1.5, 0.0)})):
        torch.manual_seed(5)
        outs.append(fn(sd, None, b['protein_pos'], b['protein_v'], 3, None, path, batch_size=2, sample_num_atoms='range', **kw)
                    + (torch.rand(1),))
    for x, y in zip(outs[0][:6], outs[1][:6]):
        assert all(np.array_equal(p, q) for p, q in zip(x, y))
    assert torch.equal(outs[0][-1], outs[1][-1])                 # the same number of draws


def test_config_and_python_refusals():
    assert check_connect_guidance(None, None, 0.0) == (None, None, 0.0)
    assert check_connect_guidance(3.0, 5.0, 0) == (None, None, 0.0)          # radius and length ignored when off
    assert check_connect_guidance(2, 1, 1) == (2.0, 1.0, 1.0)
    assert sample_connect_guidance(Config()) == (None, None, 0.0)
    assert sample_connect_guidance(Config(connect_radius=2.0, connect_length=1.5, connect_strength=0.5)) == (2.0, 1.5, 0.5)
    nan, inf = float('nan'), float('inf')
    for r, b, s, msg in ((2.0, 1.5, -1.0, 'finite and >= 0'), (2.0, 1.5, nan, 'finite and >= 0'), (2.0, 1.5, inf, 'finite and >= 0'),
                         (2.0, 1.5, True, 'must be a number'), (2.0, 1.5, '1', 'must be a number'),
                         (None, 1.5, 1.0, 'needs a connect_radius'), (2.0, None, 1.0, 'needs a connect_length'),
                         (0.0, 1.5, 1.0, 'connect_radius must be a finite number > 0'), (nan, 1.5, 1.0, 'connect_radius must be'),
                         (2.0, 0.0, 1.0, 'connect_length must be a finite number > 0'), (2.0, -1.0, 1.0, 'connect_length must be'),
                         (2.0, 2.0, 1.0, 'below connect_radius'), (2.0, 3.0, 1.0, 'below connect_radius')):
        with pytest.raises(ValueError, match=msg):
            check_connect_guidance(r, b, s)
        with pytest.raises(ValueError, match=msg):
            sample_connect_guidance(Config(connect_radius=r, connect_length=b, connect_strength=s))


def test_python_entry_points_refuse_before_touching_the_engine():
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.sampling import sample_diffusion_ligand
    from targetdiff_b200.score_model import ScorePosNet3D
    m = ScorePosNet3D(default_model_config(), 27, 13)
    z = torch.zeros
    with pytest.raises(ValueError, match='needs a connect_length'):
        m.sample_diffusion(z(3, 3), z(3, 27), z(3, dtype=torch.long), z(1, 3), z(1, dtype=torch.long), z(1, dtype=torch.long), num_steps=2,
                           connect_radius=2.0, connect_strength=1.0)
    with pytest.raises(ValueError, match='below connect_radius'):
        sample_diffusion_ligand(m, None, 1, connect_radius=1.0, connect_length=1.5, connect_strength=1.0)


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
        for bad, msg in ((dict(connect_strength=1.0, connect_length=1.5), 'needs a connect_radius'),
                         (dict(connect_strength=-1.0, connect_radius=2.0, connect_length=1.5), '>= 0'),
                         (dict(connect_strength=1.0, connect_radius=2.0, connect_length=2.5), 'below connect_radius')):
            cmd[1] = _conf(tmp_path, **bad)
            with pytest.raises(ValueError, match=msg):
                main(cmd)


def test_result_field_only_when_guidance_is_on():
    assert add_connect_guidance({'a': 1}, None, None, 0.0) == {'a': 1}
    assert add_connect_guidance({'a': 1}, 2.0, 1.5, 0.5) == {'a': 1, 'connect_guidance': {'radius': 2.0, 'length': 1.5, 'strength': 0.5}}
