"""Connectivity guidance (DESIGN.md section 1) on the engine (run with -m gpu; `pytest -s` prints the numbers).

A. Off is the old chain: never set, set to 0, set then cleared give a fresh handle's bits and launches; on adds one launch per
   denoising step, two with clash guidance as well.
B. With a bond radius of 10^4 A every ligand is one piece, and the guided chain is the unguided chain bit for bit, under both mean types.
C. Controlled geometry: with every h2x xv_func's last Linear zeroed, x0 = x_t; a start at t0 = 0 with a zero start tape is the single
   decoder step, whose output is c0[0] * y_hat + ct[0] * x_t (held rows: their targets).
D. Guided chains against oracle.connect_guidance on tapes: default, respaced, 'noise', hybrid cutoff, fragment, start with kept atoms, a
   RePaint time path, and clash guidance first.
E. Batch independence (alone, reordered) and the switches (graph replay, cone, k-NN, slot keep, ligand-free cache), bit for bit.
F. The CLI writes the field; C-ABI refusals keep the setting; it survives a bind; tdiff_forward and tdiff_likelihood_terms ignore it.
G. The mechanism acts on synthetic weights: fewer disconnected final molecules with lambda = 1 than with 0.
H. Every guided step against float64: y_hat in float64 from the engine's own fp32 network output, then the step in float64.
I. The rng='cpu' driver on the 1h36 pocket against oracle.clash_guidance's driver with the connectivity hook."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import clash_guidance as cg
from oracle import connect_guidance as kg
from oracle import respaced, restate, stepwise, synth
from targetdiff_b200.sampling import resampled_time_path, respaced_time_seq

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K13 = synth.LIGAND_NUM_CLASSES
POS_RTOL, POS_ATOL, LOGIT_ATOL = 1e-4, 1e-5, 1e-3
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')
PDB_1H36 = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', '1h36_pocket10.pdb')
RHO, BOND, LAM = 1.6, 1.2, 0.5          # chains: synthetic predictions fall apart into several pieces at this radius


def _model(cfg=None, weight_seed=0, zero_xv=False):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K13)
    sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg))
    if zero_xv:                        # the last Linear of every xv_func: the position update is exactly 0
        for k in [k for k in sd if '.h2x_layers.' in k and '.xv_func.net.3.' in k]:
            sd[k] = torch.zeros_like(sd[k])
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ARGS)


def _sample(model, b, mode='protein', **kw):
    r = model.sample_diffusion(*_args(b), center_pos_mode=mode, stack_traj=True, **kw)
    return {k: (r[k].cpu() if torch.is_tensor(r[k]) else r[k]) for k in TRAJ}


def _differing(a, c):
    return [k for k in TRAJ if not (a[k] is None and c[k] is None) and not torch.equal(a[k], c[k])]


def _origin_batch(seed, sizes, n_protein=40):
    b = synth.make_batch(seed, len(sizes), n_protein=n_protein, ligand_sizes=sizes, distinct_pockets=1)
    shift = b['protein_pos'].mean(0, keepdim=True)
    b['protein_pos'], b['init_ligand_pos'] = b['protein_pos'] - shift, b['init_ligand_pos'] - shift
    return b


def _mask(b, lead=3):
    m = torch.zeros(len(b['batch_ligand']), dtype=torch.bool)
    start = 0
    for n in torch.bincount(b['batch_ligand']).tolist():
        m[start:start + min(lead, n - 1)] = True
        start += n
    return m


def _kw(rho=RHO, bond=BOND, lam=LAM):
    return dict(connect_radius=rho, connect_length=bond, connect_strength=lam)


# ------------------------------------------------------------------------------------------------ A. off, launches
def test_off_is_the_old_chain_and_launch_counts():
    from targetdiff_b200 import _lib
    lib = _lib.load()
    b = synth.make_batch(6, 3, n_protein=150, ligand_sizes=[20, 7, 12])
    seq = [999, 700, 500, 200, 0]
    path = [999, 700, 800, 500, 200, 400, 0]                  # 5 denoising, 2 re-noising steps

    def run(model, **kw):
        eng = model.engine(DEV)
        before = lib.tdiff_launch_count(eng)
        r = _sample(model, b, seed=9, **kw)
        return r, lib.tdiff_launch_count(eng) - before

    model, _ = _model(weight_seed=3)
    base, n_base = run(model, time_seq=seq)
    base_p, n_base_p = run(model, time_path=path)
    model._drop_engine()
    model, _ = _model(weight_seed=3)
    off, n_off = run(model, time_seq=seq, connect_radius=2.0, connect_length=1.5, connect_strength=0.0)
    assert not _differing(base, off) and n_off == n_base
    on, n_on = run(model, time_seq=seq, **_kw())
    assert _differing(base, on) and n_on == n_base + len(seq)
    both, n_both = run(model, time_seq=seq, clash_radius=2.5, clash_strength=1.0, **_kw())
    assert n_both == n_base + 2 * len(seq)
    cleared, n_cleared = run(model, time_seq=seq)             # sample_diffusion sets the handle's guidance on every call
    assert not _differing(base, cleared) and n_cleared == n_base
    on_p, n_on_p = run(model, time_path=path, **_kw())
    assert n_on_p == n_base_p + 5
    off_p, n_off_p = run(model, time_path=path)
    assert not _differing(base_p, off_p) and n_off_p == n_base_p
    print('launches: seq %d, guided %d, with clash guidance %d; path %d, guided %d' % (n_base, n_on, n_both, n_base_p, n_on_p))
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ B. one piece
@pytest.mark.parametrize('mean_type', ['C0', 'noise'])
def test_one_component_is_the_unguided_chain(mean_type):
    cfg = {'model_mean_type': mean_type}
    b = synth.make_batch(8, 3, n_protein=120, ligand_sizes=[10, 18, 6])
    model, _ = _model(cfg)
    seq = respaced_time_seq(1000, 12)
    base = _sample(model, b, time_seq=seq, seed=4)
    wide = _sample(model, b, time_seq=seq, seed=4, **_kw(1e4, 1.5, 1.0))
    assert not _differing(base, wide)
    full = _sample(model, b, seed=4, num_steps=20)
    wide = _sample(model, b, seed=4, num_steps=20, **_kw(1e4, 1.5, 3.0))
    assert not _differing(full, wide)
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ C. controlled geometry
def _decoder_step(model, sd, lig, rho, bond, lam, held=None):
    """One graph: ligand `lig` [Nl,3] (fp32, frame 'none') and three far protein atoms; the chain from a start at t0 = 0 with a zero
    start tape and a zero step tape; `held` [Nl] bool: kept rows (their targets are `lig`).  Returns (output positions, x_t = the start
    draw, c0[0], ct[0])."""
    n = len(lig)
    prot = torch.tensor([[200.0, 0.0, 0.0], [0.0, 200.0, 0.0], [0.0, 0.0, 200.0]])
    b = {'protein_pos': prot, 'protein_v': torch.zeros(3, synth.PROTEIN_FEATURE_DIM), 'batch_protein': torch.zeros(3, dtype=torch.long),
         'init_ligand_pos': lig, 'init_ligand_v': torch.zeros(n, dtype=torch.long), 'batch_ligand': torch.zeros(n, dtype=torch.long)}
    b['protein_v'][:, 0] = 1.0
    z3, zk = torch.zeros(n, 3), torch.zeros(n, K13)
    kw = {}
    if held is not None:
        kw = dict(fixed_mask=held.to(DEV), fixed_noise_tape=(torch.zeros(2, n, 3), torch.zeros(2, n, K13)))
    r = model.sample_diffusion(*_args(b), center_pos_mode='none', start_time=0, start_noise_tape=(z3, zk), noise_tape=(z3[None], zk[None]),
                               connect_radius=rho if lam else None, connect_length=bond if lam else None, connect_strength=lam,
                               pos_only=True, **kw)
    sa = np.sqrt(np.float32(sd['alphas_cumprod'][0].item()), dtype=np.float32)
    xt = torch.from_numpy(np.float32(sa) * lig.numpy().astype(np.float32))
    return r['pos'].cpu(), xt, float(sd['posterior_mean_c0_coef'][0]), float(sd['posterior_mean_ct_coef'][0])


def _pieces(g, centres, per=6, spread=0.5):
    return torch.cat([torch.tensor(c, dtype=torch.float32) + torch.randn(per, 3, generator=g) * spread for c in centres])


def test_controlled_geometry():
    model, sd = _model(zero_xv=True)
    g = torch.Generator().manual_seed(7)
    rho, bond = 2.0, 1.5
    # two free pieces: with lambda = 1 their closest pair ends at the bond length; every decision is the float32 oracle's
    lig = _pieces(g, [[0.0, 0.0, 0.0], [5.0, 1.0, -1.0]], spread=0.3)
    bl = torch.zeros(len(lig), dtype=torch.long)
    off, xt, c0, ct = _decoder_step(model, sd, lig, rho, bond, 0.0)
    on, _, _, _ = _decoder_step(model, sd, lig, rho, bond, 1.0)
    info = []
    want = kg.guide(xt, bl, rho, bond, 1.0, dtype=torch.float32, info=info)
    assert info[0]['n_comp'] == 2
    y_hat = (on.double() - ct * xt.double()) / c0
    (i, j), = [p for p in info[0]['pairs'].values()][:1]
    gap = float(torch.linalg.norm(y_hat[i] - y_hat[j]))
    print('two pieces: closest pair ends at %.7f for b = %.1f' % (gap, bond))
    assert abs(gap - bond) <= 2e-5
    assert float((y_hat - want.double()).abs().max()) <= 2e-5
    # a connected molecule keeps its prediction bit for bit
    conn = torch.cumsum(torch.full((12, 3), 0.6), 0)
    off_c, _, _, _ = _decoder_step(model, sd, conn, rho, bond, 0.0)
    on_c, _, _, _ = _decoder_step(model, sd, conn, rho, bond, 1.0)
    assert torch.equal(on_c, off_c)
    # held anchoring: kept rows of the first piece stay at their targets, and the free piece takes the full step towards them
    held = torch.zeros(len(lig), dtype=torch.bool)
    held[:3] = True
    onh, xth, _, _ = _decoder_step(model, sd, lig, rho, bond, 1.0, held=held)
    assert torch.equal(onh[:3], lig[:3])
    info = []
    wanth = kg.guide(xth, bl, rho, bond, 1.0, held=held, targets=lig, dtype=torch.float32, info=info)
    y_h = (onh.double() - ct * xth.double()) / c0
    q = xth.double().clone()
    q[:3] = lig[:3].double()
    moved = [c for c in range(info[0]['n_comp']) if c in info[0]['pairs']]
    for c in moved:
        i, j = info[0]['pairs'][c]
        gap = float(torch.linalg.norm(y_h[i] - q[j]))
        print('held anchor: free piece %d ends %.7f from its partner (partner held: %s)' % (c, gap, bool(held[j])))
        if held[j]:
            assert abs(gap - bond) <= 2e-5
    free = ~held
    assert float((y_h[free] - wanth.double()[free]).abs().max()) <= 2e-5
    # 1024 ligand atoms in one graph: 64 pieces of 16 atoms on a 4 x 4 x 4 lattice; 1025 is refused
    centres = [[6.0 * a, 6.0 * b_, 6.0 * c] for a in range(4) for b_ in range(4) for c in range(4)]
    big = _pieces(g, centres, per=16, spread=0.4)
    onb, xtb, _, _ = _decoder_step(model, sd, big, rho, bond, 1.0)
    info = []
    wantb = kg.guide(xtb, torch.zeros(1024, dtype=torch.long), rho, bond, 1.0, dtype=torch.float32, info=info)
    yb = (onb.double() - ct * xtb.double()) / c0
    err = float((yb - wantb.double()).abs().max())
    print('1024 atoms: %d components, max |y_hat - float32 oracle| = %.2e' % (info[0]['n_comp'], err))
    assert info[0]['n_comp'] > 1 and err <= 5e-5
    from targetdiff_b200._lib import TdiffError
    with pytest.raises(TdiffError, match='more than 1024'):
        _decoder_step(model, sd, torch.cat([big, big[:1] + 0.1]), rho, bond, 1.0)
    off1025, _, _, _ = _decoder_step(model, sd, torch.cat([big, big[:1] + 0.1]), rho, bond, 0.0)    # off: no limit
    assert torch.isfinite(off1025).all()
    # a pair at exactly rho is not bonded: two single atoms whose drawn x differ by exactly rho (fp32) are two pieces and close to b;
    # a hair inside rho they are one molecule and keep their prediction
    sa = np.sqrt(np.float32(sd['alphas_cumprod'][0].item()), dtype=np.float32)
    x0 = np.float32(20.0)
    x1 = np.float32(22.0)
    while np.float32(sa * x1) - np.float32(sa * x0) != np.float32(rho):
        x1 = np.nextafter(x1, np.float32(30.0)) if np.float32(sa * x1) - np.float32(sa * x0) < rho else np.nextafter(x1, np.float32(0.0))
    pair = torch.tensor([[float(x0), 3.0, -2.0], [float(x1), 3.0, -2.0]])
    on2, xt2, _, _ = _decoder_step(model, sd, pair, rho, bond, 1.0)
    off2, _, _, _ = _decoder_step(model, sd, pair, rho, bond, 0.0)
    assert float(xt2[1, 0] - xt2[0, 0]) == rho
    y2 = (on2.double() - ct * xt2.double()) / c0
    assert abs(float(torch.linalg.norm(y2[1] - y2[0])) - bond) <= 2e-5 and not torch.equal(on2, off2)
    pair[1, 0] = float(np.nextafter(np.float32(pair[1, 0].item()), np.float32(0.0)))
    pair[1, 0] -= 1e-3
    on3, _, _, _ = _decoder_step(model, sd, pair, rho, bond, 1.0)
    off3, _, _, _ = _decoder_step(model, sd, pair, rho, bond, 0.0)
    assert torch.equal(on3, off3)
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ D. chains against the oracle
def _case(name, b):
    n = len(b['batch_ligand'])
    g = torch.Generator().manual_seed(63)
    ft = lambda S: (torch.randn(S + 1, n, 3, generator=g), torch.rand(S + 1, n, K13, generator=g))
    if name == 'default':
        return cg.unit_path(1000, 8), {}, {'num_steps': 8}
    if name == 'respaced':
        seq = respaced_time_seq(1000, 20)
        return seq, {}, {'time_seq': seq}
    if name == 'fragment':
        seq = respaced_time_seq(1000, 20)
        m, f = _mask(b, 4), ft(20)
        return seq, dict(fixed_mask=m, fixed_tape=f), {'time_seq': seq, 'fixed_mask': m.to(DEV), 'fixed_noise_tape': f}
    if name == 'start_keep':
        seq = respaced_time_seq(1000, 12, start=400)
        m, f = _mask(b, 3), ft(12)
        st = (torch.randn(n, 3, generator=g), torch.rand(n, K13, generator=g))
        return seq, dict(fixed_mask=m, fixed_tape=f, start_time=400, start_tape=st), \
            {'time_seq': seq, 'fixed_mask': m.to(DEV), 'fixed_noise_tape': f, 'start_time': 400, 'start_noise_tape': st}
    path = resampled_time_path(respaced_time_seq(1000, 10), resamplings=2, jump_length=3)
    m, f = _mask(b, 4), ft(len(path))
    return path, dict(fixed_mask=m, fixed_tape=f), {'time_path': path, 'fixed_mask': m.to(DEV), 'fixed_noise_tape': f}


CHAIN_CFG = {'respaced_noise': {'model_mean_type': 'noise'}, 'hybrid': {'cutoff_mode': 'hybrid'}}


@pytest.mark.parametrize('name', ['default', 'respaced', 'respaced_noise', 'hybrid', 'fragment', 'start_keep', 'path', 'with_clash'])
def test_guided_chain_vs_oracle(name):
    torch.set_num_threads(16)
    cfg = CHAIN_CFG.get(name)
    model, sd = _model(cfg)
    b = _origin_batch(61, [9, 14, 6])
    base = 'respaced' if name in CHAIN_CFG or name == 'with_clash' else name
    path, okw, ekw = _case(base, b)
    clash = dict(clash_radius=3.0, clash_strength=0.5) if name == 'with_clash' else {}
    pn, vu = synth.make_tape(62, len(path), len(b['batch_ligand']))
    got = _sample(model, b, mode='none', noise_tape=(pn, vu), **_kw(), **clash, **ekw)
    hook = kg.hook(RHO, BOND, LAM, held=okw.get('fixed_mask'), targets=b['init_ligand_pos'], clash=cg.hook(3.0, 0.5) if clash else None)
    want = cg.sample_diffusion(sd, cfg, *_args(b, 'cpu'), pn, vu, path, center_pos_mode='none', guidance=hook, **okw)
    plain = cg.sample_diffusion(sd, cfg, *_args(b, 'cpu'), pn, vu, path, center_pos_mode='none',
                                guidance=cg.hook(3.0, 0.5) if clash else None, **okw)
    first_bad = (got['v_traj'] != torch.stack(want['v_traj'])).any(1).nonzero()
    assert len(first_bad) == 0, 'atom types diverge from the oracle at step %d' % int(first_bad[0])
    torch.testing.assert_close(got['pos_traj'], torch.stack(want['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['v0_traj'], torch.stack(want['v0_traj']), rtol=0, atol=LOGIT_ATOL)
    moved = float((torch.stack(want['pos_traj']) - torch.stack(plain['pos_traj'])).abs().max())
    print('%s: %d steps, max |pos - oracle| %.2e, guidance moved the oracle chain by up to %.2f A'
          % (name, len(path), float((got['pos_traj'] - torch.stack(want['pos_traj'])).abs().max()), moved))
    assert moved > 1e-3
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ E. batch independence, switches
def test_batch_independence():
    """A cfg3-shaped batch (64 pockets x 10 samples = 640 graphs of 300 protein + 20 ligand atoms) on a tape: graph 5 alone and the
    whole batch in reversed-and-rotated graph order give each graph's guided chain the same bits."""
    model, _ = _model()
    G = 640
    b = synth.make_batch(21, G, n_protein=300, n_ligand=20, distinct_pockets=64)
    seq = respaced_time_seq(1000, 5)
    pn, vu = synth.make_tape(22, len(seq), len(b['batch_ligand']))
    kw = dict(time_seq=seq, **_kw(2.0, 1.5, 1.0))
    full = _sample(model, b, noise_tape=(pn, vu), **kw)
    prot_rows = [(b['batch_protein'] == g).nonzero().reshape(-1) for g in range(G)]
    lig_rows = [(b['batch_ligand'] == g).nonzero().reshape(-1) for g in range(G)]
    rev = list(range(G - 1, -1, -1))
    for order in ([5], rev[37:] + rev[:37]):
        pr = torch.cat([prot_rows[g] for g in order])
        lr = torch.cat([lig_rows[g] for g in order])
        sub = {'protein_pos': b['protein_pos'][pr], 'protein_v': b['protein_v'][pr], 'init_ligand_pos': b['init_ligand_pos'][lr],
               'init_ligand_v': b['init_ligand_v'][lr],
               'batch_protein': torch.repeat_interleave(torch.arange(len(order)), torch.tensor([len(prot_rows[g]) for g in order])),
               'batch_ligand': torch.repeat_interleave(torch.arange(len(order)), torch.tensor([len(lig_rows[g]) for g in order]))}
        got = _sample(model, sub, noise_tape=(pn[:, lr], vu[:, lr]), **kw)
        assert torch.equal(got['pos_traj'], full['pos_traj'][:, lr]) and torch.equal(got['v_traj'], full['v_traj'][:, lr]), len(order)
        assert torch.equal(got['pos'], full['pos'][lr])
    plain = _sample(model, b, noise_tape=(pn, vu), time_seq=seq)
    assert not torch.equal(plain['pos'], full['pos'])
    model._drop_engine()


@pytest.mark.parametrize('env', ['TDIFF_NO_GRAPH', 'TDIFF_NO_RESTRICT', 'TDIFF_KNN_FULL', 'TDIFF_NO_SLOT_KEEP', 'TDIFF_FREE_DEPTH'])
def test_switches_change_nothing(monkeypatch, env):
    b = synth.make_batch(33, 3, n_protein=120, ligand_sizes=[12, 20, 7])
    path = resampled_time_path(respaced_time_seq(1000, 8), resamplings=2, jump_length=2)
    kw = dict(time_path=path, fixed_mask=_mask(b).to(DEV), seed=77, **_kw())
    model, _ = _model()
    base = _sample(model, b, **kw)
    model._drop_engine()
    monkeypatch.setenv(env, '0' if env == 'TDIFF_FREE_DEPTH' else '1')
    other = _sample(model, b, **kw)
    model._drop_engine()
    assert not _differing(base, other)


# ------------------------------------------------------------------------------------------------ F. CLI and C-ABI
@pytest.mark.parametrize('command', ['sample_for_pocket', 'sample_pockets'])
def test_cli_writes_the_field(tmp_path, command):
    import shutil
    import yaml
    from targetdiff_b200.cli import main
    from targetdiff_b200.config import Config, default_model_config
    cfg = dict(num_diffusion_timesteps=20)
    _, sd = _model(cfg)
    mc = default_model_config()
    mc.update(cfg)
    torch.save({'config': Config(model=mc, data={'transform': {'ligand_atom_mode': 'add_aromatic'}}), 'model': sd}, tmp_path / 'ckpt.pt')
    for strength, out in ((1.0, 'on'), (0.0, 'off')):
        conf = {'model': {'checkpoint': str(tmp_path / 'ckpt.pt')},
                'sample': {'seed': 1, 'num_samples': 2, 'num_steps': 20, 'pos_only': False, 'center_pos_mode': 'protein',
                           'sample_num_atoms': 'range', 'connect_radius': 2.0, 'connect_length': 1.5, 'connect_strength': strength}}
        with open(tmp_path / 'sample.yml', 'w') as f:
            yaml.safe_dump(conf, f)
        if command == 'sample_for_pocket':
            main([command, str(tmp_path / 'sample.yml'), '--pdb_path', PDB_1H36, '--result_path', str(tmp_path / out), '--device', DEV])
            r = torch.load(tmp_path / out / 'sample.pt', weights_only=False)
        else:
            (tmp_path / 'pockets').mkdir(exist_ok=True)
            shutil.copyfile(PDB_1H36, tmp_path / 'pockets' / '1h36_pocket10.pdb')
            main([command, str(tmp_path / 'sample.yml'), '--pocket_dir', str(tmp_path / 'pockets'), '--result_path', str(tmp_path / out),
                  '--device', DEV])
            r = torch.load(tmp_path / out / 'result_0.pt', weights_only=False)
        if strength > 0:
            assert r['connect_guidance'] == {'radius': 2.0, 'length': 1.5, 'strength': 1.0}
        else:
            assert 'connect_guidance' not in r
        assert len(r['pred_ligand_pos']) == 2


def test_cabi_refusals_bind_and_forward():
    from targetdiff_b200 import _lib
    lib = _lib.load()
    model, _ = _model()
    eng = model.engine(DEV)
    f = ctypes.c_float
    nan, inf = float('nan'), float('inf')
    for r, bl, s, msg in ((2.0, 1.5, -1.0, 'strength'), (2.0, 1.5, nan, 'strength'), (2.0, 1.5, inf, 'strength'),
                          (0.0, 1.5, 1.0, 'radius'), (-2.0, 1.5, 1.0, 'radius'), (inf, 1.5, 1.0, 'radius'), (nan, 1.5, 1.0, 'radius'),
                          (2.0, 0.0, 1.0, 'bond_length'), (2.0, -1.0, 1.0, 'bond_length'), (2.0, 2.0, 1.0, 'bond_length'),
                          (2.0, 2.5, 1.0, 'bond_length'), (2.0, nan, 1.0, 'bond_length')):
        assert lib.tdiff_set_connect_guidance(eng, f(r), f(bl), f(s)) == _lib.TDIFF_EINVAL
        assert msg in lib.tdiff_last_error().decode()
    assert lib.tdiff_set_connect_guidance(None, f(2.0), f(1.5), f(1.0)) == _lib.TDIFF_EINVAL
    assert lib.tdiff_set_connect_guidance(eng, f(nan), f(nan), f(0.0)) == _lib.TDIFF_OK          # off: radius and length ignored
    # a refusal keeps the previous setting, and the setting survives a bind: drive the chain through the C-ABI
    b = synth.make_batch(95, 2, n_protein=80, ligand_sizes=[8, 5])
    a = _args(b)
    st = model._stream(torch.device(DEV))
    lpos, lv = a[3].float().contiguous(), a[4].long().contiguous()
    out = torch.empty_like(lpos)

    def chain():
        model._bind(eng, a[0], a[1], a[2], a[5], 1)
        _lib.check(lib.tdiff_set_ligand(eng, ctypes.c_void_p(lpos.data_ptr()), ctypes.c_void_p(lv.data_ptr()), 1, st))
        _lib.check(lib.tdiff_sample(eng, 10, None, None, ctypes.c_uint64(5), None, None, None, None, 0, st))
        _lib.check(lib.tdiff_get_ligand(eng, ctypes.c_void_p(out.data_ptr()), None, 1, st))
        torch.cuda.synchronize()
        return out.cpu().clone()

    plain = chain()
    _lib.check(lib.tdiff_set_connect_guidance(eng, f(RHO), f(BOND), f(1.0)))
    guided = chain()
    assert not torch.equal(plain, guided)
    assert lib.tdiff_set_connect_guidance(eng, f(RHO), f(BOND), f(-1.0)) == _lib.TDIFF_EINVAL
    assert lib.tdiff_set_connect_guidance(eng, f(RHO), f(RHO), f(1.0)) == _lib.TDIFF_EINVAL
    assert torch.equal(chain(), guided)                        # the refused calls changed nothing; the bind in chain() kept it
    # tdiff_forward and tdiff_likelihood_terms ignore the setting
    ts = torch.tensor([300, 0])
    n = len(b['batch_ligand'])
    lk_tape = (torch.randn(n, 3, generator=torch.Generator().manual_seed(8)), torch.rand(n, K13, generator=torch.Generator().manual_seed(9)))
    fw_on = model(*a)['pred_ligand_pos'].cpu()
    lk_on = {k: v.cpu() for k, v in model.likelihood_terms(*a, ts, noise=lk_tape, return_atoms=True).items()}
    _lib.check(lib.tdiff_set_connect_guidance(eng, f(0.0), f(0.0), f(0.0)))
    fw_off = model(*a)['pred_ligand_pos'].cpu()
    lk_off = {k: v.cpu() for k, v in model.likelihood_terms(*a, ts, noise=lk_tape, return_atoms=True).items()}
    assert torch.equal(fw_on, fw_off)
    assert lk_on.keys() == lk_off.keys() and all(torch.equal(lk_on[k], lk_off[k]) for k in lk_on)
    assert torch.equal(chain(), plain)
    # the ligand-atom limit is checked at chain start, against the bound batch, before anything changes
    big = synth.make_batch(96, 1, n_protein=40, ligand_sizes=[1025])
    ab = _args(big)
    model._bind(eng, ab[0], ab[1], ab[2], ab[5], 1)
    bp, bv = ab[3].float().contiguous(), ab[4].long().contiguous()
    _lib.check(lib.tdiff_set_ligand(eng, ctypes.c_void_p(bp.data_ptr()), ctypes.c_void_p(bv.data_ptr()), 1, st))
    _lib.check(lib.tdiff_set_connect_guidance(eng, f(RHO), f(BOND), f(1.0)))
    assert lib.tdiff_sample(eng, 3, None, None, ctypes.c_uint64(5), None, None, None, None, 0, st) == _lib.TDIFF_EINVAL
    assert 'more than 1024' in lib.tdiff_last_error().decode()
    _lib.check(lib.tdiff_set_connect_guidance(eng, f(0.0), f(0.0), f(0.0)))
    _lib.check(lib.tdiff_sample(eng, 3, None, None, ctypes.c_uint64(5), None, None, None, None, 0, st))
    torch.cuda.synchronize()
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ G. the mechanism acts
def test_fewer_disconnected_molecules_with_guidance():
    """A batch of 64 graphs of the cfg3 pocket and ligand sizes (about 400 protein atoms, 20-30 ligand atoms), a 100-step respaced chain
    from one seed; disconnected = a final molecule in more than one piece at rho = 2 A.  Synthetic weights: this shows that guidance
    acts, not that it improves molecules."""
    from targetdiff_b200.analyze import ligand_components
    sizes = [20 + (7 * g) % 11 for g in range(64)]
    b = synth.make_batch(41, 64, n_protein=400, ligand_sizes=sizes, distinct_pockets=8)
    model, _ = _model()
    seq = respaced_time_seq(1000, 100)
    rho, bond = 2.0, 1.5
    counts = {}
    for lam in (0.0, 1.0):
        r = _sample(model, b, time_seq=seq, seed=123, **(_kw(rho, bond, lam) if lam else {}))
        n_comp = ligand_components(r['pos'], b['batch_ligand'], rho)
        counts[lam] = (int((n_comp > 1).sum()), int(n_comp.sum()))
    print('disconnected molecules of 64 at %.1f A: lambda = 0: %d (%d pieces), lambda = 1: %d (%d pieces)'
          % (rho, counts[0.0][0], counts[0.0][1], counts[1.0][0], counts[1.0][1]))
    assert counts[1.0][0] < counts[0.0][0]
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ H. guided steps against float64
EPS32 = 2.0 ** -23
# The guidance term of the tolerance, per atom and coordinate (absolute, before the posterior's c0 factor): the engine forms q, d and the
# shift in fp32, so each carries a few ulp of the graph's largest coordinate.  GUIDE_ULPS ulp of that.
GUIDE_ULPS = 64


@pytest.mark.parametrize('mean_type,pos_only', [('C0', False), ('noise', False), ('C0', True)])
def test_every_guided_step_vs_float64(mean_type, pos_only):
    cfg = {'model_mean_type': mean_type}
    model, sd = _model(cfg)
    b = _origin_batch(71, [9, 14, 6])
    seq = [999, 800, 600, 400, 200, 100, 50, 10, 3, 1, 0]                    # jump steps, unit steps, and t = 0
    tab = respaced.jump_tables(sd, seq)
    n = len(b['batch_ligand'])
    pn, vu = synth.make_tape(72, len(seq), n)
    r = _sample(model, b, mode='none', noise_tape=(pn, vu), time_seq=seq, pos_only=pos_only, **_kw())
    args = _args(b)
    bl = b['batch_ligand']
    worst, n_moved = 0.0, 0
    for s in range(len(seq)):
        t = seq[s]
        xt = b['init_ligand_pos'] if s == 0 else r['pos_traj'][s - 1]
        vt = b['init_ligand_v'] if s == 0 else r['v_traj'][s - 1]
        out = model(args[0], args[1], args[2], xt.to(DEV), vt.to(DEV), args[5])
        x0, logits = out['pred_ligand_pos'].cpu(), out['pred_ligand_v'].cpu()
        guide64 = lambda y: kg.guide(y, bl, RHO, BOND, LAM, dtype=torch.float64)
        ref = cg.guided_jump_step(sd, cfg, tab, s, xt, vt, x0, logits, pn[s], vu[s], guide64, pos_only=pos_only, dtype=torch.float64)
        e = stepwise.errors(r['pos_traj'][s], r['v_traj'][s], None if pos_only else r['v0_traj'][s], None if pos_only else r['vt_traj'][s],
                            ref, stepwise.MARGIN)
        n_moved += int((ref['x0_hat'] != ref['x0']).any(1).sum())
        y = ref['x0']
        gmax = torch.zeros(n, dtype=torch.float64)
        for g in range(int(bl.max()) + 1):
            gmax[bl == g] = y[bl == g].abs().max()
        c0 = float(tab['c0'][s])
        g_tol = abs(c0) * GUIDE_ULPS * EPS32 * gmax
        err = (r['pos_traj'][s].double() - ref['pos']).abs()
        allowed = stepwise.STEP_TOL['pos'] * ref['scale'] + g_tol[:, None]
        ratio = float((err / allowed).max())
        worst = max(worst, ratio)
        assert e['v_diff'] == 0, (s, t, e)
        if not pos_only:
            assert e['v0'] <= stepwise.STEP_TOL['v0'] and e['vt'] <= stepwise.STEP_TOL['vt'], (s, t, e)
        assert ratio <= 1.0, (s, t, ratio)
    print('%s pos_only=%s: %d steps, %d moved atom-steps, worst position error %.3f of the allowed' % (mean_type, pos_only, len(seq),
                                                                                                    n_moved, worst))
    assert n_moved > 0
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ I. the rng='cpu' driver
def test_1h36_driver_cpu_rng_vs_oracle():
    from targetdiff_b200 import atom_num
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand, seed_all
    torch.set_num_threads(16)
    model, sd = _model()
    data = pdb_to_pocket_data(PDB_1H36)
    seq = respaced_time_seq(1000, 8)
    seed_all(2021)
    got = sample_diffusion_ligand(model, data, 2, batch_size=2, device=DEV, sample_num_atoms='prior', rng='cpu', time_seq=seq, **_kw())
    after_engine = torch.rand(1)
    seed_all(2021)
    want = cg.sample_diffusion_ligand(sd, None, data.protein_pos, data.protein_atom_feature, 2, atom_num._table(), seq, batch_size=2,
                                      guidance=kg.hook(RHO, BOND, LAM))
    assert torch.equal(torch.rand(1), after_engine)                      # the same draws, in the same number
    seed_all(2021)
    plain = cg.sample_diffusion_ligand(sd, None, data.protein_pos, data.protein_atom_feature, 2, atom_num._table(), seq, batch_size=2)
    assert [len(p) for p in got[0]] == [len(p) for p in want[0]]
    assert np.array_equal(np.concatenate(got[1]), np.concatenate(want[1]))
    assert np.array_equal(np.concatenate(got[3], axis=1), np.concatenate(want[3], axis=1))
    np.testing.assert_allclose(np.concatenate(got[2], axis=1), np.concatenate(want[2], axis=1), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(np.concatenate(got[0]), np.concatenate(want[0]), rtol=1e-4, atol=1e-4)
    moved = float(np.abs(np.concatenate(want[0]) - np.concatenate(plain[0])).max())
    print('1h36 driver: guidance moved the oracle molecules by up to %.3f A' % moved)
    assert moved > 1e-3
    model._drop_engine()
