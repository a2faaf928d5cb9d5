"""Fixed atoms (fragment-conditioned sampling, DESIGN.md section 1) on the engine (run with -m gpu; `pytest -s` prints the errors).

A. Against the CPU oracle (oracle.fixed_atoms.sample_diffusion) on a noise tape plus a fixed-atom tape, with the
   chain tolerances of the other GPU tests: ragged batches at T = 20 through t = 0, the first 50 steps of T = 1000, and pos_only,
   model_mean_type 'noise', time_emb 'simple', cutoff_mode 'hybrid', num_blocks 2, k = 48.
B. The fixed rows do not depend on the network: over a full 1000-step chain they are the fp32 closed form of the forward process
   within a few ulps at every step, and end at the given lab-frame positions (one ulp) and classes (exactly).
C. A seeded chain equals the same chain on philox.engine_tape + fixed_atoms.fixed_tape.
D. Bit identity: a reordered batch and single graphs; an all-false mask and a cleared set equal a chain that never set one; one
   extra launch per chain and none per step.
E. Refusals."""
import ctypes
import math

import pytest
import torch

from oracle import fixed_atoms, philox, restate, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K = synth.LIGAND_NUM_CLASSES
EPS32 = 2.0 ** -23
POS_RTOL, POS_ATOL, LOGIT_ATOL = 1e-4, 1e-5, 1e-3
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')


def _model(cfg=None, weight_seed=0):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg))
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ARGS)


def _mask(b, lead=3):
    """The first `lead` atoms of every graph and the last atom of every other graph."""
    bl = b['batch_ligand']
    first = torch.cat([torch.zeros(1, dtype=torch.long), (bl[1:] != bl[:-1]).nonzero().view(-1) + 1])
    m = torch.zeros(len(bl), dtype=torch.bool)
    for g, f in enumerate(first.tolist()):
        n = int((bl == g).sum())
        m[f:f + min(lead, n - 1)] = True
        if g % 2:
            m[f + n - 1] = True
    return m


def _fixed_tape(seed, S, n):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(S + 1, n, 3, generator=g), torch.rand(S + 1, n, K, generator=g)


def _sample(model, b, S, mask=None, ft=None, tape=None, **kw):
    r = model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', noise_tape=tape, stack_traj=True,
                               fixed_mask=None if mask is None else mask.to(DEV), fixed_noise_tape=ft, **kw)
    return {k: (r[k].cpu() if torch.is_tensor(r[k]) else r[k]) for k in TRAJ}


# ------------------------------------------------------------------------------------------------ A. against the oracle
PARITY_CASES = {
    'T20': (dict(num_diffusion_timesteps=20), 20, [9, 14, 5], 40, False),
    'T1000_first_50': ({}, 50, [7, 11], 40, False),
    'pos_only': (dict(num_diffusion_timesteps=20), 20, [9, 6], 40, True),
    'noise_mean': (dict(num_diffusion_timesteps=20, model_mean_type='noise'), 20, [9, 6], 40, False),
    'time_emb_simple': (dict(num_diffusion_timesteps=20, time_emb_dim=1, time_emb_mode='simple'), 20, [9, 6], 40, False),
    'hybrid': (dict(num_diffusion_timesteps=20, cutoff_mode='hybrid'), 20, [9, 6], 40, False),
    'num_blocks_2': (dict(num_diffusion_timesteps=20, num_blocks=2), 20, [9, 6], 40, False),
    'k48': (dict(num_diffusion_timesteps=20, knn=48), 20, [9, 6], 60, False),
}


@pytest.mark.parametrize('name', list(PARITY_CASES))
def test_chain_with_fixed_atoms_vs_oracle(name):
    torch.set_num_threads(16)
    cfg, S, sizes, n_protein, pos_only = PARITY_CASES[name]
    model, sd = _model(cfg)
    b = synth.make_batch(61, len(sizes), n_protein=n_protein, ligand_sizes=sizes)
    n = len(b['batch_ligand'])
    pn, vu = synth.make_tape(62, S, n)
    ft = _fixed_tape(63, S, n)
    mask = _mask(b)
    want = fixed_atoms.sample_diffusion(sd, cfg, *_args(b, 'cpu'), pn, vu, mask, ft, num_steps=S, pos_only=pos_only)
    got = _sample(model, b, S, mask, ft, (pn, vu), pos_only=pos_only)
    first_bad = (got['v_traj'] != torch.stack(want['v_traj'])).any(1).nonzero()
    assert len(first_bad) == 0, 'atom types diverge from the oracle at step %d' % int(first_bad[0])
    torch.testing.assert_close(got['pos_traj'], torch.stack(want['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['pos'], want['pos'], rtol=POS_RTOL, atol=POS_ATOL)
    if not pos_only:
        torch.testing.assert_close(got['v0_traj'], torch.stack(want['v0_traj']), rtol=0, atol=LOGIT_ATOL)
        torch.testing.assert_close(got['vt_traj'], torch.stack(want['vt_traj']), rtol=0, atol=LOGIT_ATOL)
    if S == sd['betas'].shape[0]:
        assert torch.equal(got['v'][mask], b['init_ligand_v'][mask])


# ------------------------------------------------------------------------------------------------ B. independent of the network
def test_fixed_rows_follow_the_closed_form_over_1000_steps():
    model, sd = _model()
    T = sd['betas'].shape[0]
    b = synth.make_batch(71, 3, n_protein=50, ligand_sizes=[10, 21, 8])
    n = len(b['batch_ligand'])
    pn, vu = synth.make_tape(72, T, n)
    ft = _fixed_tape(73, T, n)
    mask = _mask(b, lead=4)
    got = _sample(model, b, T, mask, ft, (pn, vu))
    _, x0c, off = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    x0c, off, v0 = x0c[mask], off[b['batch_ligand'][mask]], b['init_ligand_v'][mask]
    worst, exempt, flips = 0.0, 0, 0
    for s in range(T - 1):
        tm = T - 2 - s
        eps, u = ft[0][s + 1][mask], ft[1][s + 1][mask]
        ac = sd['alphas_cumprod'][tm]
        x = ac.sqrt() * x0c + (1.0 - ac).sqrt() * eps + off                                 # fp32, as the kernel
        scale = x.double().abs() + off.double().abs() + eps.double().abs()
        worst = max(worst, float(((got['pos_traj'][s][mask].double() - x.double()).abs() / (EPS32 * scale)).max()))
        lq = restate.q_v_pred(sd, restate.index_to_log_onehot(v0, K).double(), torch.full((3,), tm), b['batch_ligand'][mask], K)
        sc = -torch.log(-torch.log(u.double() + 1e-30) + 1e-30) + lq
        top = sc.topk(2, dim=1).values
        ok = (top[:, 0] - top[:, 1]) > 1e-4
        exempt += int((~ok).sum())
        flips += int((got['v_traj'][s][mask][ok] != sc.argmax(1)[ok]).sum())
    final = got['pos'][mask].double()
    x0f = b['init_ligand_pos'][mask].double()
    final_ulps = float(((final - x0f).abs() / (EPS32 * x0f.abs())).max())
    print('fixed rows over %d steps: %.2f ulp of the fp32 closed form; %d type flips (%d exempt draws); final %.2f ulp of x0_f'
          % (T, worst, flips, exempt, final_ulps))
    assert worst <= 4.0 and flips == 0 and exempt <= 10
    assert final_ulps <= 1.0
    assert torch.equal(got['pos_traj'][-1][mask], got['pos'][mask])
    assert torch.equal(got['v'][mask], v0) and torch.equal(got['v_traj'][-1][mask], v0)


# ------------------------------------------------------------------------------------------------ C. seeded stream
@pytest.mark.parametrize('seed,S', [(123, 3), (2 ** 32 + 7, 7)])
def test_seeded_fixed_stream_is_fixed_tape(seed, S):
    model, sd = _model()
    T = sd['betas'].shape[0]
    b = synth.make_batch(31, 4, n_protein=50, ligand_sizes=[60, 45, 33, 37])         # 175 atoms: two blocks of the epilogue
    n = len(b['batch_ligand'])
    mask = _mask(b, lead=5)
    dev = _sample(model, b, S, mask, seed=seed)
    pn, vu = philox.engine_tape(seed, n, S, K)
    fpn, fvu = fixed_atoms.fixed_tape(seed, n, S, K)
    tape = _sample(model, b, S, mask, (fpn, fvu), (pn, vu))
    assert torch.equal(dev['v_traj'], tape['v_traj'])
    free = ~mask
    sigma0 = math.exp(0.5 * float(sd['posterior_logvar'][T - 1]))
    ulps, later = philox.stream_errors(dev['pos_traj'][:, free], tape['pos_traj'][:, free], pn[0][free], sigma0)
    _, _, off = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    off = off[b['batch_ligand'][mask]].double()
    p = tape['pos_traj'][:, mask].double()
    scale = p.abs() + (p - off).abs() + fpn[1:][:, mask].double().abs()
    fix_ulps = float(((dev['pos_traj'][:, mask].double() - p).abs() / (EPS32 * scale)).max())
    print('fixed stream seed=%d S=%d: free rows %.2f ulp / %.2e rel, fixed rows %.2f ulp' % (seed, S, ulps, later, fix_ulps))
    assert ulps <= philox.STREAM_ULPS and later <= philox.STREAM_LATER_REL
    assert fix_ulps <= philox.STREAM_ULPS


# ------------------------------------------------------------------------------------------------ D. bit identity, launches
def _regroup(b, order):
    parts, lig = [], []
    for i, g in enumerate(order):
        sp, sl = b['batch_protein'] == g, b['batch_ligand'] == g
        parts.append({k: (torch.full((int(s.sum()),), i, dtype=torch.long) if k.startswith('batch') else b[k][s])
                      for k, s in (('protein_pos', sp), ('protein_v', sp), ('batch_protein', sp), ('init_ligand_pos', sl),
                                   ('init_ligand_v', sl), ('batch_ligand', sl))})
        lig.append(sl.nonzero().view(-1))
    return {k: torch.cat([p[k] for p in parts]) for k in ARGS}, torch.cat(lig)


def _rows(r, idx):
    return {k: (r[k][idx] if k in ('pos', 'v') else r[k][:, idx]) for k in TRAJ}


def _differing(a, c):
    return [k for k in TRAJ if not torch.equal(a[k], c[k])]


def test_fixed_chain_is_bit_identical_reordered_and_per_graph():
    model, _ = _model()
    b = synth.make_batch(81, 4, n_protein=60, ligand_sizes=[12, 20, 7, 16])
    n, S = len(b['batch_ligand']), 6
    pn, vu = synth.make_tape(82, S, n)
    ft = _fixed_tape(83, S, n)
    mask = _mask(b)
    ref = _sample(model, b, S, mask, ft, (pn, vu))
    for order in ([2, 0, 3, 1], [1], [3]):
        bp, idx = _regroup(b, order)
        r = _sample(model, bp, S, mask[idx], (ft[0][:, idx], ft[1][:, idx]), (pn[:, idx], vu[:, idx]))
        assert not _differing(r, _rows(ref, idx)), (order, _differing(r, _rows(ref, idx)))


@pytest.mark.parametrize('tape', [False, True])
def test_empty_or_cleared_fixed_set_is_bit_identical_to_none(tape):
    from targetdiff_b200 import _lib
    model, _ = _model()
    b = synth.make_batch(91, 2, n_protein=60, ligand_sizes=[12, 9])
    n, S = len(b['batch_ligand']), 4
    kw = dict(tape=synth.make_tape(92, S, n)) if tape else dict(seed=5)
    plain = _sample(model, b, S, **kw)
    empty = _sample(model, b, S, torch.zeros(n, dtype=torch.bool), _fixed_tape(93, S, n) if tape else None, **kw)
    assert not _differing(plain, empty)
    # a set cleared through the C-ABI before the chain (sample_diffusion binds, sets, samples; here: bind, set, clear, sample)
    lib = _lib.load()
    eng = model.engine(DEV)
    st = model._stream(torch.device(DEV))
    args = _args(b)
    model._bind(eng, args[0], args[1], args[2], args[5], 1)
    lpos, lv = args[3].float().contiguous(), args[4].long().contiguous()
    _lib.check(lib.tdiff_set_ligand(eng, ctypes.c_void_p(lpos.data_ptr()), ctypes.c_void_p(lv.data_ptr()), 1, st))
    m = torch.ones(n, dtype=torch.uint8, device=DEV)
    _lib.check(lib.tdiff_set_fixed(eng, ctypes.c_void_p(m.data_ptr()), ctypes.c_void_p(lpos.data_ptr()), ctypes.c_void_p(lv.data_ptr()), 1, st))
    _lib.check(lib.tdiff_set_fixed(eng, None, None, None, 0, st))
    pos_traj = torch.empty(S, n, 3, device=DEV)
    v_traj = torch.empty(S, n, dtype=torch.int64, device=DEV)
    v0 = torch.empty(S, n, K, device=DEV)
    vt = torch.empty(S, n, K, device=DEV)
    tp = tuple(t.to(DEV).contiguous() for t in kw['tape']) if tape else (None, None)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(lib.tdiff_sample(eng, S, ptr(tp[0]), ptr(tp[1]), ctypes.c_uint64(kw.get('seed', 0)), ptr(pos_traj), ptr(v_traj), ptr(v0),
                                ptr(vt), 0, st))
    torch.cuda.synchronize()
    assert torch.equal(pos_traj.cpu(), plain['pos_traj']) and torch.equal(v_traj.cpu(), plain['v_traj'])
    assert torch.equal(v0.cpu(), plain['v0_traj']) and torch.equal(vt.cpu(), plain['vt_traj'])


def test_launches_one_per_chain_none_per_step():
    from targetdiff_b200 import _lib
    lib = _lib.load()
    b = synth.make_batch(6, 2, n_protein=150, ligand_sizes=[20, 7])
    mask = _mask(b)
    counts = {}
    for fixed in (False, True):
        for S in (3, 5):
            model, _ = _model(weight_seed=3)
            model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', return_traj=False,
                                   fixed_mask=mask.to(DEV) if fixed else None)
            counts[fixed, S] = lib.tdiff_launch_count(model.engine(DEV))
            model._drop_engine()
    per_step = (counts[False, 5] - counts[False, 3]) // 2
    print('launches per step %d; a chain with fixed atoms adds %d (set_fixed + the initial noising)' % (per_step, counts[True, 3] - counts[False, 3]))
    assert (counts[True, 5] - counts[True, 3]) // 2 == per_step
    assert counts[True, 3] - counts[False, 3] == 2 and counts[True, 5] - counts[False, 5] == 2


# ------------------------------------------------------------------------------------------------ E. refusals
def test_refusals():
    from targetdiff_b200 import _lib
    model, _ = _model()
    lib = _lib.load()
    eng = model.engine(DEV)
    st = model._stream(torch.device(DEV))
    with pytest.raises(_lib.TdiffError, match='before bind_batch'):
        _lib.check(lib.tdiff_set_fixed(eng, None, None, None, 0, st))
    with pytest.raises(_lib.TdiffError, match='before bind_batch'):
        _lib.check(lib.tdiff_set_fixed_tape(eng, None, None))
    b = synth.make_batch(95, 2, n_protein=60, ligand_sizes=[8, 5])
    n, S = len(b['batch_ligand']), 3
    with pytest.raises(ValueError, match='one entry per ligand atom'):
        _sample(model, b, S, torch.zeros(n + 1, dtype=torch.bool), seed=1)
    tape = synth.make_tape(96, S, n)
    with pytest.raises(_lib.TdiffError, match='fixed-atom tape'):
        _sample(model, b, S, _mask(b), None, tape)
    with pytest.raises(_lib.TdiffError, match='no noise tape'):
        _sample(model, b, S, _mask(b), _fixed_tape(97, S, n), None, seed=1)
    with pytest.raises(ValueError, match=r'\[S\+1,Nl,3\]'):
        _sample(model, b, S, _mask(b), _fixed_tape(97, S - 1, n), tape)
    with pytest.raises(ValueError, match='without fixed_mask'):
        _sample(model, b, S, None, _fixed_tape(97, S, n), tape)
    # a class >= K at a masked row (the Python path validates the rows through set_ligand first: call the C-ABI directly)
    args = _args(b)
    model._bind(eng, args[0], args[1], args[2], args[5], 1)
    lpos = args[3].float().contiguous()
    bad_v = args[4].long().clone()
    bad_v[1] = K
    m = torch.zeros(n, dtype=torch.uint8, device=DEV)
    m[1] = 1
    with pytest.raises(_lib.TdiffError, match='class index'):
        _lib.check(lib.tdiff_set_fixed(eng, ctypes.c_void_p(m.data_ptr()), ctypes.c_void_p(lpos.data_ptr()), ctypes.c_void_p(bad_v.data_ptr()), 1, st))
    m[1] = 0                                    # the same class at an unmasked row is not read
    _lib.check(lib.tdiff_set_fixed(eng, ctypes.c_void_p(m.data_ptr()), ctypes.c_void_p(lpos.data_ptr()), ctypes.c_void_p(bad_v.data_ptr()), 1, st))


def test_driver_end_to_end_fragment():
    """sample_diffusion_ligand with a fragment: every sample starts with the fragment, at the given positions and classes."""
    from targetdiff_b200.data import ProteinLigandData
    from targetdiff_b200.sampling import sample_diffusion_ligand
    model, _ = _model({'num_diffusion_timesteps': 20})
    b = synth.make_batch(99, 1, n_protein=60, ligand_sizes=[1])
    data = ProteinLigandData(protein_pos=b['protein_pos'], protein_atom_feature=b['protein_v'])
    ctr = b['protein_pos'].mean(0)
    frag = (ctr + torch.randn(3, 3, generator=torch.Generator().manual_seed(1)), torch.tensor([1, 2, 3]))
    for rng in ('device', 'cpu'):
        torch.manual_seed(0)
        out = sample_diffusion_ligand(model, data, 5, batch_size=5, device=DEV, sample_num_atoms='range', rng=rng, fixed_ligand=frag)
        assert [len(p) for p in out[0]] == [4, 4, 4, 4, 5]
        for pos, v in zip(out[0], out[1]):
            assert torch.allclose(torch.from_numpy(pos[:3]).float(), frag[0], rtol=EPS32, atol=0)
            assert v[:3].tolist() == [1, 2, 3]
