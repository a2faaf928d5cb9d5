"""Element constraints (DESIGN.md section 1) on the engine (run with -m gpu; `pytest -s` prints the numbers).

A. Off and all-allowed are the old chain: never set, cleared, and a mask of every class give a fresh handle's bits, and no launch is
   added per step, on every chain kind.
B. The guarantee: with the type head's bias favouring a forbidden class, unconstrained chains end mostly in it and constrained chains
   never; every chain kind, 'noise', K = 8, 13, 23; a single-class set ends every free row in that class with no NaN.
C. Constrained chains against oracle.type_constraints on tapes, and every step against float64 from the engine's own fp32 outputs.
D. Batch independence (alone, reordered, next to other masks; unmasked graphs as unconstrained) and the engine switches, bit for bit.
E. C-ABI: refusals keep the mask, bind clears it, pos_only refuses it, the forward and likelihood scoring ignore it; the rng='cpu'
   driver on the 1h36 pocket against the oracle driver; both CLI commands write compliant molecules."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import clash_guidance as cg
from oracle import resample, restate, stepwise, synth
from oracle import type_constraints as tc
from targetdiff_b200.analyze import type_violations
from targetdiff_b200.sampling import resampled_time_path, respaced_time_seq

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K13 = synth.LIGAND_NUM_CLASSES
POS_RTOL, POS_ATOL, LOGIT_ATOL = 1e-4, 1e-5, 1e-3
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')
PDB_1H36 = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', '1h36_pocket10.pdb')
T20 = {'num_diffusion_timesteps': 20}


def _model(cfg=None, K=K13, weight_seed=0, favour=None):
    """Engine model on synthetic weights; `favour` = class c: the type head's last bias gets +30 at c, so the network predicts c."""
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K)
    sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg), ligand_dim=K)
    if favour is not None:
        sd['v_inference.2.bias'] = sd['v_inference.2.bias'].clone()
        sd['v_inference.2.bias'][favour] += 30.0
    m.load_state_dict(sd, strict=True)
    return m.to(DEV), sd


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ARGS)


def _sample(model, b, mode='protein', **kw):
    r = model.sample_diffusion(*_args(b), center_pos_mode=mode, stack_traj=True, **kw)
    return {k: (r[k].cpu() if torch.is_tensor(r[k]) else r[k]) for k in TRAJ}


def _differing(a, c):
    return [k for k in TRAJ if not (a[k] is None and c[k] is None) and not torch.equal(a[k], c[k])]


def _origin_batch(seed, sizes, n_protein=40, K=K13):
    b = synth.make_batch(seed, len(sizes), n_protein=n_protein, ligand_sizes=sizes, distinct_pockets=1, num_classes=K)
    shift = b['protein_pos'].mean(0, keepdim=True)
    b['protein_pos'], b['init_ligand_pos'] = b['protein_pos'] - shift, b['init_ligand_pos'] - shift
    return b


def _lead(b, lead=3):
    m = torch.zeros(len(b['batch_ligand']), dtype=torch.bool)
    start = 0
    for n in torch.bincount(b['batch_ligand']).tolist():
        m[start:start + min(lead, n - 1)] = True
        start += n
    return m


def _random_mask(n, K, seed, p=0.4):
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(n, K, generator=g) < p
    m[torch.arange(n), torch.randint(0, K, (n,), generator=g)] = True          # no row empty
    return m


KINDS = ['default', 'respaced', 'fragment', 'start_keep', 'path', 'guided']


def _case(name, b, T, K=K13, seed=63, tapes=True):
    """(time path for the oracle, oracle kwargs, engine kwargs, fixed rows or None) of a chain kind; every kind ends at t = 0.  With
    tapes=False the engine kwargs carry no fixed or start tape (a chain on the device stream)."""
    out = _case_with_tapes(name, b, T, K, seed)
    if not tapes:
        for k in ('fixed_noise_tape', 'start_noise_tape'):
            out[2].pop(k, None)
    return out


def _case_with_tapes(name, b, T, K, seed):
    n = len(b['batch_ligand'])
    g = torch.Generator().manual_seed(seed)
    ft = lambda S: (torch.randn(S + 1, n, 3, generator=g), torch.rand(S + 1, n, K, generator=g))
    if name == 'default':
        return cg.unit_path(T), {}, {'num_steps': T}, None
    seq = respaced_time_seq(T, min(T, 12))
    if name in ('respaced', 'guided'):
        kw = {'time_seq': seq}
        okw = {}
        if name == 'guided':
            kw.update(clash_radius=3.0, clash_strength=0.5)
            okw['guidance'] = cg.hook(3.0, 0.5)
        return seq, okw, kw, None
    if name == 'fragment':
        m, f = _lead(b, 4), ft(len(seq))
        return seq, dict(fixed_mask=m, fixed_tape=f), {'time_seq': seq, 'fixed_mask': m.to(DEV), 'fixed_noise_tape': f}, m
    if name == 'start_keep':
        t0 = T // 2
        sseq = respaced_time_seq(T, min(t0 + 1, 8), start=t0)
        m, f = _lead(b, 3), ft(len(sseq))
        st = (torch.randn(n, 3, generator=g), torch.rand(n, K, generator=g))
        return sseq, dict(fixed_mask=m, fixed_tape=f, start_time=t0, start_tape=st), \
            {'time_seq': sseq, 'fixed_mask': m.to(DEV), 'fixed_noise_tape': f, 'start_time': t0, 'start_noise_tape': st}, m
    path = resampled_time_path(respaced_time_seq(T, min(T, 10)), resamplings=2, jump_length=3)
    m, f = _lead(b, 4), ft(len(path))
    return path, dict(fixed_mask=m, fixed_tape=f), {'time_path': path, 'fixed_mask': m.to(DEV), 'fixed_noise_tape': f}, m


# ------------------------------------------------------------------------------------------------ A. off and all-allowed
@pytest.mark.parametrize('name', KINDS)
def test_off_and_all_allowed_are_the_old_chain(name):
    from targetdiff_b200 import _lib
    lib = _lib.load()
    b = synth.make_batch(6, 3, n_protein=150, ligand_sizes=[20, 7, 12])
    n = len(b['batch_ligand'])

    def run(model, **kw):
        eng = model.engine(DEV)
        before = lib.tdiff_launch_count(eng)
        r = _sample(model, b, seed=9, **kw)
        return r, lib.tdiff_launch_count(eng) - before

    model, _ = _model(T20)
    _, _, ekw, _ = _case(name, b, 20, tapes=False)
    base, n_base = run(model, **ekw)
    model._drop_engine()
    model, _ = _model(T20)
    full, n_full = run(model, allowed_types=torch.ones(n, K13, dtype=torch.bool, device=DEV), **ekw)
    assert not _differing(base, full), name
    assert n_full == n_base + 1                                  # the mask's check launch; none per step
    few = _random_mask(n, K13, 3)
    on, n_on = run(model, allowed_types=few.to(DEV), **ekw)
    assert _differing(base, on) and n_on == n_base + 1
    cleared, n_cleared = run(model, **ekw)                       # sample_diffusion sets or clears the mask on every call
    assert not _differing(base, cleared) and n_cleared == n_base
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ B. the guarantee
def _free_violations(r, allowed, fixed):
    free = torch.ones(len(r['v']), dtype=torch.bool) if fixed is None else ~fixed
    return type_violations(r['v'][free], allowed[free]), int(free.sum())


@pytest.mark.parametrize('name,cfg,K', [(k, None, K13) for k in KINDS] + [('respaced', {'model_mean_type': 'noise'}, K13),
                                        ('respaced', None, 8), ('respaced', None, 23), ('path', None, 23), ('default', None, 8)])
def test_forbidden_class_never_ends_a_chain(name, cfg, K):
    c = 3 if K == 8 else 7
    cfg = dict(T20 if name == 'default' else {}, **(cfg or {}))
    T = restate.make_schedules(cfg)['betas'].shape[0]
    model, _ = _model(cfg, K=K, favour=c)
    b = synth.make_batch(8, 4, n_protein=120, ligand_sizes=[10, 18, 6, 15], num_classes=K)
    n = len(b['batch_ligand'])
    _, _, ekw, fixed = _case(name, b, T, K, tapes=False)
    allowed = torch.ones(n, K, dtype=torch.bool)
    allowed[:, c] = False
    if fixed is not None:
        allowed[fixed] = True
    plain = _sample(model, b, seed=4, **ekw)
    con = _sample(model, b, seed=4, allowed_types=allowed.to(DEV), **ekw)
    n_plain, n_free = _free_violations(plain, allowed, fixed)
    n_con, _ = _free_violations(con, allowed, fixed)
    print('%s K=%d cfg=%s: free atoms in the favoured class %d of %d unconstrained, %d constrained'
          % (name, K, cfg, n_plain, n_free, n_con))
    assert n_plain > n_free // 2
    assert n_con == 0
    assert not any(torch.isnan(con[k]).any() for k in ('pos_traj', 'v0_traj', 'vt_traj', 'pos'))
    if fixed is not None:
        assert torch.equal(con['v'][fixed], plain['v'][fixed])
    model._drop_engine()


def test_single_class_set():
    model, _ = _model(favour=7)
    b = synth.make_batch(9, 3, n_protein=100, ligand_sizes=[9, 14, 5])
    n = len(b['batch_ligand'])
    seq = respaced_time_seq(1000, 15)
    allowed = torch.zeros(n, K13, dtype=torch.bool)
    allowed[:, 4] = True
    r = _sample(model, b, seed=2, time_seq=seq, allowed_types=allowed.to(DEV))
    assert bool((r['v'] == 4).all())
    want = torch.full((len(seq), n, K13), float('-inf'))
    want[:, :, 4] = 0.0
    assert torch.equal(r['v0_traj'], want)
    assert torch.equal(r['vt_traj'][-1], want[-1])               # the decoder step's distribution: all mass on class 4
    assert not any(torch.isnan(r[k]).any() for k in ('pos_traj', 'v0_traj', 'vt_traj', 'pos'))
    assert bool(torch.isfinite(r['vt_traj'][:-1]).all())          # intermediate steps keep mass on every class
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ C. against the oracle
def _check_logs(got, want, allowed_rows):
    """log-probabilities [S,n,K]: -inf exactly where the oracle has -inf, within LOGIT_ATOL elsewhere."""
    ninf = torch.isneginf(want)
    assert torch.equal(torch.isneginf(got), ninf)
    assert not torch.isnan(got).any()
    assert float((got[~ninf] - want[~ninf]).abs().max()) <= LOGIT_ATOL
    assert bool(ninf[:, ~allowed_rows].all())                    # v0_hat is -inf at every forbidden entry of every step


@pytest.mark.parametrize('name,cfg', [(k, None) for k in KINDS] + [('respaced', {'model_mean_type': 'noise'}),
                                                                      ('respaced', {'cutoff_mode': 'hybrid'})])
def test_constrained_chain_vs_oracle(name, cfg):
    torch.set_num_threads(16)
    cfg = dict(T20 if name == 'default' else {}, **(cfg or {}))
    T = restate.make_schedules(cfg)['betas'].shape[0]
    model, sd = _model(cfg)
    b = _origin_batch(61, [9, 14, 6])
    n = len(b['batch_ligand'])
    path, okw, ekw, fixed = _case(name, b, T)
    allowed = _random_mask(n, K13, 5)
    if fixed is not None:
        allowed[fixed] = True
    pn, vu = synth.make_tape(62, len(path), n)
    got = _sample(model, b, mode='none', noise_tape=(pn, vu), allowed_types=allowed.to(DEV), **ekw)
    want = tc.sample_diffusion(sd, cfg, *_args(b, 'cpu'), pn, vu, path, center_pos_mode='none', allowed=allowed, **okw)
    first_bad = (got['v_traj'] != torch.stack(want['v_traj'])).any(1).nonzero()
    assert len(first_bad) == 0, 'atom types diverge from the oracle at step %d' % int(first_bad[0])
    torch.testing.assert_close(got['pos_traj'], torch.stack(want['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    _check_logs(got['v0_traj'], torch.stack(want['v0_traj']), allowed)
    _check_logs(got['vt_traj'][-1:], want['vt_traj'][-1][None], allowed)          # the decoder step: renormalised over the set
    wt = torch.stack(want['vt_traj'])[:-1]
    assert bool(torch.isfinite(wt).all()) and float((got['vt_traj'][:-1] - wt).abs().max()) <= LOGIT_ATOL
    free = torch.ones(n, dtype=torch.bool) if fixed is None else ~fixed
    assert type_violations(got['v'][free], allowed[free]) == 0
    print('%s %s: %d steps, max |pos - oracle| %.2e' % (name, cfg, len(path), float((got['pos_traj'] - torch.stack(want['pos_traj'])).abs().max())))
    model._drop_engine()


@pytest.mark.parametrize('mean_type', ['C0', 'noise'])
def test_every_constrained_step_vs_float64(mean_type):
    """Each step from the engine's own state and fp32 network outputs, against oracle.type_constraints.conditioned_step in float64."""
    cfg = {'model_mean_type': mean_type}
    model, sd = _model(cfg)
    b = _origin_batch(71, [9, 14, 6])
    n = len(b['batch_ligand'])
    seq = [999, 800, 600, 400, 200, 100, 50, 10, 3, 1, 0]
    tab = resample.path_tables(sd, seq)
    allowed = _random_mask(n, K13, 6)
    pn, vu = synth.make_tape(72, len(seq), n)
    r = _sample(model, b, mode='none', noise_tape=(pn, vu), time_seq=seq, allowed_types=allowed.to(DEV))
    args = _args(b)
    exempt = 0
    for s, t in enumerate(seq):
        xt = b['init_ligand_pos'] if s == 0 else r['pos_traj'][s - 1]
        vt = b['init_ligand_v'] if s == 0 else r['v_traj'][s - 1]
        out = model(args[0], args[1], args[2], xt.to(DEV), vt.to(DEV), args[5])
        x0, logits = out['pred_ligand_pos'].cpu(), out['pred_ligand_v'].cpu()
        ref = tc.conditioned_step(sd, cfg, tab, s, xt, vt, x0, logits, pn[s], vu[s], allowed, dtype=torch.float64)
        close = ref['margin'] <= stepwise.MARGIN
        exempt += int(close.sum())
        assert int((r['v_traj'][s] != ref['v'])[~close].sum()) == 0, (s, t)
        pos_err = float(((r['pos_traj'][s].double() - ref['pos']).abs() / ref['scale'].clamp(min=1e-30)).max())
        assert pos_err <= stepwise.STEP_TOL['pos'], (s, t, pos_err)
        for key, got in (('v0', r['v0_traj'][s]), ('vt', r['vt_traj'][s])):
            ninf = torch.isneginf(ref[key])
            assert torch.equal(torch.isneginf(got), ninf), (s, t, key)
            err = float((got.double()[~ninf] - ref[key][~ninf]).abs().max())
            assert err <= stepwise.STEP_TOL[key], (s, t, key, err)
    assert exempt <= stepwise.MAX_EXEMPT
    model._drop_engine()


# ------------------------------------------------------------------------------------------------ D. independence, switches
def test_batch_independence():
    """A cfg3-shaped batch (64 pockets x 10 samples = 640 graphs of 300 protein + 20 ligand atoms) on a tape, each graph with its own
    set and every fifth graph unconstrained: graph 5 alone and the whole batch in reversed-and-rotated order give each graph the same
    bits, and the unconstrained graphs are the unconstrained run's."""
    model, _ = _model()
    G = 640
    b = synth.make_batch(21, G, n_protein=300, n_ligand=20, distinct_pockets=64)
    seq = respaced_time_seq(1000, 5)
    n = len(b['batch_ligand'])
    pn, vu = synth.make_tape(22, len(seq), n)
    allowed = _random_mask(n, K13, 7)
    free_graphs = torch.arange(G) % 5 == 0
    allowed[free_graphs[b['batch_ligand']]] = True
    full = _sample(model, b, noise_tape=(pn, vu), time_seq=seq, allowed_types=allowed.to(DEV))
    plain = _sample(model, b, noise_tape=(pn, vu), time_seq=seq)
    rows = free_graphs[b['batch_ligand']]
    for k in TRAJ:
        x, y = (full[k][:, rows], plain[k][:, rows]) if full[k].dim() > 1 and full[k].shape[0] == len(seq) else (full[k][rows], plain[k][rows])
        assert torch.equal(x, y), k
    assert not torch.equal(full['v'][~rows], plain['v'][~rows])
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
        got = _sample(model, sub, noise_tape=(pn[:, lr], vu[:, lr]), time_seq=seq, allowed_types=allowed[lr].to(DEV))
        for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
            assert torch.equal(got[k], full[k][:, lr]), (len(order), k)
        assert torch.equal(got['pos'], full['pos'][lr]) and torch.equal(got['v'], full['v'][lr])
    model._drop_engine()


@pytest.mark.parametrize('env', ['TDIFF_NO_GRAPH', 'TDIFF_NO_RESTRICT', 'TDIFF_KNN_FULL', 'TDIFF_NO_SLOT_KEEP', 'TDIFF_FREE_DEPTH'])
def test_switches_change_nothing(monkeypatch, env):
    """At a cfg3-shaped batch of 640 graphs, a constrained chain is bit for bit the same under each engine switch."""
    G = 640
    b = synth.make_batch(33, G, n_protein=300, n_ligand=20, distinct_pockets=64)
    n = len(b['batch_ligand'])
    kw = dict(time_seq=respaced_time_seq(1000, 6), seed=77, allowed_types=_random_mask(n, K13, 8).to(DEV))
    model, _ = _model()
    base = _sample(model, b, **kw)
    model._drop_engine()
    monkeypatch.setenv(env, '0' if env == 'TDIFF_FREE_DEPTH' else '1')
    other = _sample(model, b, **kw)
    model._drop_engine()
    assert not _differing(base, other)


# ------------------------------------------------------------------------------------------------ E. C-ABI, driver, CLI
def test_cabi_refusals_bind_and_forward():
    from targetdiff_b200 import _lib
    lib = _lib.load()
    model, _ = _model()
    model._drop_engine()
    eng = model.engine(DEV)
    st = model._stream(torch.device(DEV))
    b = synth.make_batch(95, 2, n_protein=80, ligand_sizes=[8, 5])
    a = _args(b)
    n = len(b['batch_ligand'])
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    bits = lambda m: (m.to(torch.int32) << torch.arange(K13, dtype=torch.int32)).sum(1, dtype=torch.int32).to(DEV).contiguous()
    good = bits(_random_mask(n, K13, 9))
    assert lib.tdiff_set_type_mask(eng, P(good), st) == _lib.TDIFF_ESTATE          # before a bind
    lpos, lv = a[3].float().contiguous(), a[4].long().contiguous()
    out = torch.empty_like(lpos)
    out_v = torch.empty_like(lv)
    seq = _lib.i32_array([999, 700, 300, 60, 0])                              # ends at t = 0: the decoder step draws from the set
    sample = lambda pos_only=0: lib.tdiff_sample_seq(eng, seq, 5, None, None, ctypes.c_uint64(5), None, None, None, None, pos_only, st)

    def chain(mask=None, set_mask=False, pos_only=0):
        model._bind(eng, a[0], a[1], a[2], a[5], 1)
        if set_mask:
            _lib.check(lib.tdiff_set_type_mask(eng, None if mask is None else P(mask), st))
        _lib.check(lib.tdiff_set_ligand(eng, P(lpos), P(lv), 1, st))
        _lib.check(sample(pos_only))
        _lib.check(lib.tdiff_get_ligand(eng, P(out), P(out_v), 1, st))
        torch.cuda.synchronize()
        return out.cpu().clone(), out_v.cpu().clone()

    plain = chain()
    masked = chain(good, True)
    assert not torch.equal(plain[1], masked[1])
    assert all((int(good[a]) >> int(masked[1][a])) & 1 for a in range(n))
    # refusals keep the mask: a row without a class, a bit at K, a bit at 31
    for bad_row, bad_val in ((3, 0), (0, 1 << K13), (5, 1 << 31)):
        bad = good.clone()
        bad[bad_row] = torch.tensor(bad_val, dtype=torch.int64).to(torch.int32)
        assert lib.tdiff_set_type_mask(eng, P(bad), st) == _lib.TDIFF_EINVAL
        assert 'no class' in lib.tdiff_last_error().decode()
    _lib.check(lib.tdiff_set_ligand(eng, P(lpos), P(lv), 1, st))
    _lib.check(sample())
    _lib.check(lib.tdiff_get_ligand(eng, P(out), P(out_v), 1, st))
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), masked[0]) and torch.equal(out_v.cpu(), masked[1])
    # pos_only with a mask is refused, and the mask stays
    assert sample(1) == _lib.TDIFF_EINVAL
    assert 'pos_only' in lib.tdiff_last_error().decode()
    # a bind clears the mask
    assert all(torch.equal(x, y) for x, y in zip(chain(), plain))
    # tdiff_forward and tdiff_likelihood_terms ignore the mask
    ts = torch.tensor([300, 0])
    lk_pn = torch.randn(n, 3, generator=torch.Generator().manual_seed(8)).to(DEV)
    lk_vu = torch.rand(n, K13, generator=torch.Generator().manual_seed(9)).to(DEV)

    def forward_and_likelihood(mask):
        model._bind(eng, a[0], a[1], a[2], a[5], 1)
        _lib.check(lib.tdiff_set_ligand(eng, P(lpos), P(lv), 1, st))
        if mask is not None:
            _lib.check(lib.tdiff_set_type_mask(eng, P(mask), st))
        pred_pos, pred_v = torch.empty(n, 3, device=DEV), torch.empty(n, K13, device=DEV)
        _lib.check(lib.tdiff_forward(eng, P(pred_pos), P(pred_v), None, 0, st))
        outs = [torch.empty(2, device=DEV) for _ in range(4)]
        _lib.check(lib.tdiff_likelihood_terms(eng, _lib.i32_array(ts.tolist()), None, P(lk_pn), P(lk_vu),
                                              ctypes.c_uint64(0), *[P(o) for o in outs], None, None, None, None, st))
        torch.cuda.synchronize()
        return [pred_pos.cpu(), pred_v.cpu()] + [o.cpu() for o in outs]

    on, off = forward_and_likelihood(good), forward_and_likelihood(None)
    assert all(torch.equal(x, y) for x, y in zip(on, off))
    model._drop_engine()


def test_1h36_driver_cpu_rng_vs_oracle():
    from targetdiff_b200 import atom_num
    from targetdiff_b200.pocket import element_classes, pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand, seed_all
    torch.set_num_threads(16)
    model, sd = _model(favour=7)
    data = pdb_to_pocket_data(PDB_1H36)
    seq = respaced_time_seq(1000, 8)
    classes = element_classes(['C', 'N', 'O'])
    allowed = torch.zeros(K13, dtype=torch.bool)
    allowed[classes] = True
    ctr = data.protein_pos.float().mean(0)
    frag = (ctr + torch.randn(3, 3, generator=torch.Generator().manual_seed(4)), torch.tensor([1, 7, 0]))
    seed_all(2021)
    got = sample_diffusion_ligand(model, data, 2, batch_size=2, device=DEV, sample_num_atoms='prior', rng='cpu', time_seq=seq,
                                  fixed_ligand=frag, allowed_types=classes)
    after_engine = torch.rand(1)
    seed_all(2021)
    want = tc.sample_diffusion_ligand(sd, None, data.protein_pos, data.protein_atom_feature, 2, atom_num._table(), seq, batch_size=2,
                                      fixed_ligand=frag, allowed=allowed)
    assert torch.equal(torch.rand(1), after_engine)                      # the same draws, in the same number
    assert [len(p) for p in got[0]] == [len(p) for p in want[0]]
    assert np.array_equal(np.concatenate(got[1]), np.concatenate(want[1]))
    assert np.array_equal(np.concatenate(got[3], axis=1), np.concatenate(want[3], axis=1))
    np.testing.assert_allclose(np.concatenate(got[2], axis=1), np.concatenate(want[2], axis=1), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(np.concatenate(got[0]), np.concatenate(want[0]), rtol=1e-4, atol=1e-4)
    assert type_violations([v[3:] for v in got[1]], classes) == 0 and all(v[:3].tolist() == [1, 7, 0] for v in got[1])
    model._drop_engine()


def test_driver_per_atom_sets_on_a_start_ligand():
    """R-group redesign: a start ligand with kept atoms and a per-atom set; the free atoms end in their own sets."""
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand
    model, _ = _model(favour=7)
    data = pdb_to_pocket_data(PDB_1H36)
    ctr = data.protein_pos.float().mean(0)
    g = torch.Generator().manual_seed(11)
    start = (ctr + torch.randn(8, 3, generator=g) * 1.5, torch.tensor([1, 1, 3, 5, 7, 7, 1, 2]))
    per = torch.ones(8, K13, dtype=torch.bool)
    per[4:, 7] = False
    per[6] = False
    per[6, [3, 5]] = True                                                # "this position must be N or O"
    r = sample_diffusion_ligand(model, data, 6, batch_size=3, device=DEV, start_ligand=start, start_time=500, keep_atoms=[0, 1, 4],
                                allowed_types=per)
    free = torch.ones(8, dtype=torch.bool)
    free[[0, 1, 4]] = False
    for v in r[1]:
        v = torch.as_tensor(v)
        assert bool(per[free][torch.arange(int(free.sum())), v[free]].all())
        assert v[[0, 1, 4]].tolist() == [1, 1, 7]                          # kept atoms keep their classes, forbidden or not
    model._drop_engine()


@pytest.mark.parametrize('command', ['sample_for_pocket', 'sample_pockets'])
def test_cli_writes_compliant_molecules(tmp_path, command):
    import shutil
    import yaml
    from targetdiff_b200.cli import main
    from targetdiff_b200.config import Config, default_model_config
    _, sd = _model(T20, favour=7)
    mc = default_model_config()
    mc.update(T20)
    torch.save({'config': Config(model=mc, data={'transform': {'ligand_atom_mode': 'add_aromatic'}}), 'model': sd}, tmp_path / 'ckpt.pt')
    conf = {'model': {'checkpoint': str(tmp_path / 'ckpt.pt')},
            'sample': {'seed': 1, 'num_samples': 4, 'num_steps': 20, 'pos_only': False, 'center_pos_mode': 'protein',
                       'sample_num_atoms': 'range', 'allowed_elements': ['C', 'N', 'O']}}
    with open(tmp_path / 'sample.yml', 'w') as f:
        yaml.safe_dump(conf, f)
    if command == 'sample_for_pocket':
        main([command, str(tmp_path / 'sample.yml'), '--pdb_path', PDB_1H36, '--result_path', str(tmp_path / 'out'), '--device', DEV])
        r = torch.load(tmp_path / 'out' / 'sample.pt', weights_only=False)
    else:
        (tmp_path / 'pockets').mkdir()
        shutil.copyfile(PDB_1H36, tmp_path / 'pockets' / '1h36_pocket10.pdb')
        main([command, str(tmp_path / 'sample.yml'), '--pocket_dir', str(tmp_path / 'pockets'), '--result_path', str(tmp_path / 'out'),
              '--device', DEV])
        r = torch.load(tmp_path / 'out' / 'result_0.pt', weights_only=False)
    assert r['allowed_classes'] == [1, 2, 3, 4, 5, 6]
    assert len(r['pred_ligand_v']) == 4 and type_violations(r['pred_ligand_v'], r['allowed_classes']) == 0
