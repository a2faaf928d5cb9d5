"""Likelihood scoring (DESIGN.md section 1) on the engine (run with -m gpu; `pytest -s` prints the errors).

1. tdiff_likelihood_terms on tapes against the oracle (oracle.likelihood.terms) at mixed t including 0, 1 and T - 1, priors included,
   and against model.likelihood_estimation on the same noise.
2. Per-atom terms against float64, on the engine's own x_t, v_t and its own forward at them.
3. The seeded stream's x_t, v_t against the host restatement (oracle.likelihood.likelihood_tape).
4. Batch independence, bit for bit: a ligand alone and inside a shuffled cfg3-shaped batch of 640 graphs; ligand_nll at batch sizes 1,
   7 and 640.
5. Engine state: the ligand is restored, a later chain equals a fresh engine's, launches per call are the forward's plus 2.
6. Options: time embedding, K = 8 and 23, hybrid cutoff, num_blocks 2.
7. The rng='cpu' driver against the reference's pins.
8. The CLI end to end.
9. C-ABI refusals."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import likelihood, philox, restate, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K13 = synth.LIGAND_NUM_CLASSES
EPS32 = 2.0 ** -23
RTOL, ATOL = 1e-4, 1e-5
# a per-atom position KL is the square of a difference with the network's prediction, so it carries twice the forward's relative error
ATOM_POS_RTOL = 3e-4
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
PDB_1H36 = os.path.join(GOLDEN, '1h36_pocket10.pdb')
OUTS = ('kl_pos', 'kl_v', 'prior_pos', 'prior_v')
# per-atom terms against float64 (test 2), limits about 4x the largest error measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit
# (DESIGN.md section 2).  Position terms and the position prior: |engine - float64| / (|float64| + the median term), measured 1.01e-5.
# Type terms and the type prior are small differences of K products each (the prior about 1e-7 from terms of size 1/K), so their error is
# measured in units of the magnitudes they are computed from (oracle.likelihood's return_scale), measured 1.26e-7.
F64_POS_REL = 4e-5
F64_TYPE_S = 5e-7


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


def _cpu(r):
    return {k: v.cpu() for k, v in r.items()}


def _close(got, want, keys=OUTS):
    for k in keys:
        torch.testing.assert_close(got[k], want[k], rtol=RTOL, atol=ATOL, msg=lambda m: '%s: %s' % (k, m))


# ------------------------------------------------------------------------------------------------ 1, 6. against the oracle on tapes
OPTIONS = [({}, K13), ({'time_emb_dim': 1, 'time_emb_mode': 'simple'}, K13), ({}, 8), ({}, 23), ({'cutoff_mode': 'hybrid'}, K13),
           ({'num_blocks': 2}, K13)]


@pytest.mark.parametrize('cfgd,K', OPTIONS, ids=['default', 'time_emb', 'K8', 'K23', 'hybrid', 'blocks2'])
def test_terms_vs_oracle_on_tapes(cfgd, K):
    model, sd = _model(cfgd, K=K)
    T = model.num_timesteps
    b = synth.make_batch(21, 5, n_protein=64, ligand_sizes=[9, 12, 7, 10, 8], num_classes=K)
    ts = [0, 1, T - 1, 417, 2]
    pn, vu = likelihood.likelihood_tape(77, ts, None, b['batch_ligand'], K)
    got = _cpu(model.likelihood_terms(*_args(b), ts, noise=(pn, vu), return_atoms=True))
    want = likelihood.terms(sd, cfgd, *(b[k] for k in ARGS), torch.tensor(ts), pn, vu, return_atoms=True)
    assert torch.equal(got['vt'], want['vt'])
    torch.testing.assert_close(got['xt'], want['xt'], rtol=0, atol=0)
    _close(got, want)
    torch.testing.assert_close(got['atom_kl_pos'], want['atom_kl_pos'], rtol=ATOM_POS_RTOL, atol=ATOL)
    _close(got, want, ('atom_kl_v',))
    if not cfgd.get('cutoff_mode'):
        # model.likelihood_estimation (the reference-signature entry) on the same noise gives the same per-graph terms
        kp, kv = model.likelihood_estimation(*_args(b), torch.tensor(ts, device=DEV), noise=(pn, vu))
        torch.testing.assert_close(kp.cpu(), got['kl_pos'], rtol=RTOL, atol=ATOL)
        torch.testing.assert_close(kv.cpu(), got['kl_v'], rtol=RTOL, atol=ATOL)


# ------------------------------------------------------------------------------------------------ 2. per-atom terms against float64
@pytest.mark.parametrize('K', [K13, 23])
def test_atom_terms_vs_float64(K):
    model, sd = _model(K=K)
    T = model.num_timesteps
    b = synth.make_batch(31, 6, n_protein=64, ligand_sizes=[9, 12, 7, 10, 8, 6], num_classes=K)
    ts = [0, 1, 2, 300, T - 2, T - 1]
    r = _cpu(model.likelihood_terms(*_args(b), ts, seed=5, return_atoms=True))
    # the engine's own forward on its x_t, v_t (centred frame, center_mode 0)
    pp, x0, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    out = model(pp.to(DEV), b['protein_v'].to(DEV), b['batch_protein'].to(DEV), r['xt'].to(DEV), r['vt'].to(DEV), b['batch_ligand'].to(DEV))
    t_atom = torch.tensor(ts)[b['batch_ligand']]
    tp, tv, sv = likelihood.atom_terms(sd, x0, b['init_ligand_v'], r['xt'], r['vt'], out['pred_ligand_pos'].cpu(),
                                       out['pred_ligand_v'].cpu(), t_atom, K, dtype=torch.float64, return_scale=True)
    ep, ev, spv = likelihood.prior_atom_terms(sd, x0, b['init_ligand_v'], K, dtype=torch.float64, return_scale=True)
    mean = lambda v: restate._scatter_mean_rows(v, b['batch_ligand'], len(ts))       # noqa: E731
    rel = lambda got, want: float(((got.double() - want).abs() / (want.abs() + float(want.abs().median()))).max())   # noqa: E731
    errs = {'pos': rel(r['atom_kl_pos'], tp), 'prior_pos': rel(r['prior_pos'], mean(ep)),
            'v': float(((r['atom_kl_v'].double() - tv).abs() / sv).max()),
            'prior_v': float(((r['prior_v'].double() - mean(ev)).abs() / mean(spv)).max())}
    print('errors against float64:', errs)
    assert errs['pos'] <= F64_POS_REL and errs['prior_pos'] <= F64_POS_REL, errs
    assert errs['v'] <= F64_TYPE_S and errs['prior_v'] <= F64_TYPE_S, errs


# ------------------------------------------------------------------------------------------------ 3. the seeded stream
def test_seeded_stream_vs_host_restatement():
    model, sd = _model()
    b = synth.make_batch(41, 4, n_protein=64, ligand_sizes=[9, 12, 7, 10])
    ts, keys = [0, 999, 500, 17], [7, 123456, 0, 2 ** 32 - 1]
    seeded = _cpu(model.likelihood_terms(*_args(b), ts, keys=keys, seed=2024, return_atoms=True))
    pn, vu = likelihood.likelihood_tape(2024, ts, keys, b['batch_ligand'], K13)
    taped = _cpu(model.likelihood_terms(*_args(b), ts, noise=(pn, vu), return_atoms=True))
    assert torch.equal(seeded['vt'], taped['vt'])
    # positions: the kernel's logf / sqrtf / cospif against float64 rounded once; within philox.STREAM_ULPS ulps of |x_t| + sigma |eps|
    _, x0, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    ac = sd['alphas_cumprod'][torch.tensor(ts)][b['batch_ligand']].unsqueeze(-1)
    scale = taped['xt'].double().abs() + ac.sqrt() * x0.abs() + (1 - ac).sqrt() * pn.double().abs()
    ulps = float(((seeded['xt'].double() - taped['xt'].double()).abs() / (EPS32 * scale)).max())
    print('seeded x_t vs host stream: %.3f ulps' % ulps)
    assert ulps <= philox.STREAM_ULPS


# ------------------------------------------------------------------------------------------------ 4. batch independence
def test_ligand_alone_equals_ligand_in_shuffled_cfg3_batch():
    model, _ = _model()
    T = model.num_timesteps
    g = torch.Generator().manual_seed(3)
    n_graphs = 640
    pockets = [synth.make_pocket(100 + i, n_protein=300) for i in range(64)]
    graphs = []
    for i in range(n_graphs):
        pos, feat = pockets[i % 64]
        centre = pos.mean(0)
        lig = centre + 1.5 * torch.randn(20, 3, generator=g)
        graphs.append((pos, feat, lig, torch.randint(0, K13, (20,), generator=g), int(torch.randint(0, T, (1,), generator=g)), i))
    perm = torch.randperm(n_graphs, generator=g).tolist()
    graphs = [graphs[p] for p in perm]

    def run(gs):
        pp = torch.cat([x[0] for x in gs]); pf = torch.cat([x[1] for x in gs])
        bp = torch.repeat_interleave(torch.arange(len(gs)), torch.tensor([len(x[0]) for x in gs]))
        lp = torch.cat([x[2] for x in gs]); lv = torch.cat([x[3] for x in gs])
        bl = torch.repeat_interleave(torch.arange(len(gs)), torch.tensor([len(x[2]) for x in gs]))
        a = (pp, pf, bp, lp, lv, bl)
        return _cpu(model.likelihood_terms(*(x.to(DEV) for x in a), [x[4] for x in gs], keys=[x[5] for x in gs], seed=99, return_atoms=True))

    full = run(graphs)
    for pos_in_batch in (0, 1, 317, n_graphs - 1):
        alone = run([graphs[pos_in_batch]])
        a0 = sum(len(graphs[j][2]) for j in range(pos_in_batch))
        for k in OUTS:
            assert torch.equal(alone[k][0], full[k][pos_in_batch]), k
        for k in ('atom_kl_pos', 'atom_kl_v', 'xt', 'vt'):
            assert torch.equal(alone[k], full[k][a0:a0 + 20]), k


def test_ligand_nll_independent_of_batch_size():
    from targetdiff_b200.likelihood import ligand_nll
    from targetdiff_b200.pocket import pdb_to_pocket_data
    model, _ = _model()
    data = pdb_to_pocket_data(PDB_1H36)
    centre = torch.as_tensor(data['protein_pos']).float().mean(0)
    g = torch.Generator().manual_seed(5)
    ligs = [(centre + 1.4 * torch.randn(n, 3, generator=g), torch.randint(0, K13, (n,), generator=g)) for n in (9, 14, 11, 20, 6)]
    runs = [ligand_nll(model, data, ligs, batch_size=bs, device=DEV, seed=11) for bs in (1, 7, 640)]
    for r in runs[1:]:
        for a, c in zip(runs[0], r):
            assert torch.equal(a['kl_pos'], c['kl_pos']) and torch.equal(a['kl_v'], c['kl_v']) and a['nll'] == c['nll']
    # and a ligand scored with others equals the ligand scored alone under the same key
    alone = ligand_nll(model, data, ligs[:1], batch_size=640, device=DEV, seed=11)[0]
    assert torch.equal(alone['kl_pos'], runs[0][0]['kl_pos']) and torch.equal(alone['kl_v'], runs[0][0]['kl_v'])
    assert runs[0][0]['kl_pos'].shape == (11,)
    assert np.isfinite([r['nll'] for r in runs[0]]).all()


# ------------------------------------------------------------------------------------------------ 5. engine state
def _launches(model):
    from targetdiff_b200 import _lib
    return _lib.load().tdiff_launch_count(model.engine(DEV))


def test_state_restored_and_launch_count():
    from targetdiff_b200 import _lib
    model, _ = _model()
    lib = _lib.load()
    b = synth.make_batch(51, 3, n_protein=64, ligand_sizes=[9, 12, 7])
    a = _args(b)
    model.likelihood_terms(*a, [0, 5, 999], seed=3)
    eng = model.engine(DEV)
    st = model._stream(torch.device(DEV))
    pos = torch.empty(len(b['batch_ligand']), 3, device=DEV)
    v = torch.empty(len(b['batch_ligand']), dtype=torch.int64, device=DEV)
    _lib.check(lib.tdiff_get_ligand(eng, ctypes.c_void_p(pos.data_ptr()), ctypes.c_void_p(v.data_ptr()), 1, st))
    assert torch.equal(v.cpu(), b['init_ligand_v'])
    torch.testing.assert_close(pos.cpu(), b['init_ligand_pos'], rtol=0, atol=4 * EPS32 * float(b['init_ligand_pos'].abs().max()))
    # launches: bind + set_ligand + the forward + 2, the forward's count taken from tdiff_forward on the same batch
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    n0 = _launches(model)
    model.likelihood_terms(*a, [0, 5, 999], seed=3)
    n_call = _launches(model) - n0
    n0 = _launches(model)
    model._bind(eng, a[0], a[1], a[2], a[5], 1)
    lpos, lv = a[3].float().contiguous(), a[4].long().contiguous()
    _lib.check(lib.tdiff_set_ligand(eng, ctypes.c_void_p(lpos.data_ptr()), ctypes.c_void_p(lv.data_ptr()), 1, st))
    _lib.check(lib.tdiff_forward(eng, None, None, None, 0, st))
    n_fwd = _launches(model) - n0
    print('launches: likelihood call %d, bind + set_ligand + forward %d' % (n_call, n_fwd))
    assert n_call == n_fwd + 2


def test_chain_after_likelihood_equals_fresh_engine():
    model, _ = _model()
    b = synth.make_batch(61, 3, n_protein=64, ligand_sizes=[9, 12, 7])
    pn, vu = synth.make_tape(4, 5, len(b['batch_ligand']))
    model.likelihood_terms(*_args(b), [0, 5, 999], seed=3)
    model.likelihood_terms(*_args(b), [1, 2, 3], noise=likelihood.likelihood_tape(1, [1, 2, 3], None, b['batch_ligand'], K13))
    r1 = model.sample_diffusion(*_args(b), num_steps=5, center_pos_mode='protein', noise_tape=(pn, vu), stack_traj=True)
    fresh, _ = _model()
    r2 = fresh.sample_diffusion(*_args(b), num_steps=5, center_pos_mode='protein', noise_tape=(pn, vu), stack_traj=True)
    for k in ('pos', 'v', 'pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
        assert torch.equal(r1[k].cpu(), r2[k].cpu()), k
    # and the scores after a chain equal those on a fresh engine
    s1 = _cpu(model.likelihood_terms(*_args(b), [0, 5, 999], seed=3))
    s2 = _cpu(_model()[0].likelihood_terms(*_args(b), [0, 5, 999], seed=3))
    for k in OUTS:
        assert torch.equal(s1[k], s2[k]), k


def test_empty_ligand_graph_scores_zero():
    model, sd = _model()
    b = synth.make_ragged_batch(71, [40, 50, 45], [6, 0, 8])
    ts = [3, 7, 900]
    pn, vu = likelihood.likelihood_tape(8, ts, None, b['batch_ligand'], K13)
    got = _cpu(model.likelihood_terms(*_args(b), ts, noise=(pn, vu)))
    for k in OUTS:
        assert got[k][1] == 0
    want = likelihood.terms(sd, None, *(b[k] for k in ARGS), torch.tensor(ts), pn, vu)
    _close(got, want)


# ------------------------------------------------------------------------------------------------ 7. the driver against the reference pins
@pytest.mark.parametrize('name', ['default_bs4', 'default_bs1', 'time_emb', 'K23', '1h36'])
def test_driver_cpu_rng_vs_reference_pins(name):
    from targetdiff_b200.likelihood import data_likelihood_estimation
    from targetdiff_b200.sampling import seed_all
    case = torch.load(os.path.join(GOLDEN, 'reference_pins_likelihood_driver.pt'), weights_only=False)[name]
    model, _ = _model(case['cfg'], weight_seed=case['weight_seed'], K=case['K'])
    seed_all(case['seed'])
    kp, kv, sp, sv = data_likelihood_estimation(model, case['data'], case['time_steps'], batch_size=case['batch_size'], device=DEV, rng='cpu')
    torch.testing.assert_close(kp, case['kl_pos'], rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(kv, case['kl_v'], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose([sp, sv], [case['sum_kl_pos'], case['sum_kl_v']], rtol=RTOL, atol=ATOL)


# ------------------------------------------------------------------------------------------------ 8. CLI
def _write_ckpt_and_config(tmp_path, cfg, time_emb=False):
    import yaml
    from targetdiff_b200.config import Config, default_model_config
    _, sd = _model(cfg)
    mc = default_model_config()
    mc.update(cfg)
    torch.save({'config': Config(model=mc, data={'transform': {'ligand_atom_mode': 'add_aromatic'}}), 'model': sd}, tmp_path / 'ckpt.pt')
    conf = {'model': {'checkpoint': str(tmp_path / 'ckpt.pt')},
            'sample': {'seed': 1, 'num_samples': 3, 'num_steps': 20, 'pos_only': False, 'center_pos_mode': 'protein',
                       'sample_num_atoms': 'prior'}}
    with open(tmp_path / 'sample.yml', 'w') as f:
        yaml.safe_dump(conf, f)
    return tmp_path / 'sample.yml'


def test_cli_score_samples_and_ligands(tmp_path):
    from targetdiff_b200.cli import main
    from targetdiff_b200.likelihood import ligand_nll
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import seed_all
    cfg = dict(num_diffusion_timesteps=20)
    yml = _write_ckpt_and_config(tmp_path, cfg)
    main(['sample_for_pocket', str(yml), '--pdb_path', PDB_1H36, '--result_path', str(tmp_path / 'out'), '--device', DEV])
    main(['score_ligands', str(yml), '--samples', str(tmp_path / 'out' / 'sample.pt'), '--result_path', str(tmp_path / 's1'),
          '--time_steps', 'all', '--device', DEV, '--batch_size', '7'])
    scores = torch.load(tmp_path / 's1' / 'scores.pt', weights_only=False)
    r = torch.load(tmp_path / 'out' / 'sample.pt', weights_only=False)
    assert len(scores) == len(r['pred_ligand_pos']) == 3
    model, _ = _model(cfg)
    seed_all(1)                                                   # the CLI draws the stream's seed right after seeding
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    want = ligand_nll(model, r['data'], list(zip(r['pred_ligand_pos'], r['pred_ligand_v'])), time_steps=list(range(20)), device=DEV,
                      seed=seed)
    for i, (s, w) in enumerate(zip(scores, want)):
        assert s['sample_index'] == i and s['kl_pos'].shape == (21,)
        assert torch.equal(s['kl_pos'], w['kl_pos']) and torch.equal(s['kl_v'], w['kl_v']) and s['nll'] == w['nll']
    # --ligand with two files and --embedding
    data = pdb_to_pocket_data(PDB_1H36)
    for i in range(2):
        np.savez(tmp_path / ('l%d.npz' % i), pos=np.asarray(r['pred_ligand_pos'][i], np.float32), v=np.asarray(r['pred_ligand_v'][i]))
    files = [str(tmp_path / 'l0.npz'), str(tmp_path / 'l1.npz')]
    main(['score_ligands', str(yml), '--pdb_path', PDB_1H36, '--ligand', *files, '--embedding', '--result_path', str(tmp_path / 's2'),
          '--device', DEV])
    sc2 = torch.load(tmp_path / 's2' / 'scores.pt', weights_only=False)
    assert [s['source'] for s in sc2] == files
    for i, s in enumerate(sc2):
        n = len(r['pred_ligand_v'][i])
        assert s['kl_pos'].shape == (11,) and np.isfinite(s['nll'])
        assert s['pred_ligand_v'].shape == (n, K13) and s['final_ligand_h'].shape == (n, 128)
        assert s['final_h'].shape == (len(data['protein_pos']) + n, 128)
        one = model.fetch_embedding(torch.as_tensor(data['protein_pos']).float().to(DEV), torch.as_tensor(data['protein_atom_feature']).float().to(DEV),
                                    torch.zeros(len(data['protein_pos']), dtype=torch.long, device=DEV),
                                    torch.as_tensor(np.asarray(r['pred_ligand_pos'][i], np.float32)).to(DEV),
                                    torch.as_tensor(np.asarray(r['pred_ligand_v'][i])).long().to(DEV), torch.zeros(n, dtype=torch.long, device=DEV))
        torch.testing.assert_close(s['final_ligand_h'], one['final_ligand_h'].cpu(), rtol=RTOL, atol=1e-4)
    # --embedding with a time embedding is refused
    yml2 = _write_ckpt_and_config(tmp_path, dict(num_diffusion_timesteps=20, time_emb_dim=1, time_emb_mode='simple'))
    with pytest.raises(ValueError, match='time embedding'):
        main(['score_ligands', str(yml2), '--pdb_path', PDB_1H36, '--ligand', files[0], '--embedding', '--result_path', str(tmp_path / 's3'),
              '--device', DEV])


# ------------------------------------------------------------------------------------------------ 9. C-ABI refusals
def test_cabi_refusals():
    from targetdiff_b200 import _lib
    model, sd = _model()
    T = model.num_timesteps
    lib = _lib.load()
    eng = model.engine(DEV)
    st = model._stream(torch.device(DEV))
    b = synth.make_batch(95, 2, n_protein=60, ligand_sizes=[8, 5])
    a = _args(b)
    n = len(b['batch_ligand'])
    vp = lambda t: ctypes.c_void_p(t.data_ptr())                                    # noqa: E731
    pn, vu = torch.zeros(n, 3, device=DEV), torch.full((n, K13), 0.5, device=DEV)

    def call(ts, p=None, u=None, e=eng):
        return lib.tdiff_likelihood_terms(e, _lib.i32_array(ts), None, p, u, ctypes.c_uint64(1), None, None, None, None, None, None, None, None, st)

    assert call([0, 1], e=None) == _lib.TDIFF_ESTATE
    fresh = _model()[0]
    assert call([0, 1], e=fresh.engine(DEV)) == _lib.TDIFF_ESTATE                  # before bind
    model._bind(eng, a[0], a[1], a[2], a[5], 1)
    assert call([0, 1]) == _lib.TDIFF_ESTATE                                         # before set_ligand
    lpos, lv = a[3].float().contiguous(), a[4].long().contiguous()
    _lib.check(lib.tdiff_set_ligand(eng, vp(lpos), vp(lv), 1, st))
    for ts in ([0, T], [-1, 0]):
        assert call(ts) == _lib.TDIFF_EINVAL and b'outside 0..' in lib.tdiff_last_error()
    assert call([0, 1], vp(pn), None) == _lib.TDIFF_EINVAL and b'both' in lib.tdiff_last_error()
    assert call([0, 1], None, vp(vu)) == _lib.TDIFF_EINVAL
    assert call([0, 1], vp(pn), vp(vu)) == _lib.TDIFF_OK
    assert call([0, 1]) == _lib.TDIFF_OK
    noise_model = _model({'model_mean_type': 'noise'})[0]
    ne = noise_model.engine(DEV)
    noise_model._bind(ne, a[0], a[1], a[2], a[5], 1)
    _lib.check(lib.tdiff_set_ligand(ne, vp(lpos), vp(lv), 1, st))
    assert call([0, 1], e=ne) == _lib.TDIFF_EINVAL and b'C0' in lib.tdiff_last_error()
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match='noise shapes'):
        model.likelihood_terms(*a, [0, 1], noise=(pn[:-1], vu))
    with pytest.raises(ValueError, match='one entry per graph'):
        model.likelihood_terms(*a, [0, 1, 2])
