"""Ligand class counts other than 13, and the parts of a forward that only end-to-end tests reached, against float64 (run with -m gpu;
`pytest -s` prints every measured error beside the fp32 oracle's on the same inputs).

a. K = 8 ('basic'), 23 ('full') and 24 (the largest K the engine accepts): forward and chains against the oracle (which equals the
   reference pins of tests/golden/reference_pins_class_counts.pt at K = 8 and 23), the seeded chain against its host Philox tape,
   every step against float64, likelihood_estimation with and without the time embedding, and the sampling driver at K = 23.
b. The embeddings (`protein_embed_kernel`, `init_h_kernel` with the time column): with the last Linear of every hv_func zeroed, every
   x2h sub-layer adds exactly 0, so final_h is the embedding, protein and ligand rows alike.
c. The type head (`head_kernel`) on the engine's own final_ligand_h: synthetic weights, weights scaled so that the pre-activations
   span about +-40, and a probe head whose logits are single softplus outputs at chosen pre-activations around the threshold 20.
d. The global edge gate (`edge_const.cu`) on the engine's graph of the 1h36 pocket, at k = 8, 32, 48, also with a saturated sigmoid.
e. Every block after the first: the engine's output of b - 1 blocks through `oracle.layerwise.block` in float64 (graph rebuilt from
   the engine's coordinates, gate, layers) against the engine's output of b blocks.
f. forward(return_all=True) of a B-block network: entry b equals the output of the b-block network bit for bit."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import layerwise, philox, restate, stepwise, synth
from oracle import make_class_count_pins as ccp
from oracle import make_reference_pins as pins_mod
from oracle.make_reference_pins import LIKELIHOOD_STEPS, equal

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PDB_1H36 = os.path.join(ROOT, 'tests', 'golden', '1h36_pocket10.pdb')
LN2_F32 = 0.6931471824645996
EPS32 = 2.0 ** -23

# Limits against float64, about 3-4x the larger of the engine's and the fp32 oracle's maximum measured on one NVIDIA H100 80GB HBM3 at a
# 400 W power limit (DESIGN.md section 2 lists both).
EMBED_TOL = 2e-7          # absolute, every row of final_h with the x2h updates zeroed; measured 6.0e-8, fp32 oracle 6.0e-8
HEAD_TOL = 7e-7           # logit error / (|W2| |y| + |b2|), relative to the size of the terms the logit sums; measured 1.9e-7,
                          # fp32 oracle 2.1e-7
PROBE_ULPS = 2.5          # probe head: fp32 ulps of |softplus(z)| + ln 2; measured 0.67, fp32 oracle 0.59
GATE_TOL = 5e-7           # absolute; measured 1.4e-7, fp32 oracle 1.4e-7
GATE_TOL_SATURATED = 1.5e-5   # absolute, gate logits over +-20; measured 4.0e-6, fp32 oracle 4.0e-6


def _make(K, cfg, sd):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


def _model(K, cfg=None, seed=0):
    sd = ccp.weights(seed, K, cfg or {})
    return _make(K, cfg, sd), sd


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))


@pytest.fixture
def one_thread():
    """The pins were computed with one torch-CPU thread (reductions split by thread count)."""
    n = torch.get_num_threads()
    torch.set_num_threads(pins_mod.THREADS)
    yield
    torch.set_num_threads(n)


@pytest.fixture(scope='module')
def pins():
    return torch.load(ccp.OUT, weights_only=True)


CLASS_CASES = [(K, cfgd) for K in (8, 23, 24) for cfgd in ccp.CONFIGS]


def _cid(case):
    return ccp.case_id(*case)


# ------------------------------------------------------------------------------------------------ a. class counts
@pytest.mark.parametrize('case', CLASS_CASES, ids=_cid)
def test_class_count_forward_and_chain_vs_oracle(pins, one_thread, case):
    """Forward on the pins' inputs, their 3-step chain and a 6-step chain on the same batch: the engine within the usual
    tolerances of the oracle, types equal; at K = 8 and 23 the oracle outputs compared are the reference's own (pins, bit for bit)."""
    K, cfgd = case
    want_pin = pins.get(_cid(case))
    model, sd = _model(K, cfgd)
    b, pp, lp, t = ccp.forward_inputs(K)
    want = restate.forward(sd, cfgd, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], time_step=t)
    if want_pin is not None:
        assert all(equal(want[k], want_pin['forward'][k]) for k in want_pin['forward'])
    out = model(pp.to(DEV), b['protein_v'].to(DEV), b['batch_protein'].to(DEV), lp.to(DEV), b['init_ligand_v'].to(DEV),
                b['batch_ligand'].to(DEV), time_step=t.to(DEV))
    assert out['pred_ligand_v'].shape == (16, K)
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=1e-3)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=1e-4, atol=1e-4)
    b, pn, vu = ccp.chain_inputs(K)
    for S in (3, 6):
        pn, vu = synth.make_tape(5, S, 16, num_classes=K)
        w = restate.sample_diffusion(sd, cfgd, *_args(b, 'cpu'), pn, vu, num_steps=S)
        if S == 3 and want_pin is not None:
            assert all(equal(list(w[k]) if k.endswith('traj') else w[k], want_pin['chain'][k]) for k in want_pin['chain'])
        got = model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', noise_tape=(pn, vu), stack_traj=True)
        assert torch.equal(got['v_traj'], torch.stack(w['v_traj']))
        torch.testing.assert_close(got['pos_traj'], torch.stack(w['pos_traj']), rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(got['v0_traj'], torch.stack(w['v0_traj']), rtol=0, atol=1e-3)
        torch.testing.assert_close(got['vt_traj'], torch.stack(w['vt_traj']), rtol=0, atol=1e-3)


@pytest.mark.parametrize('K', [8, 23, 24])
def test_class_count_device_stream_is_engine_tape(K):
    """The seeded chain equals the same chain on philox.engine_tape(seed, ..., K): ceil(K / 4) class counters per atom and step."""
    model, sd = _model(K)
    b = synth.make_batch(31, 4, n_protein=50, ligand_sizes=[60, 45, 33, 37], num_classes=K)
    n, S, seed = len(b['batch_ligand']), 3, 2 ** 32 + 7
    kw = dict(num_steps=S, center_pos_mode='protein', stack_traj=True)
    dev = model.sample_diffusion(*_args(b), seed=seed, **kw)
    pn, vu = philox.engine_tape(seed, n, S, K)
    tape = model.sample_diffusion(*_args(b), noise_tape=(pn, vu), **kw)
    assert torch.equal(dev['v_traj'], tape['v_traj'])
    assert torch.equal(dev['v0_traj'][0], tape['v0_traj'][0]) and torch.equal(dev['vt_traj'][0], tape['vt_traj'][0])
    T = sd['betas'].shape[0]
    sigma = float(np.exp(0.5 * float(sd['posterior_logvar'][T - 1])))
    ulps, later = philox.stream_errors(dev['pos_traj'], tape['pos_traj'], pn[0], sigma)
    print('K=%d stream: step 0 %.2f ulp, later steps %.2e rel' % (K, ulps, later))
    assert ulps <= philox.STREAM_ULPS and later <= philox.STREAM_LATER_REL


def _centred_batch(seed, sizes, K, n_protein=60):
    b = synth.make_batch(seed, len(sizes), n_protein=n_protein, ligand_sizes=sizes, distinct_pockets=1, num_classes=K)
    shift = b['protein_pos'].mean(0, keepdim=True)
    b['protein_pos'] = b['protein_pos'] - shift
    b['init_ligand_pos'] = b['init_ligand_pos'] - shift
    return b


@pytest.mark.parametrize('time_emb', [False, True], ids=['plain', 'time_emb'])
@pytest.mark.parametrize('K', [8, 23, 24])
def test_class_count_each_step_vs_float64(K, time_emb):
    """Every step of a T = 20 chain (through t = 0) against oracle.stepwise in float64, at STEP_TOL: log K, the K-wide log-softmax
    and posterior, the Gumbel-max over K classes."""
    cfg = dict({'num_diffusion_timesteps': 20}, **(ccp.TIME_EMB if time_emb else {}))
    model, sd = _model(K, cfg)
    b = _centred_batch(41, [9, 14], K)
    pn, vu = synth.make_tape(41, 20, len(b['batch_ligand']), num_classes=K)
    rows = stepwise.engine_steps_vs_float64('K=%d %s' % (K, 'time_emb' if time_emb else ''), model, sd, cfg, b, pn, vu, range(20), DEV)
    stepwise.check_steps('K=%d' % K, rows)


@pytest.mark.parametrize('case', CLASS_CASES, ids=_cid)
def test_class_count_likelihood_vs_oracle(pins, one_thread, case):
    """likelihood_estimation at the pins' two time-step vectors and at the prior, with the pins' noise, against the oracle (the
    reference's values at K = 8 and 23), with and without the time embedding."""
    K, cfgd = case
    want_pin = pins.get(_cid(case))
    model, sd = _model(K, cfgd, seed=5)
    b, pn, vu = ccp.likelihood_inputs(K)
    for steps in LIKELIHOOD_STEPS:
        t = ccp.likelihood_time_steps(steps)
        want = restate.likelihood_estimation(sd, cfgd, *_args(b, 'cpu'), t, pn[0], vu[0])
        if want_pin is not None:
            assert all(torch.equal(w, p) for w, p in zip(want, want_pin['likelihood'][str(steps)]))
        got = model.likelihood_estimation(*_args(b), time_step=t.to(DEV), noise=(pn[0], vu[0]))
        for g, w in zip(got, want):
            tol = dict(rtol=1e-5, atol=1e-6) if steps is None else dict(rtol=1e-4, atol=1e-5)
            torch.testing.assert_close(g.cpu(), w, **tol)


def test_driver_rng_cpu_class_count_23_vs_oracle():
    """sample_diffusion_ligand(rng='cpu') at K = 23 on the 1h36 pocket, prior sizes, 3 steps, 2 batches: the same CPU draws as
    oracle.restate.sample_diffusion_ligand (the K-wide initial-type draw included), the same types, positions within tolerance."""
    import random
    from targetdiff_b200.pocket import pdb_to_pocket_data
    from targetdiff_b200.sampling import sample_diffusion_ligand, seed_all
    K = 23
    model, sd = _model(K)
    data = pdb_to_pocket_data(PDB_1H36)
    prior = json.load(open(os.path.join(ROOT, 'targetdiff_b200', 'data', 'atom_num_prior.json')))
    seed_all(2021)
    got = sample_diffusion_ligand(model, data, 3, batch_size=2, device=DEV, num_steps=3, rng='cpu')
    torch.manual_seed(2021)
    np.random.seed(2021)
    random.seed(2021)
    want = restate.sample_diffusion_ligand(sd, None, data.protein_pos, data.protein_atom_feature, 3, prior, batch_size=2, num_steps=3)
    assert [len(p) for p in got[0]] == [len(p) for p in want[0]]
    for i in (1, 3):                                  # final types, type trajectories
        assert all(np.array_equal(g, w) for g, w in zip(got[i], want[i]))
    for i in (0, 2):                                  # final positions, position trajectories
        for g, w in zip(got[i], want[i]):
            torch.testing.assert_close(torch.from_numpy(g), torch.from_numpy(w), rtol=1e-4, atol=1e-5)
    for i in (4, 5):                                  # v0, vt trajectories
        for g, w in zip(got[i], want[i]):
            assert g.shape[-1] == K
            torch.testing.assert_close(torch.from_numpy(g), torch.from_numpy(w), rtol=0, atol=1e-3)


# ------------------------------------------------------------------------------------------------ b. embeddings
def _zero_x2h_values(sd, num_layers):
    sd = dict(sd)
    for l in range(num_layers):
        for s in ('weight', 'bias'):
            k = 'refine_net.base_block.%d.x2h_layers.0.hv_func.net.3.%s' % (l, s)
            sd[k] = torch.zeros_like(sd[k])
    return sd


@pytest.mark.parametrize('K,time_emb', [(13, False), (13, True), (23, True), (8, False)])
def test_embedding_vs_float64(K, time_emb):
    """final_h with every x2h value MLP zeroed is the embedding: protein rows W_p f + b_p (indicator 0), ligand rows W_l[:, v] + b_l
    + w_time t / T (indicator 1), at several t per graph."""
    cfg = ccp.TIME_EMB if time_emb else {}
    sd = _zero_x2h_values(ccp.weights(3, K, cfg), synth.DEFAULT_MODEL_CONFIG['num_layers'])
    model = _make(K, cfg, sd)
    b = synth.make_batch(7, 3, n_protein=70, ligand_sizes=[12, 5, 20], num_classes=K)
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    b = dict(b, protein_pos=pp, init_ligand_pos=lp)
    for steps in ([0, 999, 417], [1, 500, 13], [998, 3, 250]) if time_emb else (None,):
        t = None if steps is None else torch.tensor(steps)
        kw = {} if t is None else {'time_step': t.to(DEV)}
        out = model(*_args(b), **kw)
        h = out['final_h'].cpu()
        h64, lig = layerwise.embedding(sd, cfg, b, t)
        h32, _ = layerwise.embedding(sd, cfg, b, t, dtype=torch.float32)
        assert torch.equal(h[lig, -1], torch.ones(int(lig.sum()))) and torch.equal(h[~lig, -1], torch.zeros(int((~lig).sum())))
        e = [float((x.double() - h64)[rows].abs().max()) for x in (h, h32) for rows in (~lig, lig)]
        print('embedding K=%-2d t=%-15s engine: protein %.2e ligand %.2e   fp32 oracle: protein %.2e ligand %.2e' % ((K, steps) + tuple(e)))
        assert max(e[:2]) <= EMBED_TOL, e


# ------------------------------------------------------------------------------------------------ c. type head
def _head_errors(sd, lig_h, logits):
    """(engine error, fp32 oracle error) of the logits of head(lig_h), each max |logit - ref64| / (|W2| |y64| + |b2|)."""
    ref64 = layerwise.head(sd, lig_h)
    ref32 = layerwise.head(sd, lig_h, dtype=torch.float32)
    w1, b1 = sd['v_inference.0.weight'].double(), sd['v_inference.0.bias'].double()
    y = torch.nn.functional.softplus(lig_h.double() @ w1.T + b1) - LN2_F32
    scale = y.abs() @ sd['v_inference.2.weight'].double().abs().T + sd['v_inference.2.bias'].double().abs()
    err = lambda x: float(((x.double() - ref64).abs() / scale).max())
    return err(logits), err(ref32)


def _scaled_head(sd, lig_h, span=40.0):
    """The head's first Linear scaled so that its pre-activations on `lig_h` reach +-span."""
    z = lig_h.double() @ sd['v_inference.0.weight'].double().T + sd['v_inference.0.bias'].double()
    g = span / float(z.abs().max())
    sd = dict(sd, **{'v_inference.0.weight': sd['v_inference.0.weight'] * g, 'v_inference.0.bias': sd['v_inference.0.bias'] * g})
    return sd, z * g


@pytest.mark.parametrize('K', [8, 13, 23])
def test_head_vs_float64(K):
    """pred_ligand_v against the float64 head on the engine's own final_ligand_h, with synthetic weights and with the first Linear
    scaled so that its pre-activations span +-40 (identity branch above 20, log1p(exp z) below, exp z underflowing next to ln 2);
    layer_pred_ligand_v[0] of return_all (the head on the embedding) against the float64 head on the float64 embedding."""
    model, sd = _model(K)
    b = synth.make_batch(5, 3, n_protein=60, ligand_sizes=[14, 9, 30], num_classes=K)
    out = model(*_args(b), return_all=True)
    lig_h = out['final_ligand_h'].cpu()
    e = _head_errors(sd, lig_h, out['pred_ligand_v'].cpu())
    h64, lig = layerwise.embedding(sd, None, b)
    e0 = _head_errors(sd, h64[lig], out['layer_pred_ligand_v'][0].cpu())
    sd2, z = _scaled_head(sd, lig_h)
    assert (z > 20).sum() > 100 and ((z > -20) & (z < 20)).sum() > 100 and (z < -20).sum() > 100
    out2 = _make(K, None, sd2)(*_args(b))
    assert torch.equal(out2['final_ligand_h'].cpu(), lig_h)
    e2 = _head_errors(sd2, lig_h, out2['pred_ligand_v'].cpu())
    print('head K=%-2d  engine / fp32 oracle: synthetic %.2e / %.2e   head(embedding) %.2e / %.2e   +-40 %.2e / %.2e' % ((K,) + e + e0 + e2))
    assert max(e[0], e0[0], e2[0]) <= HEAD_TOL, (e, e0, e2)


# pre-activations the probe head evaluates: both sides of the threshold 20, of z = 10, where log1p(exp z) - z is 4.5e-5, and far out
PROBE_Z = sorted(set(np.round(np.linspace(-40.0, 40.0, 81), 6).tolist()) |
                 {-88.0, -87.0, -17.5, -1e-3, 1e-3, 9.99, 10.01, 10.5, 11.0, 12.0, 13.5, 15.0, 17.0, 19.5, 19.99, 19.999, 20.001, 20.01, 88.0})


def test_head_softplus_probe_vs_float64():
    """A probe head: W1 = 0, b1 = the probe pre-activations, W2 selects one hidden unit per class, b2 = 0.  Each logit is then
    softplus(z) - ln 2 of one z, computed by the kernel with nothing else rounded into it (a sum of zeros and one term).  K = 23,
    as many heads as the probes need; every ligand atom of a ragged batch must give the same value."""
    K = 23
    _, sd = _model(K)
    b = synth.make_batch(6, 2, n_protein=40, ligand_sizes=[5, 11], num_classes=K)
    zs = torch.tensor(PROBE_Z, dtype=torch.float32)
    worst = worst32 = 0.0
    for i in range(0, len(zs), K):
        chunk = zs[i:i + K]
        b1 = torch.zeros(128)
        b1[:len(chunk)] = chunk
        w2 = torch.zeros(K, 128)
        w2[torch.arange(len(chunk)), torch.arange(len(chunk))] = 1.0
        sdp = dict(sd, **{'v_inference.0.weight': torch.zeros(128, 128), 'v_inference.0.bias': b1, 'v_inference.2.weight': w2,
                          'v_inference.2.bias': torch.zeros(K)})
        logits = _make(K, None, sdp)(*_args(b))['pred_ligand_v'].cpu()[:, :len(chunk)]
        assert torch.equal(logits, logits[:1].expand_as(logits))
        z = chunk.double()
        sp = torch.where(z > 20, z, torch.log1p(torch.exp(z)))
        ulp = lambda y: (y.double() - (sp - LN2_F32)).abs() / (EPS32 * (sp.abs() + LN2_F32))
        ulps = ulp(logits[0])
        worst = max(worst, float(ulps.max()))
        worst32 = max(worst32, float(ulp(torch.nn.functional.softplus(chunk) - LN2_F32).max()))
        assert float(ulps.max()) <= PROBE_ULPS, {float(a): float(u) for a, u in zip(chunk, ulps) if u > PROBE_ULPS}
    print('head softplus probe: %d pre-activations, engine %.2f ulp, fp32 oracle %.2f ulp' % (len(zs), worst, worst32))


# ------------------------------------------------------------------------------------------------ d. global edge gate
def _gate_inputs(k, saturate):
    from targetdiff_b200.pocket import pdb_to_pocket_data
    data = pdb_to_pocket_data(PDB_1H36)
    sizes = [20, 13]
    n_prot = data.protein_pos.shape[0]
    g = torch.Generator().manual_seed(5)
    b = {'protein_pos': data.protein_pos.repeat(2, 1), 'protein_v': data.protein_atom_feature.float().repeat(2, 1),
         'batch_protein': torch.repeat_interleave(torch.arange(2), n_prot),
         'batch_ligand': torch.repeat_interleave(torch.arange(2), torch.tensor(sizes))}
    b['init_ligand_pos'] = data.protein_pos.mean(0, keepdim=True) + 1.5 * torch.randn(sum(sizes), 3, generator=g)
    b['init_ligand_v'] = torch.randint(0, 13, (sum(sizes),), generator=g)
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    b.update(protein_pos=pp, init_ligand_pos=lp)
    cfg = {'knn': k}
    sd = synth.make_state_dict(0, cfg, schedules=restate.make_schedules(cfg))
    if saturate:        # gate logits over about +-20: the sigmoid within 3e-8 of 0 and 2e-9 of 1
        sd['refine_net.edge_pred_layer.net.3.weight'] = sd['refine_net.edge_pred_layer.net.3.weight'] * 40
        sd['refine_net.edge_pred_layer.net.3.bias'] = sd['refine_net.edge_pred_layer.net.3.bias'] * 40 - 20
    return cfg, sd, b


@pytest.mark.parametrize('saturate', [False, True], ids=['synthetic', 'saturated'])
@pytest.mark.parametrize('k', [8, 32, 48])
def test_global_gate_vs_float64(k, saturate):
    """return_edge_weight against layerwise.global_edge_weight in float64 on the engine's own graph and block-0 coordinates."""
    cfg, sd, b = _gate_inputs(k, saturate)
    out = _make(13, cfg, sd)(*_args(b), return_edge_weight=True)
    ei, ew = out['edge_index'].cpu(), out['edge_weight'].cpu()
    _, x, _, _ = restate.compose_context(torch.zeros(len(b['protein_pos']), 1), torch.zeros(len(b['init_ligand_pos']), 1),
                                         b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    ref64 = layerwise.global_edge_weight(sd, x, ei)
    ref32 = layerwise.global_edge_weight(sd, x, ei, dtype=torch.float32)
    e, o = float((ew.double() - ref64).abs().max()), float((ref32.double() - ref64).abs().max())
    print('gate k=%-2d %-10s range %.2e .. %.6f   engine %.2e   fp32 oracle %.2e' % (k, 'saturated' if saturate else '',
                                                                                    float(ref64.min()), float(ref64.max()), e, o))
    if saturate:
        assert float(ref64.min()) < 1e-6
    assert e <= (GATE_TOL_SATURATED if saturate else GATE_TOL)


# ------------------------------------------------------------------------------------------------ e, f. later blocks, return_all
BLOCK_CASES = [({}, 1, 4), ({'ew_net_type': 'r'}, 1, 4), ({'cutoff_mode': 'hybrid', 'knn': 8}, 1, 4), ({}, 3, 2)]


def _bid(case):
    cfgd, L, B = case
    return ','.join(['%s=%s' % kv for kv in cfgd.items()] + ['layers=%d' % L, 'blocks=%d' % B])


@pytest.mark.parametrize('case', BLOCK_CASES, ids=_bid)
def test_later_blocks_vs_float64_and_return_all(case):
    """For b = 1 .. B: the engine's output of b - 1 blocks (b = 1: the float64 embedding and the initial coordinates) through
    layerwise.block in float64 against the engine's output of b blocks: its edge_index equals the graph rebuilt from the engine's
    own coordinates (as an edge set for hybrid), h and x within the per-layer limits (LAYER_TOL).  Entry b of the B-block network's
    return_all lists equals the b-block network's output bit for bit (entry 0: the input coordinates)."""
    torch.set_num_threads(16)
    cfgd, L, B = case
    cfg = dict(cfgd, num_layers=L)
    sd = synth.make_state_dict(4, cfg, schedules=restate.make_schedules(cfg))
    b = synth.make_batch(12, 3, n_protein=80, ligand_sizes=[11, 3, 17])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    b = dict(b, protein_pos=pp, init_ligand_pos=lp)
    h, lig = layerwise.embedding(sd, cfg, b)
    _, x, batch_all, _ = restate.compose_context(torch.zeros(len(pp), 1), torch.zeros(len(lp), 1), pp, lp, b['batch_protein'], b['batch_ligand'])
    full = _make(13, dict(cfg, num_blocks=B), sd)(*_args(b), return_all=True)
    assert len(full['layer_pred_ligand_pos']) == len(full['layer_pred_ligand_v']) == B + 1
    assert torch.equal(full['layer_pred_ligand_pos'][0].cpu(), lp)
    hybrid = cfg.get('cutoff_mode') == 'hybrid'
    rows = []
    for nb in range(1, B + 1):
        out = _make(13, dict(cfg, num_blocks=nb), sd)(*_args(b))
        assert torch.equal(full['layer_pred_ligand_pos'][nb], out['pred_ligand_pos']), nb
        assert torch.equal(full['layer_pred_ligand_v'][nb], out['pred_ligand_v']), nb
        h64, x64, ei64, _ = layerwise.block(sd, cfg, h, x, lig, batch_all)
        h32, x32, _, _ = layerwise.block(sd, cfg, h, x, lig, batch_all, dtype=torch.float32)
        ei = out['edge_index'].cpu()
        if hybrid:
            assert torch.equal(layerwise._sorted_edges(ei), layerwise._sorted_edges(ei64)), nb
        else:
            assert torch.equal(ei, ei64), nb
        h_gpu = out['final_h'].cpu()
        x_gpu = x.clone()
        x_gpu[lig] = out['pred_ligand_pos'].cpu()
        r = (nb,) + layerwise.summary(layerwise.row_error(h_gpu, h64, h)) + layerwise.summary(layerwise.row_error(x_gpu, x64, x, lig)) + \
            layerwise.summary(layerwise.row_error(h32, h64, h)) + layerwise.summary(layerwise.row_error(x32, x64, x, lig))
        print('%-34s block %d  h %.2e / %.2e  x %.2e / %.2e   fp32 oracle: h %.2e / %.2e  x %.2e / %.2e' % ((_bid(case),) + r))
        rows.append(r)
        h, x = h_gpu, x_gpu
    layerwise.check_layers(rows, k=cfg.get('knn', 32))
