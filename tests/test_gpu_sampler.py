"""The step epilogue (`step_epilogue_kernel`, targetdiff_b200/csrc/sampler.cu) against exact arithmetic, and its device random
stream against the host restatement (run with -m gpu; `pytest -s` prints the per-step error tables).

A. The device stream equals oracle/philox.py.  A chain run with `seed=` and the same chain run on `philox.engine_tape(seed, ...)`
   must draw the same atom types at every step (the uniforms are exact) and positions within a few ulps at the first step (the
   tape's normals are float64 rounded once, the kernel's are fp32 logf / sqrtf / cospif / sinpif).  Seeds with and without a high
   key word, S on both sides of the eager / CUDA-graph boundary (S > 2 replays a captured step), a ragged batch of more than one
   128-atom block, K = 13 (the last 4-lane Philox block is partly used), pos_only.
B. Each step against float64.  A chain on a noise tape with center_pos_mode='none' and the pocket at the origin: the engine's
   offset is zero, so pos_traj[s] is the state itself (step 0, whose input is the caller's initial state, checks that).  For
   chosen steps, x0 and the logits come from a stand-alone forward on that step's input state; `oracle.stepwise.step` in float64
   on the same inputs is the reference.  Errors: positions per coordinate relative to |c0 x0| + |ct xt| + |sigma noise|, v0 and
   vt absolute, v equal wherever the float64 Gumbel margin exceeds MARGIN.  The fp32 oracle's own error is printed beside it.
C. The device noise's distribution, without the restatement: one step on 10^4 atoms with the seed and with a zero position tape
   gives the noise as (pos_seed - pos_zero) / sigma_{T-1}; moments, KS, cross-coordinate and squared-coordinate correlations,
   neighbouring atoms.  The sampled types against the step's posterior (vt at step 0 does not depend on the noise)."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import philox, restate, stepwise, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K = synth.LIGAND_NUM_CLASSES
Z_MAX, P_MIN = 5.0, 1e-6
# Limits of A (philox.STREAM_ULPS, STREAM_LATER_REL) and B (stepwise.STEP_TOL), with the measured maxima behind them: oracle/philox.py
# and oracle/stepwise.py.


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
    return tuple(b[k].to(dev) for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))


def _sigma(sd, t):
    return math.exp(0.5 * float(sd['posterior_logvar'][t])) if t > 0 else 0.0


# ------------------------------------------------------------------------------------------------ A. device stream == engine_tape
@pytest.fixture(scope='module')
def stream_setup():
    model, sd = _model()
    b = synth.make_batch(31, 4, n_protein=50, ligand_sizes=[60, 45, 33, 37])     # 175 atoms: two blocks, the second partly used
    return model, sd, b


def _stream_case(setup, seed, S, pos_only):
    model, sd, b = setup
    n = len(b['batch_ligand'])
    assert n > 128 and n % 128
    kw = dict(num_steps=S, center_pos_mode='protein', pos_only=pos_only, stack_traj=True)
    dev = model.sample_diffusion(*_args(b), seed=seed, **kw)
    pn, vu = philox.engine_tape(seed, n, S, K, pos_only=pos_only)
    tape = model.sample_diffusion(*_args(b), noise_tape=(pn, vu), **kw)
    assert torch.equal(dev['v_traj'], tape['v_traj'])
    if pos_only:
        assert torch.equal(dev['v_traj'][-1], b['init_ligand_v'])
    else:
        assert torch.equal(dev['v0_traj'][0], tape['v0_traj'][0]) and torch.equal(dev['vt_traj'][0], tape['vt_traj'][0])
    T = sd['betas'].shape[0]
    ulps, later = philox.stream_errors(dev['pos_traj'], tape['pos_traj'], pn[0], _sigma(sd, T - 1))
    print('stream seed=%-20d S=%d pos_only=%d  step 0: %.2f ulp  later steps: %.2e rel' % (seed, S, pos_only, ulps, later))
    assert ulps <= philox.STREAM_ULPS and later <= philox.STREAM_LATER_REL, (ulps, later)


@pytest.mark.parametrize('S', [1, 2, 3, 7])
@pytest.mark.parametrize('seed', [0, 123, 2 ** 32 + 7, 2 ** 62 - 1])
def test_device_stream_is_engine_tape(stream_setup, seed, S):
    _stream_case(stream_setup, seed, S, False)


@pytest.mark.parametrize('seed,S', [(2 ** 32 + 7, 3), (123, 2)])
def test_device_stream_is_engine_tape_pos_only(stream_setup, seed, S):
    _stream_case(stream_setup, seed, S, True)


# ------------------------------------------------------------------------------------------------ B. each step vs float64
def _centred_batch(seed, sizes, n_protein=60):
    """A batch with the pocket(s) at the origin: in center_pos_mode='none' the network then sees the coordinates the default
    mode would give it (it is not translation invariant without centring)."""
    b = synth.make_batch(seed, len(sizes), n_protein=n_protein, ligand_sizes=sizes, distinct_pockets=1)
    shift = b['protein_pos'].mean(0, keepdim=True)
    b['protein_pos'] = b['protein_pos'] - shift
    b['init_ligand_pos'] = b['init_ligand_pos'] - shift
    return b


def _steps_vs_float64(label, cfg, S, check, pos_only=False, seed=41):
    model, sd = _model(cfg)
    b = _centred_batch(seed, [9, 14])
    pn, vu = synth.make_tape(seed, S, len(b['batch_ligand']))
    rows = stepwise.engine_steps_vs_float64(label, model, sd, cfg, b, pn, vu, check, DEV, pos_only=pos_only)
    stepwise.check_steps(label, rows)
    return rows


STEP_CASES = {
    'T2': ({'num_diffusion_timesteps': 2}, 2, None, False),
    'T20': ({'num_diffusion_timesteps': 20}, 20, None, False),
    'T1000': (None, 1000, [0, 1, 500, 997, 998, 999], False),
    'T20_noise_mean': ({'num_diffusion_timesteps': 20, 'model_mean_type': 'noise'}, 20, None, False),
    'T1000_noise_mean': ({'model_mean_type': 'noise'}, 3, None, False),
    'T20_pos_only': ({'num_diffusion_timesteps': 20}, 20, None, True),
    'T20_time_emb': ({'num_diffusion_timesteps': 20, 'time_emb_dim': 1, 'time_emb_mode': 'simple'}, 20, None, False),
}


@pytest.mark.parametrize('name', list(STEP_CASES))
def test_each_step_vs_float64(name):
    cfg, S, check, pos_only = STEP_CASES[name]
    _steps_vs_float64(name, cfg, S, range(S) if check is None else check, pos_only=pos_only)


# ------------------------------------------------------------------------------------------------ C. device noise distribution
def _z_corr(a, b):
    return float(np.corrcoef(a.ravel(), b.ravel())[0, 1]) * math.sqrt(a.size)


def test_device_noise_distribution():
    """One step on 10^4 atoms: the device's position noise is N(0, 1) per coordinate, independent across coordinates (and their
    squares) and neighbouring atoms; the sampled types follow the step's posterior."""
    model, sd = _model()
    T = sd['betas'].shape[0]
    b = synth.make_batch(51, 20, n_protein=60, n_ligand=500)
    n = len(b['batch_ligand'])
    seed = 2 ** 40 + 12345
    r1 = model.sample_diffusion(*_args(b), num_steps=1, center_pos_mode='protein', seed=seed, stack_traj=True)
    zero = (torch.zeros(1, n, 3), torch.full((1, n, K), 0.5))
    r0 = model.sample_diffusion(*_args(b), num_steps=1, center_pos_mode='protein', noise_tape=zero, stack_traj=True)
    assert torch.equal(r1['vt_traj'], r0['vt_traj'])
    nz = ((r1['pos_traj'][0].double() - r0['pos_traj'][0].double()) / _sigma(sd, T - 1)).numpy()
    for d in range(3):
        x = nz[:, d]
        assert abs(x.mean()) * math.sqrt(n) <= Z_MAX, d
        assert abs(x.var() - 1.0) / math.sqrt(2.0 / n) <= Z_MAX, d
        assert stats.kstest(x, 'norm').pvalue >= P_MIN, d
        assert abs(_z_corr(x[1:], x[:-1])) <= Z_MAX, d
    for i, j in ((0, 1), (0, 2), (1, 2)):
        assert abs(_z_corr(nz[:, i], nz[:, j])) <= Z_MAX, (i, j)
        assert abs(_z_corr(nz[:, i] ** 2, nz[:, j] ** 2)) <= Z_MAX, (i, j)
    p = r1['vt_traj'][0].double().exp()
    v = r1['v_traj'][0]
    z = []
    for c in range(K):
        var = float((p[:, c] * (1 - p[:, c])).sum())
        if var > 1.0:
            z.append((int((v == c).sum()) - float(p[:, c].sum())) / math.sqrt(var))
    print('device noise: %d atoms, type count z scores %s' % (n, ' '.join('%.2f' % x for x in z)))
    assert len(z) >= 3 and max(abs(x) for x in z) <= Z_MAX
