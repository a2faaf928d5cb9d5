"""The two CPU references of tests/test_gpu_sampler.py, checked on their own (CPU only).

oracle/philox.py restates the engine's device random stream: Philox4x32-10 against the Random123 known-answer vectors, and the
stream at the engine's counter layout against the distributions it is meant to have.  oracle/stepwise.py restates one sampling
step: at fp32 it must be restate.sample_diffusion's loop body bit for bit, and in float64 it must agree with fp32 to fp32 rounding.

The statistical checks use fixed seeds, so every threshold (|z| <= 5, p >= 1e-6) is deterministic."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import philox, restate, stepwise, synth

Z_MAX, P_MIN = 5.0, 1e-6
SEEDS = [12345, 0x0123456789ABCDEF]                    # without and with a high key word
N_ATOMS, N_STEPS = 4096, 256                           # 2^20 (atom, step) pairs, the engine's counter layout
K = synth.LIGAND_NUM_CLASSES


# ------------------------------------------------------------------------------------------------ Philox4x32-10
KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize('ctr,key,want', KAT, ids=['zeros', 'ones', 'pi'])
def test_philox_known_answers(ctr, key, want):
    got = philox.philox4x32_10(*ctr, *key)
    assert tuple(int(w) for w in got) == want
    # vectorised: the same counter in every element of an array
    arr = philox.philox4x32_10(*(np.full(5, c, np.uint32) for c in ctr), *key)
    assert all((w == v).all() and w.dtype == np.uint32 for w, v in zip(arr, want))


def test_engine_tape_layout():
    """engine_tape is the kernel's counter layout: position words from (a, s, 0, 'pst\\0'), class c from word c % 4 of
    (a, s, 1 + c // 4, 'vuni'), key (seed low, seed high), uniforms the top 24 bits of a word."""
    seed, S, n = 2 ** 40 + 99, 3, 7
    pn, vu = philox.engine_tape(seed, n, S, K)
    assert pn.shape == (S, n, 3) and vu.shape == (S, n, K) and pn.dtype == vu.dtype == torch.float32
    a, s = 5, 2
    x, y, z, w = (int(v) for v in philox.philox4x32_10(a, s, 0, 0x70737400, seed & 0xffffffff, seed >> 32))
    u = lambda word: (word >> 8) / 2.0 ** 24
    r0, r2 = math.sqrt(-2 * math.log(1 - u(x))), math.sqrt(-2 * math.log(1 - u(z)))
    want = [r0 * math.cos(2 * math.pi * u(y)), r0 * math.sin(2 * math.pi * u(y)), r2 * math.cos(2 * math.pi * u(w))]
    assert pn[s, a].tolist() == [float(np.float32(v)) for v in want]
    for c in range(K):
        word = int(philox.philox4x32_10(a, s, 1 + c // 4, 0x76756e69, seed & 0xffffffff, seed >> 32)[c % 4])
        assert float(vu[s, a, c]) == u(word)
    pn2, vu2 = philox.engine_tape(seed, n, S, K, pos_only=True)
    assert torch.equal(pn2, pn) and not vu2.any()
    # the last step of a longer chain is the same draw: the stream depends on (seed, atom, step) only
    pn3, vu3 = philox.engine_tape(seed, n + 130, S + 4, K)
    assert torch.equal(pn3[:S, :n], pn) and torch.equal(vu3[:S, :n], vu)


@pytest.fixture(scope='module', params=SEEDS, ids=['seed_low', 'seed_high'])
def stream(request):
    pn, vu = philox.engine_tape(request.param, N_ATOMS, N_STEPS, K)
    return request.param, pn.double().numpy(), vu.double().numpy()


def _z_corr(a, b):
    """Pearson correlation of two samples, as a z score under independence."""
    return float(np.corrcoef(a.ravel(), b.ravel())[0, 1]) * math.sqrt(a.size)


def test_normals_moments_and_ks(stream):
    _, pn, _ = stream
    for d in range(3):
        x = pn[..., d].ravel()
        n = x.size
        assert abs(x.mean()) * math.sqrt(n) <= Z_MAX, d
        assert abs(x.var() - 1.0) / math.sqrt(2.0 / n) <= Z_MAX, d
        assert abs((x ** 4).mean() - 3.0) / math.sqrt(96.0 / n) <= Z_MAX, d                  # Var(x^4) = 105 - 9
        assert stats.kstest(x, 'norm').pvalue >= P_MIN, d


def test_normals_independent(stream):
    """Across coordinates, their squares (a radius shared by two coordinates correlates their squares by 0.5), neighbouring steps
    and neighbouring atoms."""
    _, pn, _ = stream
    for i, j in ((0, 1), (0, 2), (1, 2)):
        assert abs(_z_corr(pn[..., i], pn[..., j])) <= Z_MAX, (i, j)
        assert abs(_z_corr(pn[..., i] ** 2, pn[..., j] ** 2)) <= Z_MAX, (i, j)
    for d in range(3):
        assert abs(_z_corr(pn[1:, :, d], pn[:-1, :, d])) <= Z_MAX, d
        assert abs(_z_corr(pn[:, 1:, d], pn[:, :-1, d])) <= Z_MAX, d


def test_uniforms_range_ks_and_histogram(stream):
    _, _, vu = stream
    assert vu.min() >= 0.0 and vu.max() <= 1.0 - 2.0 ** -24
    assert (vu * 2 ** 24 == np.floor(vu * 2 ** 24)).all()                     # exact multiples of 2^-24
    for c in range(K):
        x = vu[..., c].ravel()
        assert stats.kstest(x, 'uniform').pvalue >= P_MIN, c
        counts = np.bincount((x * 64).astype(np.int64), minlength=64)
        assert stats.chisquare(counts).pvalue >= P_MIN, c
    for c in range(K - 1):                                                    # neighbouring lanes, also across Philox blocks
        assert abs(_z_corr(vu[..., c], vu[..., c + 1])) <= Z_MAX, c
    assert abs(_z_corr(vu[1:, :, 0], vu[:-1, :, 0])) <= Z_MAX
    assert abs(_z_corr(vu[:, 1:, 0], vu[:, :-1, 0])) <= Z_MAX


def test_high_key_word_changes_the_stream():
    """Seeds that differ only in the high word of the key give unrelated streams."""
    n, S = 512, 64
    for lo in (0, 7):
        pa, va = philox.engine_tape(lo, n, S, K)
        for hi in (1, 2 ** 31):
            pb, vb = philox.engine_tape(lo + (hi << 32), n, S, K)
            assert float((va == vb).double().mean()) < 1e-4
            for d in range(3):
                assert abs(_z_corr(pa[..., d].double().numpy(), pb[..., d].double().numpy())) <= Z_MAX
            assert abs(_z_corr(va.double().numpy(), vb.double().numpy())) <= Z_MAX


# ------------------------------------------------------------------------------------------------ one step vs restate
STEP_CASES = {
    'C0': ({}, 3, False),
    'noise_mean': ({'model_mean_type': 'noise'}, 3, False),
    'pos_only': ({}, 3, True),
    'T20_to_t0': ({'num_diffusion_timesteps': 20}, 20, False),
    'T2_noise_mean_pos_only': ({'num_diffusion_timesteps': 2, 'model_mean_type': 'noise'}, 2, True),
}


def _chain(cfg, S, pos_only, seed=3):
    """restate.sample_diffusion with every step's time, input state, network outputs and new positions (centred) recorded."""
    sd = synth.make_state_dict(seed, cfg, schedules=restate.make_schedules(cfg))
    b = synth.make_batch(seed + 2, 2, n_protein=40, ligand_sizes=[7, 10])
    pn, vu = synth.make_tape(seed + 4, S, len(b['batch_ligand']))
    _, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    steps = []
    state = [lp, b['init_ligand_v']]

    def cb(s, t, preds, pos, v):
        steps.append((t, state[0], state[1], preds['pred_ligand_pos'], preds['pred_ligand_v'], pos))
        state[:] = [pos, v]

    r = restate.sample_diffusion(sd, cfg, b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'],
                                 b['init_ligand_v'], b['batch_ligand'], pn, vu, num_steps=S, step_callback=cb, pos_only=pos_only)
    return sd, pn, vu, steps, r


@pytest.mark.parametrize('name', list(STEP_CASES))
def test_stepwise_fp32_is_restate_and_fp64_agrees(name):
    """fp32: the trajectories of restate.sample_diffusion bit for bit.  float64 on the same inputs: positions within 1e-6 of the
    step's scale (fp32 rounds each of the ~4 operations to 6e-8; measured 1.3e-7), log-probabilities within 1e-5 absolute
    (measured 1.4e-6; values down to about -70 have an fp32 ulp of 8e-6), and the same atom types wherever the Gumbel margin
    exceeds 1e-4."""
    cfg, S, pos_only = STEP_CASES[name]
    T = cfg.get('num_diffusion_timesteps', synth.DEFAULT_MODEL_CONFIG['num_diffusion_timesteps'])
    sd, pn, vu, steps, r = _chain(cfg, S, pos_only)
    assert [st[0] for st in steps] == list(range(T - 1, T - 1 - S, -1))
    worst = {'pos': 0.0, 'v0': 0.0, 'vt': 0.0, 'exempt': 0}
    for s, (t, xt, vt, x0, logits, pos_next) in enumerate(steps):
        got = stepwise.step(sd, cfg, t, xt, vt, x0, logits, pn[s], vu[s], pos_only=pos_only)
        assert got['pos'].dtype == torch.float32
        assert torch.equal(got['pos'], pos_next) and torch.equal(got['v'], r['v_traj'][s])
        if not pos_only:
            assert torch.equal(got['v0'], r['v0_traj'][s]) and torch.equal(got['vt'], r['vt_traj'][s])
        ref = stepwise.step(sd, cfg, t, xt, vt, x0, logits, pn[s], vu[s], pos_only=pos_only, dtype=torch.float64)
        assert ref['pos'].dtype == torch.float64 and torch.get_default_dtype() == torch.float32
        e = stepwise.errors(got['pos'], got['v'], got['v0'], got['vt'], ref)
        assert e['v_diff'] == 0, (s, t, e)
        for k in worst:
            worst[k] = max(worst[k], e[k])
    print('%-24s fp32 vs float64: pos %.2e  v0 %.2e  vt %.2e  exempt %d' % (name, worst['pos'], worst['v0'], worst['vt'], worst['exempt']))
    assert worst['pos'] < 1e-6 and worst['v0'] < 1e-5 and worst['vt'] < 1e-5 and worst['exempt'] <= 1, (name, worst)
