"""Ligand class counts other than 13 on the CPU: K = 8 (ligand_atom_mode 'basic') and K = 23 ('full') with and without the time
embedding, the restatement against the unmodified reference (tests/golden/reference_pins_class_counts.pt, made by
oracle/make_class_count_pins.py) bit for bit; the engine's class-lane layout of the device random stream at K = 8, 23 and 24; the
engine's K range; and the checkpoint loader's ligand_atom_mode -> K mapping.  tests/test_gpu_class_counts.py runs the engine at
these K."""
import ctypes
import math

import pytest
import torch

from oracle import philox, restate, synth
from oracle import make_class_count_pins as ccp
from oracle import make_reference_pins as pins_mod
from oracle.make_reference_pins import LIKELIHOOD_STEPS, equal

CASES = [(K, cfgd) for K in ccp.CLASS_COUNTS for cfgd in ccp.CONFIGS]


def _id(case):
    return ccp.case_id(*case)


@pytest.fixture(scope='module')
def pins():
    n = torch.get_num_threads()
    torch.set_num_threads(pins_mod.THREADS)       # the thread count the pins were computed with
    yield torch.load(ccp.OUT, weights_only=True)
    torch.set_num_threads(n)


def test_pins_cover_every_case(pins):
    assert sorted(pins) == sorted(_id(c) for c in CASES)


def test_default_class_count_draws_unchanged():
    """The ligand_dim / num_classes keywords at their default K = 13 consume the generators as before they existed."""
    sd = synth.make_state_dict(0, schedules=restate.make_schedules())
    sd13 = synth.make_state_dict(0, schedules=restate.make_schedules(), ligand_dim=13)
    assert all(torch.equal(sd[k], sd13[k]) for k in sd)
    b, b13 = synth.make_batch(3, 2, n_protein=60, ligand_sizes=[9, 7]), synth.make_batch(3, 2, n_protein=60, ligand_sizes=[9, 7], num_classes=13)
    assert all(torch.equal(b[k], b13[k]) for k in b)


@pytest.mark.parametrize('case', CASES, ids=_id)
def test_class_count_restatement_bit_exact(pins, case):
    """State dict layout, forward, a 3-step chain with all four trajectories, and likelihood_estimation at two time-step vectors
    and at the prior: the restatement equals the reference bit for bit at K = 8 and 23, with and without the time embedding."""
    K, cfgd = case
    want = pins[_id(case)]
    sd = ccp.weights(0, K, cfgd)
    assert equal(list(sd.keys()), want['keys'])
    assert sd['v_inference.2.weight'].shape[0] == K
    assert sd['ligand_atom_emb.weight'].shape[1] == K + cfgd.get('time_emb_dim', 0)
    b, pp, lp, t = ccp.forward_inputs(K)
    got = restate.forward(sd, cfgd, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], time_step=t)
    for k in ('pred_ligand_pos', 'pred_ligand_v', 'final_h', 'final_ligand_h'):
        assert equal(got[k], want['forward'][k]), k
    b, pn, vu = ccp.chain_inputs(K)
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    w = restate.sample_diffusion(sd, cfgd, *args, pn, vu, num_steps=3)
    assert equal(w['pos'], want['chain']['pos']) and equal(w['v'], want['chain']['v'])
    for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
        assert equal(list(w[k]), want['chain'][k]), k
    sd = ccp.weights(5, K, cfgd)
    b, pn, vu = ccp.likelihood_inputs(K)
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    for steps in LIKELIHOOD_STEPS:
        got = restate.likelihood_estimation(sd, cfgd, *args, ccp.likelihood_time_steps(steps), pn[0], vu[0])
        for g, w in zip(got, want['likelihood'][str(steps)]):
            assert g.shape == w.shape == (2,) and torch.equal(g, w), (steps, g, w)


@pytest.mark.parametrize('K', [8, 23, 24])
def test_engine_tape_class_lanes(K):
    """Class c of the device stream is word c % 4 of counter (a, s, 1 + c // 4, 'vuni') whatever K is: K = 8 and 24 fill their last
    4-lane block, 23 leaves one lane of it unused.  A K-class tape is the first K lanes of the 24-class one."""
    seed, S, n = 2 ** 33 + 5, 3, 9
    pn, vu = philox.engine_tape(seed, n, S, K)
    assert vu.shape == (S, n, K)
    u = lambda word: (word >> 8) / 2.0 ** 24
    for a, s in ((0, 0), (8, 2), (3, 1)):
        for c in range(K):
            word = int(philox.philox4x32_10(a, s, 1 + c // 4, 0x76756e69, seed & 0xffffffff, seed >> 32)[c % 4])
            assert float(vu[s, a, c]) == u(word), (a, s, c)
    pn24, vu24 = philox.engine_tape(seed, n, S, 24)
    assert torch.equal(pn, pn24) and torch.equal(vu, vu24[..., :K])
    assert math.ceil(K / 4) == (K + 3) // 4


def _create(num_classes):
    from targetdiff_b200 import _lib
    lib = _lib.load()
    cfg = _lib.tdiff_config(128, 16, 9, 32, 20, num_classes, 27, 1000)
    rc = lib.tdiff_create(ctypes.byref(cfg), (_lib.tdiff_tensor * 1)(), 0, 0, ctypes.byref(ctypes.c_void_p()))
    return rc, lib.tdiff_last_error()


def test_tdiff_create_class_count_range():
    """tdiff_create accepts K = 1 .. 24 (the step epilogue holds the classes in registers, TD_CMAX = 24) and refuses the rest with
    TDIFF_EINVAL before it looks for a device."""
    from targetdiff_b200 import _lib
    for K in (0, 25, -1):
        rc, msg = _create(K)
        assert rc == _lib.TDIFF_EINVAL and b'num_classes=%d' % K in msg, (K, rc, msg)
    for K in (1, 8, 23, 24):       # past the class-count check; on a machine without a device it stops at the device lookup
        rc, msg = _create(K)
        assert b'num_classes' not in msg, (K, rc, msg)


@pytest.mark.parametrize('mode,K', [('basic', 8), ('add_aromatic', 13), ('full', 23)])
def test_load_model_class_count_from_ligand_atom_mode(tmp_path, mode, K):
    """cli._load_model takes K from the checkpoint's data.transform.ligand_atom_mode, like the reference's featuriser
    (scripts/sample_diffusion.py:141-161), and loads the weights strictly: a K-class state dict loads, a 13-class one does not
    unless K = 13."""
    from targetdiff_b200 import cli
    from targetdiff_b200.config import Config
    sd = synth.make_state_dict(2, schedules=restate.make_schedules(), ligand_dim=K)
    ckpt = {'config': Config({'model': dict(synth.DEFAULT_MODEL_CONFIG), 'data': {'transform': {'ligand_atom_mode': mode}}}), 'model': sd}
    path = tmp_path / 'ckpt.pt'
    torch.save(ckpt, path)
    model = cli._load_model(Config({'model': {'checkpoint': str(path)}}), 'cpu')
    assert model.num_classes == K
    got = model.state_dict()
    assert list(got) == list(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    if K != 13:
        ckpt['model'] = synth.make_state_dict(2, schedules=restate.make_schedules())
        torch.save(ckpt, path)
        with pytest.raises(RuntimeError, match='size mismatch'):
            cli._load_model(Config({'model': {'checkpoint': str(path)}}), 'cpu')
