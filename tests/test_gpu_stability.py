"""The stability screen (`check_stability_kernel`, targetdiff_b200/csrc/stability.cu) at its bond-length thresholds and at shapes the
random test never reaches, and the atom-type draw of the step epilogue and of fixed rows (targetdiff_b200/csrc/sampler.cu) at exact
ties (run with -m gpu).

A. Every boundary pair and molecule of oracle/stability_cases.py against what the unmodified reference returned on the same float64
   positions (tests/golden/reference_pins_stability_thresholds.pt): molecule flags, stable counts, atom counts and per-atom bond
   counts bit for bit, as one batch and one molecule at a time.  The 'fma' pairs fail a kernel whose squared distance is contracted.
B. Shapes against `restate.check_stability`: about 1000 ragged molecules with empty ones among them, molecules of 31, 32, 33, 64 and
   65 atoms (the lane loop's boundaries), one of 600 atoms.  An unknown element refuses the batch and leaves the device usable; positions
   that are not fp32 values are refused instead of being rounded.
C. Exact ties in the Gumbel-max draws.  The reference's argmax returns the first maximal index, and so must the kernels' strict `>`.
   Step: the type head's last Linear has identical rows for two or three classes, so their logits and posteriors are identical, and
   the tape gives them equal uniforms at chosen atoms and steps.  Fixed rows: every class other than v0_f has the same log-probability,
   and the fixed tape gives two of them equal uniforms.  Every other draw of both tapes has one class ahead by a Gumbel margin of about
   15, so the whole chain is compared without a margin filter."""
import numpy as np
import pytest
import torch

from oracle import fixed_atoms, make_class_count_pins as ccp, make_stability_pins as msp, restate, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ELEMENT_Z = [1, 6, 7, 8, 9, 15, 16, 17]
ELEMENT_P = [0.1, 0.5, 0.12, 0.15, 0.03, 0.02, 0.05, 0.03]


@pytest.fixture(scope='module')
def pins():
    return torch.load(msp.OUT, weights_only=True)


def _split(pins):
    cuts = np.cumsum([0] + pins['counts'].tolist())
    pos, z = pins['pos'].numpy(), pins['z'].numpy()
    return [pos[a:b] for a, b in zip(cuts[:-1], cuts[1:])], [z[a:b] for a, b in zip(cuts[:-1], cuts[1:])], cuts


# ------------------------------------------------------------------------------------------------ A. boundary pairs vs the reference
@pytest.mark.parametrize('hs', [False, True])
def test_boundary_cases_equal_reference_pins(pins, hs):
    from targetdiff_b200 import analyze
    pos, zs, cuts = _split(pins)
    want = pins['result'][:, int(hs)].numpy()
    want_nb = pins['nr_bonds'][:, int(hs)].numpy()
    ms, ns, na, nb = analyze.check_stability_batch(pos, zs, hs=hs)
    got = np.stack([ms.astype(np.int64), ns, na], 1)
    bad = [pins['names'][m] for m in range(len(pos)) if not (np.array_equal(got[m], want[m]) and
                                                             np.array_equal(nb[cuts[m]:cuts[m + 1]], want_nb[cuts[m]:cuts[m + 1]]))]
    assert not bad, 'batch, hs=%s: %d cases differ from the reference: %s' % (hs, len(bad), ' '.join(bad))
    bad = []
    for m in range(len(pos)):
        one = analyze.check_stability(pos[m], zs[m], hs=hs, return_nr_bonds=True)
        if [int(one[0]), one[1], one[2]] != want[m].tolist() or not np.array_equal(one[3], want_nb[cuts[m]:cuts[m + 1]]):
            bad.append(pins['names'][m])
    assert not bad, 'one at a time, hs=%s: %d cases differ from the reference: %s' % (hs, len(bad), ' '.join(bad))


# ------------------------------------------------------------------------------------------------ B. shapes, errors, input contract
def _molecule(rng, n):
    pos = np.cumsum(rng.normal(scale=0.85, size=(n, 3)), axis=0) + rng.uniform(-30, 30, size=(1, 3))
    return pos.astype(np.float32).astype(np.float64), rng.choice(ELEMENT_Z, size=n, p=ELEMENT_P)


def _check_against_restatement(pos, zs, hs):
    from targetdiff_b200 import analyze
    ms, ns, na, nb = analyze.check_stability_batch(pos, zs, hs=hs)
    off = 0
    for m, (p, z) in enumerate(zip(pos, zs)):
        w = restate.check_stability(p, z, hs=hs)
        assert (bool(ms[m]), int(ns[m]), int(na[m])) == (bool(w[0]), w[1], w[2]), (m, len(z))
        assert np.array_equal(nb[off:off + len(z)], w[3]), (m, len(z))
        off += len(z)
    assert off == len(nb)


@pytest.mark.parametrize('hs', [False, True])
def test_ragged_batch_with_empty_molecules(hs):
    rng = np.random.RandomState(11)
    sizes = [int(n) for n in rng.randint(1, 40, size=997)]
    for i in range(3, 997, 97):
        sizes[i] = 0                                                 # empty molecules between others
    assert len(sizes) % 8 and sizes[-1] > 0
    pos, zs = zip(*[_molecule(rng, n) for n in sizes])
    _check_against_restatement(list(pos), list(zs), hs)


@pytest.mark.parametrize('hs', [False, True])
def test_lane_loop_boundaries_and_a_large_molecule(hs):
    rng = np.random.RandomState(12)
    pos, zs = zip(*[_molecule(rng, n) for n in (31, 32, 33, 64, 65, 600, 1)])
    _check_against_restatement(list(pos), list(zs), hs)


def test_unknown_element_refuses_the_batch_and_the_device_stays_usable():
    from targetdiff_b200 import _lib, analyze
    rng = np.random.RandomState(13)
    mols = [_molecule(rng, n) for n in (9, 12, 7)]
    pos, zs = [m[0] for m in mols], [m[1].copy() for m in mols]
    zs[1][5] = 5                                                     # boron: not in the reference's table (KeyError there)
    with pytest.raises(_lib.TdiffError, match='outside the reference'):
        analyze.check_stability_batch(pos, zs)
    zs[1][5] = 6
    _check_against_restatement(pos, zs, False)


def test_positions_must_be_fp32_values():
    from targetdiff_b200 import analyze
    rng = np.random.RandomState(14)
    pos, z = _molecule(rng, 20)
    want = analyze.check_stability_batch([pos], [z])
    off = pos.copy()
    off[7, 1] = np.nextafter(off[7, 1], np.inf)                      # one coordinate between two fp32 values
    with pytest.raises(ValueError, match='fp32'):
        analyze.check_stability_batch([off], [z])
    with pytest.raises(ValueError, match='fp32'):
        analyze.check_stability(off, z)
    with pytest.raises(ValueError, match='fp32'):
        analyze.check_stability_batch(torch.from_numpy(off), [z])
    for same in ([pos.astype(np.float32)], torch.from_numpy(pos), torch.from_numpy(pos).float()):   # fp32 values, widened or not
        got = analyze.check_stability_batch(same, [z])
        assert all(np.array_equal(a, b) for a, b in zip(got, want))


# ------------------------------------------------------------------------------------------------ C. exact ties in the type draws
U_WIN = float(np.float32(1.0 - 2.0 ** -24))          # the largest fp32 uniform below 1: Gumbel about 16.6
TIE_SETS = {13: (4, 9), 23: (2, 5, 11)}
TIE_STEPS = (1, 3, 5)
S_TIE = 6


def _decisive_uniforms(rng, shape, winners):
    """Uniforms [..., K] in (1e-6, 0.5) (Gumbel below 0.37) with U_WIN at the classes `winners` [..., K] bool."""
    u = rng.uniform(1e-6, 0.5, size=shape).astype(np.float32)
    u[winners] = U_WIN
    return torch.from_numpy(u)


def step_tie_case(K, seed=0):
    """(sd, batch, tape, tie_atoms): the type head's last Linear has the rows of TIE_SETS[K] equal to the first's (weights and bias).
    On the tape every (step, atom) has one winning class; at steps TIE_STEPS the tie atoms' winners are the whole tied set, and at the
    other steps class 0 or 1, so that the class current before a tie step is never a tied one."""
    tied = list(TIE_SETS[K])
    sd = ccp.weights(seed, K, {})
    for key in ('v_inference.2.weight', 'v_inference.2.bias'):
        sd[key][tied[1:]] = sd[key][tied[0]].clone()
    b = synth.make_batch(seed + 101, 2, n_protein=60, ligand_sizes=[9, 14], num_classes=K)
    n = len(b['batch_ligand'])
    tie_atoms = np.arange(0, n, 3)
    b['init_ligand_v'][tie_atoms] = 0
    rng = np.random.RandomState(seed + 102)
    win = np.zeros((S_TIE, n, K), dtype=bool)
    win[np.arange(S_TIE)[:, None], np.arange(n)[None, :], rng.randint(0, K, size=(S_TIE, n))] = True
    for s in range(S_TIE):
        win[s, tie_atoms] = False
        if s in TIE_STEPS:
            win[s][np.ix_(tie_atoms, tied)] = True
        else:
            win[s, tie_atoms, s % 2] = True
    pn = torch.from_numpy(rng.normal(size=(S_TIE, n, 3)).astype(np.float32))
    return sd, b, (pn, _decisive_uniforms(rng, (S_TIE, n, K), win)), tie_atoms


def fixed_tie_case(seed=0):
    """(sd, batch, tape, fixed tape, mask, tie rows): K = 13; every draw of the fixed tape gives fixed row a two classes other than
    v0_f (chosen per draw) the same uniform U_WIN, which beats v0_f's class at every draw of the chain."""
    K = synth.LIGAND_NUM_CLASSES
    sd = synth.make_state_dict(seed, schedules=restate.make_schedules())
    b = synth.make_batch(seed + 111, 2, n_protein=60, ligand_sizes=[9, 14])
    n = len(b['batch_ligand'])
    mask = torch.zeros(n, dtype=torch.bool)
    rows = np.array([0, 2, 5, 9, 10, 16])
    mask[rows] = True
    rng = np.random.RandomState(seed + 112)
    win = np.zeros((S_TIE, n, K), dtype=bool)
    win[np.arange(S_TIE)[:, None], np.arange(n)[None, :], rng.randint(0, K, size=(S_TIE, n))] = True
    pn = torch.from_numpy(rng.normal(size=(S_TIE, n, 3)).astype(np.float32))
    tape = (pn, _decisive_uniforms(rng, (S_TIE, n, K), win))
    v0 = b['init_ligand_v'].numpy()
    fwin = np.zeros((S_TIE + 1, n, K), dtype=bool)
    for d in range(S_TIE + 1):
        for a in rows:
            pair = rng.choice([c for c in range(K) if c != v0[a]], size=2, replace=False)
            fwin[d, a, pair] = True
    fpn = torch.from_numpy(rng.normal(size=(S_TIE + 1, n, 3)).astype(np.float32))
    return sd, b, tape, (fpn, _decisive_uniforms(rng, (S_TIE + 1, n, K), fwin)), mask, fwin


def _engine(K, sd):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    m = ScorePosNet3D(default_model_config(), synth.PROTEIN_FEATURE_DIM, K)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')


@pytest.mark.parametrize('K', sorted(TIE_SETS))
def test_step_type_draw_takes_the_lowest_tied_class(K):
    sd, b, (pn, vu), tie_atoms = step_tie_case(K)
    tied = list(TIE_SETS[K])
    r = _engine(K, sd).sample_diffusion(*(b[k].to(DEV) for k in ARGS), num_steps=S_TIE, center_pos_mode='protein',
                                        noise_tape=(pn, vu), stack_traj=True)
    v0, vt, v = r['v0_traj'].cpu(), r['vt_traj'].cpu(), r['v_traj'].cpu()
    # the precondition: the tied classes' log-softmax and posterior are bitwise equal on the engine, at every atom and step
    for c in tied[1:]:
        assert torch.equal(v0[..., c], v0[..., tied[0]]), 'the engine\'s logits of the identical head rows %d and %d differ' % (tied[0], c)
    for s in TIE_STEPS:
        for c in tied[1:]:
            assert torch.equal(vt[s, tie_atoms, c], vt[s, tie_atoms, tied[0]]), 'posteriors of the tied classes differ at step %d' % s
        assert (v[s - 1, tie_atoms] < tied[0]).all()                 # the current class is not a tied one
        assert (v[s, tie_atoms] == tied[0]).all(), 'step %d: the tie went to %s' % (s, v[s, tie_atoms].tolist())
    want = restate.sample_diffusion(sd, None, *(b[k] for k in ARGS), pn, vu, num_steps=S_TIE)
    assert torch.equal(v, torch.stack(want['v_traj']))                # every atom, every step: no margin filter


def test_fixed_row_type_draw_takes_the_lower_tied_class():
    sd, b, tape, ft, mask, fwin = fixed_tie_case()
    K = synth.LIGAND_NUM_CLASSES
    r = _engine(K, sd).sample_diffusion(*(b[k].to(DEV) for k in ARGS), num_steps=S_TIE, center_pos_mode='protein',
                                        noise_tape=tape, stack_traj=True, fixed_mask=mask.to(DEV), fixed_noise_tape=ft)
    v = r['v_traj'].cpu()
    lower = torch.from_numpy(fwin.argmax(-1))                        # the first tied class of each draw
    for s in range(S_TIE):                                           # draw s + 1 after step s
        assert torch.equal(v[s][mask], lower[s + 1][mask]), 'step %d: %s, want %s' % (s, v[s][mask].tolist(), lower[s + 1][mask].tolist())
    want = fixed_atoms.sample_diffusion(sd, None, *(b[k] for k in ARGS), *tape, mask, ft, num_steps=S_TIE)
    assert torch.equal(v, torch.stack(want['v_traj']))
