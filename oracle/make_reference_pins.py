"""Run the UNMODIFIED reference (under oracle/shims) on the cases of tests/test_oracle_vs_reference.py and store what it returns in
tests/golden/reference_pins.pt, so that the restatement is pinned against the reference on any machine.

    TARGETDIFF_REFERENCE=<reference checkout> python -m oracle.make_reference_pins
"""
import os

import torch

from oracle import refload, restate, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'reference_pins.pt')
POCKET = os.path.join(ROOT, 'tests', 'golden', '1h36_pocket10.pdb')

OPTION_CONFIGS = [{'num_blocks': 2}, {'ew_net_type': 'r'}, {'ew_net_type': 'm'}, {'ew_net_type': 'none'}, {'x2h_out_fc': True},
                  {'time_emb_dim': 1, 'time_emb_mode': 'simple'}, {'num_blocks': 2, 'ew_net_type': 'r', 'x2h_out_fc': True, 'time_emb_dim': 1},
                  {'cutoff_mode': 'hybrid'}, {'cutoff_mode': 'hybrid', 'knn': 8, 'num_blocks': 2}]
LIKELIHOOD_STEPS = [[0, 999], [417, 3], None]
STABILITY_SIZES = (1, 2, 9, 25, 40)
# torch-CPU reductions split their work by thread count: one thread makes the bits independent of the machine's core count
THREADS = 1


def digest(x):
    """Bit-exact fingerprint of a tensor (dtype, shape, bytes) or of a list of state_dict keys."""
    import hashlib
    h = hashlib.sha256()
    if isinstance(x, torch.Tensor):
        x = x.detach().contiguous().cpu()
        h.update(('%s %s ' % (x.dtype, tuple(x.shape))).encode())
        h.update(x.view(-1).view(torch.uint8).numpy().tobytes() if x.numel() else b'')
    else:
        h.update(repr(x).encode())
    return 'sha256:' + h.hexdigest()


def pin(x):
    """What is stored for a reference output: small tensors as they are, large ones and key lists as their digest."""
    if isinstance(x, torch.Tensor):
        return x.clone() if x.numel() <= 256 else digest(x)
    if isinstance(x, dict):
        return {k: pin(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)) and x and all(isinstance(v, str) or isinstance(v, tuple) for v in x):
        return digest(list(x))
    if isinstance(x, (list, tuple)):
        return [pin(v) for v in x]
    return x


def equal(got, pinned):
    """Bit-exact comparison of a restated output with a stored pin."""
    if isinstance(pinned, str) and pinned.startswith('sha256:'):
        return digest(got if isinstance(got, torch.Tensor) else list(got)) == pinned
    if isinstance(pinned, torch.Tensor):
        return torch.equal(got, pinned)
    if isinstance(pinned, list):
        return len(got) == len(pinned) and all(equal(g, p) for g, p in zip(got, pinned))
    return got == pinned


def option_id(cfgd):
    return ','.join('%s=%s' % kv for kv in cfgd.items())


def _chain(model, seed, batch_seed, n_protein, sizes, tape_seed, tape_atoms=None):
    sd = synth.make_state_dict(seed, schedules=restate.make_schedules())
    model.load_state_dict(sd, strict=True)
    b = synth.make_batch(batch_seed, 2, n_protein=n_protein, ligand_sizes=sizes)
    pn, vu = synth.make_tape(tape_seed, 3, tape_atoms or len(b['batch_ligand']))
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    with torch.no_grad(), refload.noise_tape(pn, vu):
        r = model.sample_diffusion(*args, num_steps=3, center_pos_mode='protein')
    return {k: r[k] for k in ('pos', 'v', 'pos_traj', 'v_traj', 'v0_traj', 'vt_traj')}


def make():
    import numpy as np
    ref = refload.import_reference()
    cfg = refload.default_model_config()
    pins = {'model_config': dict(cfg)}
    model = ref.ScorePosNet3D(cfg, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES).eval()
    sd0 = model.state_dict()
    pins['state_dict_layout'] = [(k, tuple(v.shape)) for k, v in sd0.items()]
    pins['state_dict_size'] = len(sd0)
    pins['schedules'] = {k: sd0[k].clone() for k in synth.SCHEDULE_KEYS}

    sd = synth.make_state_dict(0, schedules=restate.make_schedules())
    model.load_state_dict(sd, strict=True)
    b = synth.make_batch(1, 2, n_protein=60, ligand_sizes=[9, 7])
    with torch.no_grad():
        pp, lp, _ = ref.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
        want = model(pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'])
    pins['forward'] = {'protein_pos': pp, 'ligand_pos': lp, **{k: want[k] for k in ('pred_ligand_pos', 'pred_ligand_v', 'final_h', 'final_ligand_h')}}

    pins['chain'] = _chain(model, 3, 2, 48, [8, 6], 7)

    pins['likelihood'] = {}
    sd = synth.make_state_dict(5, schedules=restate.make_schedules())
    model.load_state_dict(sd, strict=True)
    b = synth.make_batch(4, 2, n_protein=52, ligand_sizes=[7, 10])
    pn, vu = synth.make_tape(9, 1, len(b['batch_ligand']))
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    for steps in LIKELIHOOD_STEPS:
        t = torch.tensor(steps) if steps is not None else torch.full((2,), 1000)
        with torch.no_grad(), refload.noise_tape(pn, vu):
            pins['likelihood'][str(steps)] = list(model.likelihood_estimation(*args, time_step=t))

    cfg_n = refload.default_model_config()
    cfg_n.update({'model_mean_type': 'noise'})
    model_n = ref.ScorePosNet3D(cfg_n, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES).eval()
    pins['chain_noise'] = _chain(model_n, 6, 8, 48, [8, 6], 7)

    pins['options'] = {}
    for cfgd in OPTION_CONFIGS:
        c = refload.default_model_config()
        c.update(cfgd)
        m = ref.ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES).eval()
        sd = synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd))
        m.load_state_dict(sd, strict=True)
        b = synth.make_batch(3, 2, n_protein=60, ligand_sizes=[9, 7])
        pn, vu = synth.make_tape(5, 3, 16)
        args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
        with torch.no_grad(), refload.noise_tape(pn, vu):
            r = m.sample_diffusion(*args, num_steps=3, center_pos_mode='protein')
        pins['options'][option_id(cfgd)] = {'keys': list(m.state_dict().keys()),
                                            **{k: r[k] for k in ('pos', 'v', 'pos_traj', 'v0_traj', 'vt_traj')}}

    sd_mod, sfp = refload.import_reference_scripts()
    import utils.misc as misc
    import utils.transforms as trans
    data = trans.FeaturizeProteinAtom()(sfp.pdb_to_pocket_data(POCKET))
    sd = synth.make_state_dict(0, schedules=restate.make_schedules())
    model = ref.ScorePosNet3D(refload.default_model_config(), synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES).eval()
    model.load_state_dict(sd, strict=True)
    misc.seed_all(2021)
    out = sd_mod.sample_diffusion_ligand(model, data, 3, batch_size=2, device='cpu', num_steps=2, center_pos_mode='protein', sample_num_atoms='prior')
    pins['driver'] = {'protein_pos': data.protein_pos, 'protein_atom_feature': data.protein_atom_feature,
                      'outputs': [[torch.from_numpy(np.asarray(x)) for x in a] for a in out[:6]]}

    import importlib
    analyze = importlib.import_module('utils.evaluation.analyze')
    rng = np.random.RandomState(0)
    pins['stability'] = []
    for n in STABILITY_SIZES:
        for hs in (False, True):
            pos = np.cumsum(rng.normal(scale=0.85, size=(n, 3)), axis=0)
            z = rng.choice([1, 6, 7, 8, 9, 15, 16, 17], size=n, p=[0.1, 0.5, 0.12, 0.15, 0.03, 0.02, 0.05, 0.03])
            w = analyze.check_stability(pos, z, hs=hs, return_nr_bonds=True)
            pins['stability'].append({'pos': torch.from_numpy(pos), 'z': torch.from_numpy(z), 'hs': hs,
                                      'result': [bool(w[0]), int(w[1]), int(w[2])], 'nr_bonds': torch.from_numpy(np.asarray(w[3]))})
    likelihood = pins.pop('likelihood')
    pins = pin(pins)
    pins['likelihood'] = likelihood
    return pins


if __name__ == '__main__':
    torch.set_num_threads(THREADS)
    torch.save(make(), OUT)
    print(OUT, os.path.getsize(OUT))
