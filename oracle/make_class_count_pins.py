"""Run the UNMODIFIED reference (under oracle/shims) at ligand class counts other than 13 -- K = 8 (ligand_atom_mode 'basic') and
K = 23 ('full'), each without and with time_emb_mode 'simple' -- and store what it returns in tests/golden/reference_pins_class_counts.pt,
so that the restatement is pinned against the reference at those K on any machine.  Same recipe as oracle/make_layer_form_pins.py.

    TARGETDIFF_REFERENCE=<reference checkout> python -m oracle.make_class_count_pins
"""
import os

import torch

from oracle import refload, restate, synth
from oracle.make_reference_pins import LIKELIHOOD_STEPS, THREADS, option_id, pin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'reference_pins_class_counts.pt')

CLASS_COUNTS = (8, 23)
TIME_EMB = {'time_emb_dim': 1, 'time_emb_mode': 'simple'}
CONFIGS = [{}, TIME_EMB]
FORWARD_TIME_STEPS = [500, 17]            # read by the forward only with the time embedding


def case_id(K, cfgd):
    return 'K=%d' % K + (',' + option_id(cfgd) if cfgd else '')


def forward_inputs(K):
    b = synth.make_batch(1, 2, n_protein=60, ligand_sizes=[9, 7], num_classes=K)
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    return b, pp, lp, torch.tensor(FORWARD_TIME_STEPS)


def chain_inputs(K):
    b = synth.make_batch(3, 2, n_protein=60, ligand_sizes=[9, 7], num_classes=K)
    pn, vu = synth.make_tape(5, 3, 16, num_classes=K)
    return b, pn, vu


def likelihood_inputs(K):
    b = synth.make_batch(4, 2, n_protein=52, ligand_sizes=[7, 10], num_classes=K)
    pn, vu = synth.make_tape(9, 1, len(b['batch_ligand']), num_classes=K)
    return b, pn, vu


def likelihood_time_steps(steps):
    return torch.tensor(steps) if steps is not None else torch.full((2,), 1000)


def weights(seed, K, cfgd):
    return synth.make_state_dict(seed, cfgd, schedules=restate.make_schedules(cfgd), ligand_dim=K)


def make():
    ref = refload.import_reference()
    pins = {}
    for K in CLASS_COUNTS:
        for cfgd in CONFIGS:
            c = refload.default_model_config()
            c.update(cfgd)
            m = ref.ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K).eval()
            m.load_state_dict(weights(0, K, cfgd), strict=True)
            entry = {'keys': list(m.state_dict().keys())}
            b, pp, lp, t = forward_inputs(K)
            with torch.no_grad():
                w = m(pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], time_step=t)
            entry['forward'] = {k: w[k] for k in ('pred_ligand_pos', 'pred_ligand_v', 'final_h', 'final_ligand_h')}
            b, pn, vu = chain_inputs(K)
            args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
            with torch.no_grad(), refload.noise_tape(pn, vu):
                r = m.sample_diffusion(*args, num_steps=3, center_pos_mode='protein')
            entry['chain'] = {k: r[k] for k in ('pos', 'v', 'pos_traj', 'v_traj', 'v0_traj', 'vt_traj')}
            m.load_state_dict(weights(5, K, cfgd), strict=True)
            b, pn, vu = likelihood_inputs(K)
            args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
            entry['likelihood'] = {}
            for steps in LIKELIHOOD_STEPS:
                with torch.no_grad(), refload.noise_tape(pn, vu):
                    entry['likelihood'][str(steps)] = list(m.likelihood_estimation(*args, time_step=likelihood_time_steps(steps)))
            pins[case_id(K, cfgd)] = entry
    return pin(pins)


if __name__ == '__main__':
    torch.set_num_threads(THREADS)
    torch.save(make(), OUT)
    print(OUT, os.path.getsize(OUT))
