"""Run the UNMODIFIED reference (under oracle/shims) on the layer forms of AttentionLayerO2TwoUpdateNodeGeneral (num_x2h, num_h2x,
sync_twoup; reference models/uni_transformer.py:143-210) and on forward(..., return_all=True), and store what it returns in
tests/golden/reference_pins_layer_forms.pt, so that the restatement is pinned against the reference on any machine.
Same recipe as the backbone options of oracle/make_reference_pins.py.

    TARGETDIFF_REFERENCE=<reference checkout> python -m oracle.make_layer_form_pins
"""
import os

import torch

from oracle import refload, restate, synth
from oracle.make_reference_pins import THREADS, option_id, pin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'reference_pins_layer_forms.pt')

LAYER_FORM_CONFIGS = [{'num_x2h': 2}, {'num_h2x': 2}, {'num_h2x': 0}, {'num_x2h': 0}, {'sync_twoup': True},
                      {'num_x2h': 2, 'num_h2x': 3, 'sync_twoup': True, 'ew_net_type': 'r'},
                      {'num_x2h': 2, 'ew_net_type': 'm', 'x2h_out_fc': True},
                      {'num_blocks': 2, 'num_h2x': 2, 'cutoff_mode': 'hybrid'}]
RETURN_ALL_BLOCKS = (1, 2)


def chain_inputs():
    """Weights seed, batch and tape of the 3-step chain (the recipe of the backbone options)."""
    b = synth.make_batch(3, 2, n_protein=60, ligand_sizes=[9, 7])
    pn, vu = synth.make_tape(5, 3, 16)
    return b, pn, vu


def return_all_inputs():
    b = synth.make_batch(1, 2, n_protein=60, ligand_sizes=[9, 7])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    return b, pp, lp


def make():
    ref = refload.import_reference()
    pins = {}
    for cfgd in LAYER_FORM_CONFIGS:
        c = refload.default_model_config()
        c.update(cfgd)
        m = ref.ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES).eval()
        sd = synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd))
        m.load_state_dict(sd, strict=True)
        b, pn, vu = chain_inputs()
        args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
        with torch.no_grad(), refload.noise_tape(pn, vu):
            r = m.sample_diffusion(*args, num_steps=3, center_pos_mode='protein')
        entry = {'keys': list(m.state_dict().keys()), **{k: r[k] for k in ('pos', 'v', 'pos_traj', 'v0_traj', 'vt_traj')}}
        for nb in RETURN_ALL_BLOCKS:
            cb = dict(cfgd, num_blocks=nb)
            c = refload.default_model_config()
            c.update(cb)
            m = ref.ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES).eval()
            m.load_state_dict(synth.make_state_dict(1, cb, schedules=restate.make_schedules(cb)), strict=True)
            b, pp, lp = return_all_inputs()
            with torch.no_grad():
                w = m(pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], return_all=True)
            entry['return_all_%d' % nb] = {k: w[k] for k in ('pred_ligand_pos', 'pred_ligand_v', 'final_h', 'layer_pred_ligand_pos',
                                                              'layer_pred_ligand_v')}
        pins[option_id(cfgd)] = entry
    return pin(pins)


if __name__ == '__main__':
    torch.set_num_threads(THREADS)
    torch.save(make(), OUT)
    print(OUT, os.path.getsize(OUT))
