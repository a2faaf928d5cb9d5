"""Run the UNMODIFIED reference likelihood driver, scripts/likelihood_est_diffusion.data_likelihood_estimation, on CPU under the oracle
shims and store what it returns in tests/golden/reference_pins_likelihood_driver.pt, so that the restated driver
(oracle.likelihood.data_likelihood_estimation) and the engine's rng='cpu' driver are pinned against the reference on any machine.

Cases: the default config at 10 timesteps with batch_size 4 (batches of 4, 4 and 2) and 1; the time embedding; K = 23; the 1h36 pocket
with a synthetic ligand.  Each run follows misc.seed_all(seed) on one thread; the pins hold the inputs (pocket and ligand arrays, the
config options, K and the weight seed of oracle.synth.make_state_dict) and the script's 4-tuple.

    TARGETDIFF_REFERENCE=<reference checkout> python -m oracle.make_likelihood_pins
"""
import os

import torch

from oracle import refload, restate, synth
from oracle.make_reference_pins import THREADS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'reference_pins_likelihood_driver.pt')
POCKET = os.path.join(ROOT, 'tests', 'golden', '1h36_pocket10.pdb')
TIME_STEPS = list(range(0, 1000, 100))                     # the script's time steps (likelihood_est_diffusion.py:77)
TIME_EMB = {'time_emb_dim': 1, 'time_emb_mode': 'simple'}
# name -> (config options, K, batch_size, pocket: 'synthetic' | '1h36')
CASES = {
    'default_bs4': ({}, 13, 4, 'synthetic'),
    'default_bs1': ({}, 13, 1, 'synthetic'),
    'time_emb': (TIME_EMB, 13, 4, 'synthetic'),
    'K23': ({}, 23, 4, 'synthetic'),
    '1h36': ({}, 13, 4, '1h36'),
}
WEIGHT_SEED, SEED = 0, 2021


def case_data(pocket, K, sfp=None, trans=None):
    """(protein_pos, protein_atom_feature, protein_element, ligand_pos, ligand_atom_feature_full, ligand_element) of a case."""
    if pocket == 'synthetic':
        b = synth.make_batch(6, 1, n_protein=70, ligand_sizes=[11], num_classes=K)
        ppos, pfeat = b['protein_pos'], b['protein_v']
        lpos, lv = b['init_ligand_pos'], b['init_ligand_v']
    else:
        d = trans.FeaturizeProteinAtom()(sfp.pdb_to_pocket_data(POCKET))
        ppos, pfeat = d.protein_pos.float(), d.protein_atom_feature.float()
        g = torch.Generator().manual_seed(7)
        centre = ppos.mean(0)
        lpos = centre + 1.3 * torch.randn(14, 3, generator=g)
        lv = torch.randint(0, K, (14,), generator=g)
    return {'protein_pos': ppos.float(), 'protein_atom_feature': pfeat.float(), 'protein_element': torch.zeros(len(ppos), dtype=torch.long),
            'ligand_pos': lpos.float(), 'ligand_atom_feature_full': lv.long(), 'ligand_element': torch.zeros(len(lpos), dtype=torch.long)}


def make():
    ref = refload.import_reference()
    sd_mod, sfp = refload.import_reference_scripts()
    import importlib
    lik = importlib.import_module('scripts.likelihood_est_diffusion')
    import utils.misc as misc
    import utils.transforms as trans
    from torch_geometric.data import Data
    pins = {}
    for name, (cfgd, K, bs, pocket) in CASES.items():
        c = refload.default_model_config()
        c.update(cfgd)
        model = ref.ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K).eval()
        model.load_state_dict(synth.make_state_dict(WEIGHT_SEED, cfgd, schedules=restate.make_schedules(cfgd), ligand_dim=K), strict=True)
        arrays = case_data(pocket, K, sfp, trans)
        misc.seed_all(SEED)
        with torch.no_grad():
            out = lik.data_likelihood_estimation(model, Data(**arrays), torch.tensor(TIME_STEPS), batch_size=bs, device='cpu')
        pins[name] = {'cfg': dict(cfgd), 'K': K, 'batch_size': bs, 'weight_seed': WEIGHT_SEED, 'seed': SEED, 'time_steps': TIME_STEPS,
                      'data': {k: arrays[k] for k in ('protein_pos', 'protein_atom_feature', 'ligand_pos', 'ligand_atom_feature_full')},
                      'kl_pos': out[0], 'kl_v': out[1], 'sum_kl_pos': out[2], 'sum_kl_v': out[3]}
    return pins


if __name__ == '__main__':
    torch.set_num_threads(THREADS)
    torch.save(make(), OUT)
    print(OUT, os.path.getsize(OUT))
