"""GPU: compare the three edge-MLP execution modes (FP32 FFMA, wgmma 3-term, wgmma 6-term) against the CPU oracle."""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import restate, synth  # noqa: E402
from targetdiff_b200.config import default_model_config  # noqa: E402
from targetdiff_b200.score_model import ScorePosNet3D  # noqa: E402

dev = torch.device('cuda:0')
sd = synth.make_state_dict(1, schedules=restate.make_schedules())
b = synth.make_batch(31, 2, n_protein=200, ligand_sizes=[20, 33])
pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
tr = {}
want = restate.forward(sd, None, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
for mode in sys.argv[1:] or ['simt', 'tc6', 'tc3']:
    os.environ['TDIFF_EDGE_MLP'] = mode
    m = ScorePosNet3D(default_model_config(), 27, 13)
    m.load_state_dict(sd)
    m = m.to(dev)
    args = (pp.to(dev), b['protein_v'].to(dev), b['batch_protein'].to(dev), lp.to(dev), b['init_ligand_v'].to(dev), b['batch_ligand'].to(dev))
    out = m(*args)
    torch.cuda.synchronize()
    t0 = time.time()
    out = m(*args)
    torch.cuda.synchronize()
    dt = time.time() - t0
    ep = (out['pred_ligand_pos'].cpu() - want['pred_ligand_pos']).abs().max().item()
    rp = ((out['pred_ligand_pos'].cpu() - want['pred_ligand_pos']).abs() / want['pred_ligand_pos'].abs().clamp_min(1e-3)).max().item()
    el = (out['pred_ligand_v'].cpu() - want['pred_ligand_v']).abs().max().item()
    eh = (out['final_h'].cpu() - want['final_h']).abs().max().item()
    rh = eh / want['final_h'].abs().max().item()
    print('%-5s edge_index_equal=%s  pos max_abs=%.3e max_rel=%.3e  logits max_abs=%.3e  final_h max_abs=%.3e (rel to max %.3e)  %.1f ms' % (
        mode, torch.equal(out['edge_index'].cpu(), tr['edge_index']), ep, rp, el, eh, rh, dt * 1e3), flush=True)
    del m
