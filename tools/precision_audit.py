#!/usr/bin/env python
"""Precision audit of the engine's arithmetic modes over a FULL 1000-step free-running chain (run on a GPU box):

    python tools/precision_audit.py [--out audit.json]

For every golden chain the unmodified reference wrote (tests/golden/chain_1000_cfg1*.npz: default weights and a stressed variant with
all Linear weights scaled up, a stand-in for the sharper attention of a trained checkpoint) and every edge-MLP execution mode
(tc3 = default 2-piece bf16 split / 3 products, tc6 = 3 pieces / 6 products, simt = FP32 FFMA), the same noise tape is replayed and
compared with the reference trajectory: first step with a different sampled atom type, worst relative position error per 100 steps, and the
agreement of the k-NN graphs rebuilt from both trajectories (fraction of steps with identical edge_index, first differing step)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import restate, synth  # noqa: E402
from oracle.make_golden import GOLDEN, LONG_CASES  # noqa: E402

DEV = 'cuda:0'


def knn_agreement(b, pos_traj_a, pos_traj_b, k):
    """edge lists of every step's INPUT graph, rebuilt (tdiff_knn_graph) from two lab-frame trajectories of the same single-graph batch"""
    from targetdiff_b200 import ops
    S, nl = pos_traj_a.shape[0], pos_traj_a.shape[1]
    pp = b['protein_pos'].to(DEV)
    off = pp.mean(0, keepdim=True)
    n_p = pp.shape[0]
    same = []
    for traj in (pos_traj_a, pos_traj_b):
        lig = torch.cat([b['init_ligand_pos'][None].to(DEV), traj[:-1].to(DEV)], 0)              # input of step s = state after step s-1
        x = torch.cat([(pp - off)[None].expand(S, n_p, 3), lig - off], 1).reshape(-1, 3).contiguous()
        batch = torch.repeat_interleave(torch.arange(S, device=DEV), n_p + nl)
        slots, _ = ops.knn_slots(x, k, batch)
        same.append(slots.view(S, -1))
    eq = (same[0] == same[1]).all(1)
    bad = (~eq).nonzero()
    return {'identical_edge_index_fraction': float(eq.float().mean()), 'first_differing_step': int(bad[0]) if len(bad) else None}


def run(name, mode):
    from test_gpu_reference_golden import _args, _model, chain_divergence
    case = LONG_CASES[name]
    path = os.path.join(GOLDEN, name + '.npz')
    if not os.path.exists(path):
        return None
    g = {k: torch.from_numpy(v) for k, v in np.load(path).items()}
    if mode == 'tc3':
        os.environ.pop('TDIFF_EDGE_MLP', None)
    else:
        os.environ['TDIFF_EDGE_MLP'] = mode
    model, sd = _model(case['weight_seed'], case['cfg'], gain=case.get('gain', 1.0))
    b = synth.make_batch(**case['batch'])
    S = case['num_steps'] or sd['betas'].shape[0]
    pn, vu = synth.make_tape(case['tape_seed'], S, len(b['batch_ligand']))
    got = model.sample_diffusion(*_args(b), num_steps=case['num_steps'], center_pos_mode='protein', noise_tape=(pn, vu), stack_traj=True)
    rep = chain_divergence(got['pos_traj'], got['v_traj'], g['pos_traj'], g['v_traj'].long())
    rep.update(knn_agreement(b, got['pos_traj'], g['pos_traj'], model.config.knn))
    st = case['stride']
    rep['max_abs_v0_err'] = float((got['v0_traj'][::st] - g['v0_traj']).abs().max())
    rep['within_tolerance'] = rep['first_type_mismatch_step'] is None and rep['max_rel_pos_err'] <= 1e-4 and rep['max_abs_v0_err'] <= 1e-3
    del model
    return rep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'r02_precision_audit.json'))
    ap.add_argument('--cases', default='chain_1000_cfg1,chain_1000_cfg1_gain3')
    ap.add_argument('--modes', default='tc3,tc6,simt')
    a = ap.parse_args()
    out = {'what': __doc__.split('\n\n')[0], 'tolerances': {'pos_rel': 1e-4, 'log_prob_abs': 1e-3, 'types': 'identical'}, 'results': {}}
    for name in a.cases.split(','):
        for mode in a.modes.split(','):
            r = run(name, mode)
            if r is not None:
                out['results']['%s/%s' % (name, mode)] = r
                print(name, mode, json.dumps(r), flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
