"""Sampling-step time with fixed atoms (fragment-conditioned sampling) at the cfg3 shape, next to the same chain with none fixed.

    python tools/fixed_atoms_step_time.py [--steps 20] [--warmup 3] [--repeats 3] [--fixed 8]

cfg3 = 640 graphs of 300 protein + 20 ligand atoms.  Two arms on one engine build: no fixed set, and the first `fixed` atoms of every
ligand fixed.  Each arm: `warmup` steps, then the chain timed with CUDA events as (time of warmup + steps steps) - (time of warmup
steps), so binding, set_fixed, the initial noising launch, the ligand-free cache build and the first (eager) step cancel.  The arms
are alternated within each repeat.  Prints one JSON line with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import restate, synth  # noqa: E402

CFG3 = dict(pockets=64, samples=10, n_protein=300, n_ligand=20, knn=32)


def _model():
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(knn=CFG3['knn'])
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(synth.make_state_dict(0, None, schedules=restate.make_schedules()), strict=True)
    return m.to('cuda:0')


def _chain_ms(model, args, steps, mask):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    model.sample_diffusion(*args, num_steps=steps, center_pos_mode='protein', return_traj=False, seed=1, fixed_mask=mask)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--fixed', type=int, default=8, help='atoms fixed at the head of every ligand')
    a = ap.parse_args()
    w = CFG3
    b = synth.make_batch(0, w['pockets'] * w['samples'], n_protein=w['n_protein'], n_ligand=w['n_ligand'], distinct_pockets=w['pockets'])
    args = tuple(b[k].to('cuda:0') for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))
    mask = (torch.arange(len(b['batch_ligand'])) % w['n_ligand'] < a.fixed).to('cuda:0')
    model = _model()
    arms = [('none fixed', None), ('%d of %d fixed' % (a.fixed, w['n_ligand']), mask)]
    for _, m in arms:
        _chain_ms(model, args, a.warmup, m)
    res = [[] for _ in arms]
    for _ in range(a.repeats):
        for i, (_, m) in enumerate(arms):
            res[i].append((_chain_ms(model, args, a.warmup + a.steps, m) - _chain_ms(model, args, a.warmup, m)) / a.steps)
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    print(json.dumps({'workload': 'cfg3', 'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': q, 'steps': a.steps,
                      'arms': [{'arm': name, 'ms_per_step': r} for (name, _), r in zip(arms, res)]}))


if __name__ == '__main__':
    main()
