"""Sampling-step time of layer forms (num_x2h, num_h2x, sync_twoup) at a bench workload's shape, next to the default form.

    python tools/layer_form_step_time.py [--workload cfg3] [--steps 20] [--warmup 3] [--repeats 3]

For each form: one engine, `warmup` steps, then the chain timed with CUDA events as (time of warmup + steps steps) - (time of warmup
steps), so binding, the ligand-free cache build and the first (eager) step cancel.  Forms are alternated within each repeat.  Prints one
JSON line with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import restate, synth  # noqa: E402

WORKLOADS = {'cfg3': dict(pockets=64, samples=10, n_protein=300, n_ligand=20, knn=32)}
FORMS = [{}, {'num_x2h': 2}, {'num_h2x': 2}]


def _model(cfgd, knn):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(dict(cfgd, knn=knn))
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd)), strict=True)
    return m.to('cuda:0')


def _chain_ms(model, args, steps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    model.sample_diffusion(*args, num_steps=steps, center_pos_mode='protein', return_traj=False, seed=1)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='cfg3', choices=sorted(WORKLOADS))
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=3)
    a = ap.parse_args()
    w = WORKLOADS[a.workload]
    b = synth.make_batch(0, w['pockets'] * w['samples'], n_protein=w['n_protein'], n_ligand=w['n_ligand'], distinct_pockets=w['pockets'])
    args = tuple(b[k].to('cuda:0') for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))
    models = [_model(f, w['knn']) for f in FORMS]
    for m in models:
        _chain_ms(m, args, a.warmup)
    res = [[] for _ in FORMS]
    for _ in range(a.repeats):
        for i, m in enumerate(models):
            res[i].append((_chain_ms(m, args, a.warmup + a.steps) - _chain_ms(m, args, a.warmup)) / a.steps)
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    print(json.dumps({'workload': a.workload, 'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': q, 'steps': a.steps,
                      'forms': [{'form': f or 'default', 'ms_per_step': r} for f, r in zip(FORMS, res)]}))


if __name__ == '__main__':
    main()
