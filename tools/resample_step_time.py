"""Cost of resampled sampling (re-noising steps on a time path) at the bench workloads' shapes, with held atoms.

    python tools/resample_step_time.py [--workloads cfg3,cfg2,cfg5] [--respaced-steps 100] [--fixed 8] [--repeats 3]

Batches come from bench.make_workload; the first `fixed` atoms of every ligand (at most all but one) are held, as a fragment.  The base
is sampling.respaced_time_seq(T, respaced_steps).  Three arms on one engine build, alternated within each repeat, each a complete chain
timed whole with CUDA events (binding, table upload, the fixed atoms' initial launch and the eager first step included):
  r1      the base itself (resamplings = 1): n denoising steps;
  r5_j1   resampled_time_path(base, 5, 1): 5 (n - 1) + 1 denoising and 4 (n - 1) re-noising steps;
  r5_j10  resampled_time_path(base, 5, 10): the same denoising steps and 4 ceil((n - 1) / 10) re-noising steps.
Reports ms per denoising step (r1's chain over its steps) and molecules/s of each whole chain.  A re-noising step costs too little to
show in the difference of r5_j1 and r5_j10 above their run-to-run spread, so it is timed on two more paths with the same n_runs + 2
denoising steps, alternated with the others:
  up_sparse  T-1, then n_runs times 0, T-2, then 0: n_runs re-noising steps;
  up_dense   T-1, then n_runs times 0, 1, ..., T-2, then 0: n_runs (T - 2) re-noising steps;
us per re-noising step = (up_dense - up_sparse) over the difference in re-noising steps, what a user pays per step with the launches
issued from the host.  Prints one JSON line per workload with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import restate, synth  # noqa: E402


def _model(knn):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(knn=knn)
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(synth.make_state_dict(0, None, schedules=restate.make_schedules()), strict=True)
    return m.to('cuda:0')


def _chain_ms(model, args, mask, path):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    model.sample_diffusion(*args, center_pos_mode='protein', return_traj=False, seed=1, fixed_mask=mask, time_path=path)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def _held(batch_ligand, n_fixed):
    """The first n_fixed atoms of every ligand, leaving at least one free."""
    counts = torch.bincount(batch_ligand)
    first = torch.cumsum(counts, 0) - counts
    rank = torch.arange(len(batch_ligand)) - first[batch_ligand]
    return (rank < torch.clamp(counts - 1, max=n_fixed)[batch_ligand]).to('cuda:0')


def main():
    from targetdiff_b200.sampling import resampled_time_path, respaced_time_seq
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='cfg3,cfg2,cfg5')
    ap.add_argument('--respaced-steps', type=int, default=100)
    ap.add_argument('--fixed', type=int, default=8)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--n-runs', type=int, default=40, help='upward runs of the up_sparse / up_dense paths (at most 63 at T = 1000)')
    a = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    for name in a.workloads.split(','):
        w = argparse.Namespace(workload=name, **bench.WORKLOADS[name])
        b, G, _, _ = bench.make_workload(w, 0)
        args = tuple(b[k].to('cuda:0') for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v',
                                                 'batch_ligand'))
        mask = _held(b['batch_ligand'], a.fixed)
        model = _model(w.knn)
        base = respaced_time_seq(model.num_timesteps, a.respaced_steps)
        T = model.num_timesteps
        arms = {'r1': base, 'r5_j1': resampled_time_path(base, 5, 1), 'r5_j10': resampled_time_path(base, 5, 10),
                'up_sparse': [T - 1] + [0, T - 2] * a.n_runs + [0], 'up_dense': [T - 1] + list(range(T - 1)) * a.n_runs + [0]}
        steps = {k: (sum(1 for s, t in enumerate(p) if s + 1 == len(p) or p[s + 1] < t), sum(1 for s, t in enumerate(p[:-1]) if p[s + 1] > t))
                 for k, p in arms.items()}
        _chain_ms(model, args, mask, base[:3])                                  # warm up: module load, binding, the free cache
        ms = {k: [] for k in arms}
        for _ in range(a.repeats):
            for k, p in arms.items():
                ms[k].append(_chain_ms(model, args, mask, p))
        up = steps['up_dense'][1] - steps['up_sparse'][1]
        out = {'workload': name, 'graphs': G, 'held_atoms': int(mask.sum()), 'ligand_atoms': len(mask), 'gpu': torch.cuda.get_device_name(0),
               'nvidia_smi': q, 'base_steps': len(base), 'steps_denoise_renoise': steps, 'chain_ms': ms,
               'ms_per_denoising_step': [x / steps['r1'][0] for x in ms['r1']],
               'us_per_renoising_step': [1e3 * (x - y) / up for x, y in zip(ms['up_dense'], ms['up_sparse'])],
               'molecules_per_s': {k: [G / (x / 1e3) for x in v] for k, v in ms.items() if k.startswith('r')}}
        print(json.dumps(out), flush=True)
        model._drop_engine()
        del model


if __name__ == '__main__':
    main()
