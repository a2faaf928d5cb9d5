"""Step time and throughput of chains from a start ligand next to the default chain, at the bench workloads' shapes.

    python tools/start_step_time.py [--workloads cfg3,cfg2,cfg5] [--start-time 500] [--respaced-steps 50] [--steps 20] [--warmup 3]
                                    [--repeats 3]

Batches come from bench.make_workload; the start ligand is the batch's initial ligand.  Three arms on one engine build, alternated
within each repeat:
  default   the default chain (t = T-1, T-2, ...), timed with CUDA events as (time of warmup + steps steps) - (time of warmup steps),
            so binding, the ligand-free cache build and the first (eager) step cancel;
  unit      the complete chain from start_time with unit steps (start_time + 1 steps), timed whole;
  respaced  the complete chain of sampling.respaced_time_seq(T, respaced_steps, start=start_time), timed whole.
The whole-chain arms include binding, the table upload, the start draw and the eager first step: what a user pays for one batch of
molecules.  Reports ms per step of each arm and molecules/s of each complete chain, and of a complete T-step default chain at the
measured step time.  Prints one JSON line per workload with the card name and its power limit."""
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


def _chain_ms(model, args, **kw):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    model.sample_diffusion(*args, center_pos_mode='protein', return_traj=False, seed=1, **kw)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    from targetdiff_b200.sampling import respaced_time_seq
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='cfg3,cfg2,cfg5')
    ap.add_argument('--start-time', type=int, default=500)
    ap.add_argument('--respaced-steps', type=int, default=50)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=3)
    a = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    for name in a.workloads.split(','):
        w = argparse.Namespace(workload=name, **bench.WORKLOADS[name])
        b, G, _, _ = bench.make_workload(w, 0)
        args = tuple(b[k].to('cuda:0') for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v',
                                                 'batch_ligand'))
        model = _model(w.knn)
        T = model.num_timesteps
        t0 = a.start_time
        seq = respaced_time_seq(T, a.respaced_steps, start=t0)
        _chain_ms(model, args, num_steps=a.warmup)
        _chain_ms(model, args, start_time=t0, time_seq=seq)
        default, unit, resp = [], [], []
        for _ in range(a.repeats):
            default.append((_chain_ms(model, args, num_steps=a.warmup + a.steps) - _chain_ms(model, args, num_steps=a.warmup)) / a.steps)
            unit.append(_chain_ms(model, args, start_time=t0))
            resp.append(_chain_ms(model, args, start_time=t0, time_seq=seq))
        print(json.dumps({'workload': name, 'graphs': G, 'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': q, 'T': T, 'start_time': t0,
                          'default_ms_per_step': default, 'default_molecules_per_s_at_T_steps': [G / (T * ms / 1e3) for ms in default],
                          'unit_steps': t0 + 1, 'unit_chain_ms': unit, 'unit_ms_per_step': [ms / (t0 + 1) for ms in unit],
                          'unit_molecules_per_s': [G / (ms / 1e3) for ms in unit],
                          'respaced_steps': len(seq), 'respaced_chain_ms': resp, 'respaced_ms_per_step': [ms / len(seq) for ms in resp],
                          'respaced_molecules_per_s': [G / (ms / 1e3) for ms in resp]}), flush=True)
        model._drop_engine()
        del model


if __name__ == '__main__':
    main()
