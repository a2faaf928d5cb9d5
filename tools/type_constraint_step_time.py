"""Cost and effect of element constraints at the bench workloads' shapes.

    python tools/type_constraint_step_time.py [--workloads cfg2,cfg3,cfg5] [--respaced-steps 100] [--classes 1,2,3,4,5,6] [--repeats 3]

Batches come from bench.make_workload, synthetic weights.  Two arms on one engine build, alternated within each repeat, each a complete
respaced chain of `respaced_steps` steps from one seed, timed whole with CUDA events (binding, the mask upload and check, table upload
and the eager first step included):
  off   no mask, the unconstrained chain;
  on    every ligand atom restricted to `classes` (default C, N, O of the 'add_aromatic' mode).
Reports ms per step of each arm, each arm's count of final atoms outside the set (analyze.type_violations), and in a separate profiled
run of each arm (torch.profiler, every step eager under TDIFF_NO_GRAPH=1) the mean device time of step_epilogue_kernel per launch.
Synthetic weights: the counts show that the constraint holds, not that molecules are sensible.  Prints one JSON line per workload with
the card name and its power limit."""
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

ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')


def _model(knn):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(knn=knn)
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(synth.make_state_dict(0, None, schedules=restate.make_schedules()), strict=True)
    return m.to('cuda:0')


def _chain(model, args, seq, allowed):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = model.sample_diffusion(*args, center_pos_mode='protein', return_traj=False, seed=1, time_seq=seq, allowed_types=allowed)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r['v'].cpu()


def _kernel_us(knn, args, seq, allowed):
    """Mean device time of step_epilogue_kernel over a chain run eagerly under torch.profiler (a fresh engine: TDIFF_NO_GRAPH is read
    when the engine is created)."""
    from torch.profiler import ProfilerActivity, profile
    os.environ['TDIFF_NO_GRAPH'] = '1'
    try:
        model = _model(knn)
        _chain(model, args, seq[:2], allowed)                                    # module load, binding, the free cache
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _chain(model, args, seq, allowed)
        model._drop_engine()
    finally:
        del os.environ['TDIFF_NO_GRAPH']
    times = [e.device_time for e in prof.events() if 'step_epilogue_kernel' in e.name]
    return (sum(times) / len(times) if times else None), len(times)


def main():
    from targetdiff_b200.analyze import type_violations
    from targetdiff_b200.sampling import respaced_time_seq
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='cfg2,cfg3,cfg5')
    ap.add_argument('--respaced-steps', type=int, default=100)
    ap.add_argument('--classes', default='1,2,3,4,5,6')
    ap.add_argument('--repeats', type=int, default=3)
    a = ap.parse_args()
    classes = [int(c) for c in a.classes.split(',')]
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    for name in a.workloads.split(','):
        w = argparse.Namespace(workload=name, **bench.WORKLOADS[name])
        b, G, _, _ = bench.make_workload(w, 0)
        args = tuple(b[k].to('cuda:0') for k in ARGS)
        nl = len(b['batch_ligand'])
        mask = torch.zeros(nl, synth.LIGAND_NUM_CLASSES, dtype=torch.bool, device='cuda:0')
        mask[:, classes] = True
        model = _model(w.knn)
        seq = respaced_time_seq(model.num_timesteps, a.respaced_steps)
        arms = {'off': None, 'on': mask}
        _chain(model, args, seq[:3], mask)                                       # warm up: module load, binding, the free cache
        ms, violations = {k: [] for k in arms}, {}
        for _ in range(a.repeats):
            for k, m in arms.items():
                t, v = _chain(model, args, seq, m)
                ms[k].append(t)
                violations[k] = type_violations(v, classes)
        model._drop_engine()
        del model
        kernel = {k: _kernel_us(w.knn, args, seq, m) for k, m in arms.items()}
        out = {'workload': name, 'graphs': G, 'ligand_atoms': nl, 'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': q,
               'steps': len(seq), 'classes': classes, 'chain_ms': ms, 'ms_per_step': {k: [x / len(seq) for x in v] for k, v in ms.items()},
               'epilogue_kernel_us': {k: u for k, (u, _) in kernel.items()},
               'epilogue_launches_profiled': {k: n for k, (_, n) in kernel.items()}, 'atoms_outside_the_set': violations}
        print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
