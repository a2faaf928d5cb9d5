"""Cost and effect of connectivity guidance at the bench workloads' shapes.

    python tools/connect_guidance_step_time.py [--workloads cfg2,cfg3,cfg5] [--respaced-steps 100] [--radius 2.0] [--length 1.5]
                                               [--strength 1.0] [--repeats 3]

Batches come from bench.make_workload, synthetic weights.  Two arms on one engine build, alternated within each repeat, each a complete
respaced chain of `respaced_steps` steps from one seed, timed whole with CUDA events (binding, table upload and the eager first step
included):
  off   connect_strength = 0, the unguided chain;
  on    connect_radius = radius, connect_length = length, connect_strength = strength.
Reports ms per step of each arm, the disconnected final molecules of each arm (analyze.ligand_components at `radius`: molecules in more
than one piece when atoms closer than the radius are bonded), and in a separate profiled run of the guided chain (torch.profiler,
every step eager under TDIFF_NO_GRAPH=1) the mean device time of connect_guidance_kernel per launch.  Synthetic weights: the counts
show that guidance acts, not that molecules improve.  Prints one JSON line per workload with the card name and its power
limit."""
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


def _chain(model, args, seq, radius, length, strength):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = model.sample_diffusion(*args, center_pos_mode='protein', return_traj=False, seed=1, time_seq=seq,
                               connect_radius=radius if strength > 0 else None, connect_length=length if strength > 0 else None,
                               connect_strength=strength)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r['pos'].cpu()


def _kernel_us(knn, args, seq, radius, length, strength):
    """Mean device time of connect_guidance_kernel over a guided chain run eagerly under torch.profiler (a fresh engine: TDIFF_NO_GRAPH
    is read when the engine is created)."""
    from torch.profiler import ProfilerActivity, profile
    os.environ['TDIFF_NO_GRAPH'] = '1'
    try:
        model = _model(knn)
        _chain(model, args, seq[:2], radius, length, strength)                  # module load, binding, the free cache
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _chain(model, args, seq, radius, length, strength)
        model._drop_engine()
    finally:
        del os.environ['TDIFF_NO_GRAPH']
    times = [e.device_time for e in prof.events() if 'connect_guidance_kernel' in e.name]
    return (sum(times) / len(times) if times else None), len(times)


def main():
    from targetdiff_b200.analyze import ligand_components
    from targetdiff_b200.sampling import respaced_time_seq
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='cfg2,cfg3,cfg5')
    ap.add_argument('--respaced-steps', type=int, default=100)
    ap.add_argument('--radius', type=float, default=2.0)
    ap.add_argument('--length', type=float, default=1.5)
    ap.add_argument('--strength', type=float, default=1.0)
    ap.add_argument('--repeats', type=int, default=3)
    a = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    for name in a.workloads.split(','):
        w = argparse.Namespace(workload=name, **bench.WORKLOADS[name])
        b, G, _, _ = bench.make_workload(w, 0)
        args = tuple(b[k].to('cuda:0') for k in ARGS)
        model = _model(w.knn)
        seq = respaced_time_seq(model.num_timesteps, a.respaced_steps)
        arms = {'off': 0.0, 'on': a.strength}
        _chain(model, args, seq[:3], a.radius, a.length, a.strength)            # warm up: module load, binding, the free cache
        ms, pieces = {k: [] for k in arms}, {}
        for _ in range(a.repeats):
            for k, lam in arms.items():
                t, pos = _chain(model, args, seq, a.radius, a.length, lam)
                ms[k].append(t)
                n_comp = ligand_components(pos, b['batch_ligand'], a.radius)
                pieces[k] = {'disconnected_molecules': int((n_comp > 1).sum()), 'molecules': len(n_comp), 'pieces': int(n_comp.sum())}
        model._drop_engine()
        del model
        us, n = _kernel_us(w.knn, args, seq, a.radius, a.length, a.strength)
        sizes = torch.bincount(b['batch_ligand'])
        out = {'workload': name, 'graphs': G, 'max_ligand_atoms': int(sizes.max()), 'ligand_pairs': int((sizes * sizes).sum()),
               'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': q, 'steps': len(seq), 'radius': a.radius, 'length': a.length,
               'strength': a.strength, 'chain_ms': ms, 'ms_per_step': {k: [x / len(seq) for x in v] for k, v in ms.items()},
               'guidance_kernel_us': us, 'guidance_kernel_launches_profiled': n, 'components': pieces}
        print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
