"""Cost and effect of clash guidance at the bench workloads' shapes.

    python tools/clash_guidance_step_time.py [--workloads cfg2,cfg3,cfg5] [--respaced-steps 100] [--radius 4.0] [--strength 1.0]
                                             [--repeats 3]

Batches come from bench.make_workload, synthetic weights.  Two arms on one engine build, alternated within each repeat, each a complete
respaced chain of `respaced_steps` steps from one seed, timed whole with CUDA events (binding, table upload and the eager first step
included):
  off   clash_strength = 0, the unguided chain;
  on    clash_radius = radius, clash_strength = strength.
Reports ms per step of each arm, the contact counts of each arm's final molecules (analyze.protein_contacts at `radius`: ligand atoms
with a protein atom closer than the radius, and the smallest distance), and in a separate profiled run of the guided chain
(torch.profiler, every step eager under TDIFF_NO_GRAPH=1) the mean device time of clash_guidance_kernel per launch.  Synthetic weights:
the counts show that guidance acts, not that molecules improve.  Prints one JSON line per workload with the card name and its power
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


def _chain(model, args, seq, radius, strength):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = model.sample_diffusion(*args, center_pos_mode='protein', return_traj=False, seed=1, time_seq=seq,
                               clash_radius=radius if strength > 0 else None, clash_strength=strength)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r['pos'].cpu()


def _kernel_us(knn, args, seq, radius, strength):
    """Mean device time of clash_guidance_kernel over a guided chain run eagerly under torch.profiler (a fresh engine: TDIFF_NO_GRAPH
    is read when the engine is created)."""
    from torch.profiler import ProfilerActivity, profile
    os.environ['TDIFF_NO_GRAPH'] = '1'
    try:
        model = _model(knn)
        _chain(model, args, seq[:2], radius, strength)                          # module load, binding, the free cache
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _chain(model, args, seq, radius, strength)
        model._drop_engine()
    finally:
        del os.environ['TDIFF_NO_GRAPH']
    times = [e.device_time for e in prof.events() if 'clash_guidance_kernel' in e.name]
    return (sum(times) / len(times) if times else None), len(times)


def main():
    from targetdiff_b200.analyze import protein_contacts
    from targetdiff_b200.sampling import respaced_time_seq
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='cfg2,cfg3,cfg5')
    ap.add_argument('--respaced-steps', type=int, default=100)
    ap.add_argument('--radius', type=float, default=4.0)
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
        _chain(model, args, seq[:3], a.radius, a.strength)                      # warm up: module load, binding, the free cache
        ms, contacts = {k: [] for k in arms}, {}
        for _ in range(a.repeats):
            for k, lam in arms.items():
                t, pos = _chain(model, args, seq, a.radius, lam)
                ms[k].append(t)
                n_close, d_min = protein_contacts(pos, b['protein_pos'], b['batch_ligand'], b['batch_protein'], a.radius)
                contacts[k] = {'atoms_within_radius': int(n_close.sum()), 'ligand_atoms': len(pos), 'min_distance': float(d_min.min())}
        model._drop_engine()
        del model
        us, n = _kernel_us(w.knn, args, seq, a.radius, a.strength)
        pairs = int(sum(int((b['batch_protein'] == g).sum()) * int((b['batch_ligand'] == g).sum()) for g in range(G)))
        out = {'workload': name, 'graphs': G, 'ligand_protein_pairs': pairs, 'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': q,
               'steps': len(seq), 'radius': a.radius, 'strength': a.strength, 'chain_ms': ms,
               'ms_per_step': {k: [x / len(seq) for x in v] for k, v in ms.items()},
               'guidance_kernel_us': us, 'guidance_kernel_launches_profiled': n, 'contacts': contacts}
        print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
