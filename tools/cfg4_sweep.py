#!/usr/bin/env python
"""BASELINE.json configs[3] on hardware: the reference's job shape -- a test-set sweep of ragged pockets, 100 samples per pocket, 1000
steps, pockets sharded over the GPUs of one box (scripts/batch_sample_diffusion.sh:15-21 assigns pocket i to worker i % 8).

    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 tools/cfg4_sweep.py \
        --pockets 100 --samples 100 --steps 1000 --schedule round_robin --out cfg4_round_robin.json

Everything goes through the product's own command (targetdiff_b200.cli sample_pockets: checkpoint load on rank 0 + one NCCL weight
broadcast, PDB ingest, size prior, sample_diffusion_ligand, result_{i}.pt files).  The pockets are synthetic (no dataset offline):
N_p ~ U[250, 700] heavy atoms written as PDB files, seeded; the checkpoint is the seeded random-init state_dict of the default model.
Reported: per-pocket wall times, per-rank busy time, makespan, and the scheduling efficiency  sum(pocket times) / (world * makespan)
for the reference's round-robin and for longest-first."""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

ELEMENTS = {1: 'C', 2: 'N', 3: 'O', 4: 'S'}
AA = ('ALA', 'CYS', 'ASP', 'GLU', 'PHE', 'GLY', 'HIS', 'ILE', 'LYS', 'LEU', 'MET', 'ASN', 'PRO', 'GLN', 'ARG', 'SER', 'THR', 'VAL', 'TRP', 'TYR')


def write_pocket_pdb(path, seed, n_atoms):
    """A synthetic pocket (oracle.synth recipe: ball with a central cavity, 1h36 element frequencies) as fixed-column PDB ATOM records."""
    from oracle import synth
    pos, feat = synth.make_pocket(seed, n_atoms)
    el = feat[:, :6].argmax(1).tolist()
    aa = feat[:, 6:26].argmax(1).tolist()
    bb = feat[:, 26].tolist()
    with open(path, 'w') as f:
        f.write('HEADER    synthetic pocket %d\n' % seed)
        for i in range(n_atoms):
            sym = ELEMENTS[el[i]]
            name = ('CA' if bb[i] else sym + 'B')
            f.write('ATOM  %5d %-4s %3s A%4d    %8.3f%8.3f%8.3f  1.00  0.00          %2s\n' % (
                i + 1, name, AA[aa[i]], i // 8 + 1, pos[i, 0], pos[i, 1], pos[i, 2], sym))
        f.write('END\n')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pockets', type=int, default=100)
    ap.add_argument('--samples', type=int, default=100)
    ap.add_argument('--batch-size', type=int, default=100)
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--schedule', default='round_robin', choices=('round_robin', 'longest_first'))
    ap.add_argument('--min-atoms', type=int, default=250)
    ap.add_argument('--max-atoms', type=int, default=700)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from oracle import restate, synth
    from targetdiff_b200 import cli, dist as tdist
    from targetdiff_b200.config import default_model_config
    rank, world, local_rank = tdist.init_from_env()
    work = os.path.join(tempfile.gettempdir(), 'tdiff_cfg4_%s' % os.environ.get('MASTER_PORT', '0'))
    if rank == 0:
        os.makedirs(os.path.join(work, 'pockets'), exist_ok=True)
        rng = np.random.RandomState(4)
        sizes = rng.randint(a.min_atoms, a.max_atoms + 1, size=a.pockets)
        for i, n in enumerate(sizes):
            write_pocket_pdb(os.path.join(work, 'pockets', 'pocket_%03d.pdb' % i), 9000 + i, int(n))
        sd = synth.make_state_dict(0, schedules=restate.make_schedules())
        torch.save({'config': {'model': dict(default_model_config()), 'data': {'transform': {'ligand_atom_mode': 'add_aromatic'}}}, 'model': sd},
                   os.path.join(work, 'ckpt.pt'))
        with open(os.path.join(work, 'sampling.yml'), 'w') as f:
            f.write('model:\n  checkpoint: %s\nsample:\n  seed: 2021\n  num_samples: %d\n  num_steps: %d\n  pos_only: False\n'
                    '  center_pos_mode: protein\n  sample_num_atoms: prior\n' % (os.path.join(work, 'ckpt.pt'), a.samples, a.steps))
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    t0 = time.time()
    done = cli.sample_pockets([os.path.join(work, 'sampling.yml'), '--pocket_dir', os.path.join(work, 'pockets'), '--schedule', a.schedule,
                               '--batch_size', str(a.batch_size), '--result_path', os.path.join(work, 'out_' + a.schedule)])
    torch.cuda.synchronize()
    busy = time.time() - t0
    if world > 1:
        dist.barrier()
    makespan = time.time() - t0
    rec = {'rank': rank, 'busy_s': busy, 'pockets': [(int(i), int(n), float(t)) for i, n, t in done]}
    allrec = [None] * world
    if world > 1:
        dist.all_gather_object(allrec, rec)
    else:
        allrec = [rec]
    if rank == 0:
        total = sum(t for r in allrec for _, _, t in r['pockets'])
        mols = sum(n for r in allrec for _, n, _ in r['pockets'])
        out = {'config': 'cfg4: %d synthetic pockets (N_p ~ U[%d,%d]) x %d samples x %d steps, %s over %d GPUs' % (
                   a.pockets, a.min_atoms, a.max_atoms, a.samples, a.steps, a.schedule, world),
               'world': world, 'schedule': a.schedule, 'molecules': mols, 'makespan_s': makespan, 'molecules_per_s': mols / makespan,
               'sum_pocket_s': total, 'scheduling_efficiency': total / (world * makespan),
               'busy_s_per_rank': [r['busy_s'] for r in allrec], 'pockets_per_rank': [len(r['pockets']) for r in allrec],
               'pocket_times': sorted((i, n, t) for r in allrec for i, n, t in r['pockets'])}
        print(json.dumps({k: v for k, v in out.items() if k != 'pocket_times'}))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            json.dump(out, open(a.out, 'w'), indent=1)
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
