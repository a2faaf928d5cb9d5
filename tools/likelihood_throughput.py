"""Ligands scored per second by likelihood scoring on the GPU (DESIGN.md section 1), three arms alternated, `--runs` runs each:

    batched   targetdiff_b200.likelihood.ligand_nll: every (ligand, t) pair a graph, batches of up to 640 graphs
    ref_loop  the reference script's loop shape: per ligand, batches of 4 timesteps through model.likelihood_estimation, then its prior
    exact     ligand_nll at every timestep (T = 1000) for 4 ligands: the cost of an exact sum over t

on a cfg2-shaped pocket (572 protein atoms, ligands of 25 atoms) and a cfg3-shaped one (300 + 20), 64 ligands at 10 timesteps.  Also
splits one 640-graph engine call into the forward (CUDA events around tdiff_forward on the same bound batch) and the rest (bind, the
two likelihood launches, host work).  Synthetic weights and pockets; prints the card's name and power limit with the numbers.

    python tools/likelihood_throughput.py [--runs 3] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import restate, synth  # noqa: E402
from targetdiff_b200 import _lib  # noqa: E402
from targetdiff_b200.config import default_model_config  # noqa: E402
from targetdiff_b200.likelihood import data_likelihood_estimation, ligand_nll, likelihood_time_steps  # noqa: E402
from targetdiff_b200.score_model import ScorePosNet3D  # noqa: E402

DEV = 'cuda:0'
SHAPES = {'cfg2': (572, 25), 'cfg3': (300, 20)}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip()


def setup(n_protein, n_lig, n_ligands):
    m = ScorePosNet3D(default_model_config(), synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(synth.make_state_dict(0, schedules=restate.make_schedules()), strict=True)
    m = m.to(DEV)
    pos, feat = synth.make_pocket(1, n_protein)
    g = torch.Generator().manual_seed(2)
    ligs = [(pos.mean(0) + 1.5 * torch.randn(n_lig, 3, generator=g), torch.randint(0, synth.LIGAND_NUM_CLASSES, (n_lig,), generator=g))
            for _ in range(n_ligands)]
    return m, {'protein_pos': pos, 'protein_atom_feature': feat}, ligs


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def call_split(m, data, ligs, ts):
    """(ms of one 640-graph likelihood_terms call, ms of the forward on the same bound batch by CUDA events)"""
    n = 640
    part = [(i, t) for i in range(len(ligs)) for t in ts][:n]
    pp = data['protein_pos'].repeat(n, 1).to(DEV)
    pf = data['protein_atom_feature'].repeat(n, 1).to(DEV)
    bp = torch.repeat_interleave(torch.arange(n), data['protein_pos'].shape[0]).to(DEV)
    lp = torch.cat([ligs[i][0] for i, _ in part]).to(DEV)
    lv = torch.cat([ligs[i][1] for i, _ in part]).to(DEV)
    bl = torch.repeat_interleave(torch.arange(n), torch.tensor([len(ligs[i][1]) for i, _ in part])).to(DEV)
    tl = [t for _, t in part]
    for _ in range(3):
        m.likelihood_terms(pp, pf, bp, lp, lv, bl, tl, seed=1)
    call = min(timed(lambda: m.likelihood_terms(pp, pf, bp, lp, lv, bl, tl, seed=1)) for _ in range(5)) * 1e3
    lib, eng, st = _lib.load(), m.engine(DEV), m._stream(torch.device(DEV))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fw = []
    for _ in range(5):
        a.record()
        _lib.check(lib.tdiff_forward(eng, None, None, None, 0, st))
        b.record()
        torch.cuda.synchronize()
        fw.append(a.elapsed_time(b))
    return call, min(fw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--ligands', type=int, default=64)
    ap.add_argument('--out', type=str)
    a = ap.parse_args()
    info = card()
    print('card, power limit:', info)
    res = {'card': info, 'shapes': {}}
    for name, (n_p, n_l) in SHAPES.items():
        m, data, ligs = setup(n_p, n_l, a.ligands)
        ts = likelihood_time_steps(1000, 10)
        lig_data = lambda i: {'protein_pos': data['protein_pos'], 'protein_atom_feature': data['protein_atom_feature'],  # noqa: E731
                              'ligand_pos': ligs[i][0], 'ligand_atom_feature_full': ligs[i][1]}
        arms = {
            'batched': (a.ligands, lambda: ligand_nll(m, data, ligs, time_steps=ts, batch_size=640, device=DEV, seed=1)),
            'ref_loop': (a.ligands, lambda: [data_likelihood_estimation(m, lig_data(i), torch.tensor(ts), batch_size=4, device=DEV)
                                             for i in range(a.ligands)]),
            'exact': (4, lambda: ligand_nll(m, data, ligs[:4], time_steps=list(range(1000)), batch_size=640, device=DEV, seed=1)),
        }
        for _, fn in arms.values():        # warm-up of every shape
            fn()
        out = {k: [] for k in arms}
        for _ in range(a.runs):
            for k, (n, fn) in arms.items():
                out[k].append(n / timed(fn))
        call_ms, fwd_ms = call_split(m, data, ligs, ts)
        res['shapes'][name] = {'ligands_per_s': out, 'call_640_ms': call_ms, 'forward_640_ms': fwd_ms}
        print('%s (%d protein + %d ligand atoms): ligands/s %s; one 640-graph call %.2f ms, of which the forward %.2f ms'
              % (name, n_p, n_l, {k: ['%.1f' % x for x in v] for k, v in out.items()}, call_ms, fwd_ms))
        del m
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'likelihood_throughput.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
