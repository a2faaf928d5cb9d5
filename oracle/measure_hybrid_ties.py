"""How often a hybrid ligand row reaches torch.topk's unspecified tie order (DESIGN.md section 2): ligand positions drawn around the
1h36 pocket (tests/golden/1h36_pocket10.pdb; N(centre, 3 A) per coordinate, like the sampler's initial positions), and per row whether
the k-th and (k+1)-th protein atoms under the canonical (fp32 d2, index) key have equal torch.norm distance but different d2, the case
where the reference's choice may differ from the canonical one.  CPU only.

    python -m oracle.measure_hybrid_ties [n_positions]
"""
import os
import sys

import numpy as np
import torch

from oracle import restate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PDB = os.path.join(ROOT, 'tests', 'golden', '1h36_pocket10.pdb')


def count(P, L, k, chunk=5000):
    hits = 0
    idx = np.arange(len(P))
    for s in range(0, len(L), chunk):
        lig = L[s:s + chunk]
        d = torch.norm(lig.unsqueeze(1) - P.unsqueeze(0), p=2, dim=-1)
        d2 = restate._d2_fp32(lig, P)
        order = torch.from_numpy(np.lexsort((np.broadcast_to(idx, d2.shape), d2), axis=1))
        dk, d2k = d.gather(1, order[:, k - 1:k + 1]), torch.from_numpy(d2).gather(1, order[:, k - 1:k + 1])
        hits += int(((dk[:, 0] == dk[:, 1]) & (d2k[:, 0] != d2k[:, 1])).sum())
    return hits


def main(n=100000):
    from targetdiff_b200.pocket import pdb_to_pocket_data
    P = pdb_to_pocket_data(PDB).protein_pos.float()
    L = P.mean(0, keepdim=True) + 3.0 * torch.randn(n, 3, generator=torch.Generator().manual_seed(0))
    for k in (8, 21, 32):
        print('k=%d: %d of %d ligand rows with a torch.norm tie of distinct fp32 d2 across the k-th place (%d protein atoms)' %
              (k, count(P, L, k), n, len(P)))


if __name__ == '__main__':
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 100000)
