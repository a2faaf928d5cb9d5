"""Run the UNMODIFIED reference's stability screen (utils/evaluation/analyze.py:106-143 `check_stability`, return_nr_bonds=True) on
every boundary pair and molecule of oracle/stability_cases.py, with hs False and True, and store the inputs with what it returns in
tests/golden/reference_pins_stability_thresholds.pt.  Same recipe as oracle/make_hybrid_tie_pins.py.

    TARGETDIFF_REFERENCE=<reference checkout> python -m oracle.make_stability_pins
"""
import importlib
import os
import sys

import numpy as np
import torch

from oracle import refload, stability_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'reference_pins_stability_thresholds.pt')


def make():
    refload.import_reference()
    if refload.SHIMS not in sys.path:
        sys.path.insert(0, refload.SHIMS)
    import _absent                                  # inert stand-ins for analyze.py's import-only dependency matplotlib
    _absent.install()
    analyze = importlib.import_module('utils.evaluation.analyze')
    cases = stability_cases.inputs()
    results, nr_bonds = [], []
    for case in cases:
        per_hs, nb = [], []
        for hs in (False, True):
            w = analyze.check_stability(case['pos'], case['z'], hs=hs, return_nr_bonds=True)
            per_hs.append([int(w[0]), int(w[1]), int(w[2])])
            nb.append(np.asarray(w[3], dtype=np.int64))
        results.append(per_hs)
        nr_bonds.append(np.stack(nb, 1))
    # one tensor per field, molecules concatenated (counts gives the split): the file stays a few kB
    return {'names': [c['name'] for c in cases], 'counts': torch.tensor([len(c['z']) for c in cases]),
            'pos': torch.from_numpy(np.concatenate([c['pos'] for c in cases])), 'z': torch.from_numpy(np.concatenate([c['z'] for c in cases])),
            'result': torch.tensor(results),                                 # [M, hs, (molecule_stable, nr_stable_atoms, n_atoms)]
            'nr_bonds': torch.from_numpy(np.concatenate(nr_bonds))}          # [sum n, hs]

if __name__ == '__main__':
    torch.save(make(), OUT)
    print(OUT, os.path.getsize(OUT))
