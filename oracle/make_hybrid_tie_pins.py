"""Run the UNMODIFIED reference's hybrid edge builder (models/common.py:185-212, batch_hybrid_edge_connection with add_p_index=True,
under oracle/shims) on `synth.hybrid_norm_tie_graph` at k = 8, 21 and 32, and store its inputs and the edge_index it returns in
tests/golden/reference_pins_hybrid_ties.pt.  On these graphs two protein atoms have equal torch.norm distance to a ligand atom at the
k-th place but different fp32 squared distances: the reference keeps whichever torch.topk returns, `restate.hybrid_graph_canonical`
(and the engine) the one with the smaller (d2, index) key.  Same recipe as oracle/make_class_count_pins.py.

    TARGETDIFF_REFERENCE=<reference checkout> python -m oracle.make_hybrid_tie_pins
"""
import importlib
import os

import torch

from oracle import refload, synth
from oracle.make_reference_pins import THREADS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'reference_pins_hybrid_ties.pt')
KS = (8, 21, 32)


def graph_inputs(k):
    """(x [N,3], mask_ligand [N], batch [N]) of the one-graph tie case in the composed node order (protein atoms, then ligand)."""
    p, l = synth.hybrid_norm_tie_graph(k)
    x = torch.cat([torch.from_numpy(p), torch.from_numpy(l)])
    mask = torch.cat([torch.zeros(len(p), dtype=torch.long), torch.ones(len(l), dtype=torch.long)])
    return x, mask, torch.zeros(len(x), dtype=torch.long)


def make():
    refload.import_reference()
    common = importlib.import_module('models.common')
    pins = {}
    for k in KS:
        x, mask, batch = graph_inputs(k)
        pins['k=%d' % k] = {'x': x, 'mask_ligand': mask,
                            'edge_index': common.batch_hybrid_edge_connection(x, k, mask, batch, add_p_index=True)}
    return pins


if __name__ == '__main__':
    torch.set_num_threads(THREADS)
    torch.save(make(), OUT)
    print(OUT, os.path.getsize(OUT))
