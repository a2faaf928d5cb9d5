"""The neighbour-list semantics at distance ties on the CPU: the hybrid graph's tie rule (`restate.hybrid_graph_canonical`) against the
unmodified reference (tests/golden/reference_pins_hybrid_ties.pt, made by oracle/make_hybrid_tie_pins.py) and against the reference's
mirror `restate.hybrid_graph` on every input the other hybrid pins use; and the tie geometry of oracle/synth.py that
tests/test_gpu_graph_geometry.py runs the engine on."""
import numpy as np
import pytest
import torch

from oracle import layer_forms, make_hybrid_tie_pins as htp, make_layer_form_pins as lfp, restate, synth
from oracle import make_reference_pins as pins_mod


@pytest.mark.parametrize('k', htp.KS)
def test_hybrid_norm_tie_reference_pin(k):
    """At the constructed tie the reference keeps protein atom k (the larger fp32 d2), the canonical rule atom k - 1; every other edge
    is the same.  restate.hybrid_graph still mirrors the reference bit for bit."""
    pin = torch.load(htp.OUT, weights_only=True)['k=%d' % k]
    x, mask, batch = htp.graph_inputs(k)
    assert torch.equal(x, pin['x']) and torch.equal(mask, pin['mask_ligand']), \
        'synth.hybrid_norm_tie_graph no longer builds the pinned inputs (builder or torch.norm rounding changed): rerun the maker'
    want = pin['edge_index']
    assert torch.equal(restate.hybrid_graph(x, k, mask, batch), want)
    got = restate.hybrid_graph_canonical(x, k, mask, batch)
    q = int(mask.nonzero()[0])                                   # the ligand atom of the tie
    d = torch.norm(x[q] - x[[k - 1, k]], p=2, dim=-1)
    d2 = restate._d2_fp32(x[q:q + 1], x[[k - 1, k]])[0]
    assert d[0] == d[1] and d2[0] < d2[1]
    ref_row, row = want[0, want[1] == q].tolist(), got[0, got[1] == q].tolist()
    assert k in ref_row and k - 1 not in ref_row
    assert k - 1 in row and k not in row
    assert sorted(set(ref_row) - {k}) == sorted(set(row) - {k - 1})
    edges = lambda e: set(map(tuple, e.T.tolist()))
    assert edges(want) ^ edges(got) == {(k, q), (k - 1, q)}


def test_hybrid_canonical_equals_reference_mirror_on_pinned_inputs(monkeypatch):
    """Every hybrid graph built while the restatement reproduces the reference's hybrid pins (the backbone options of
    reference_pins.pt, the layer form of reference_pins_layer_forms.pt, its return_all forwards) is the same, edge for edge and in
    the same order, under the canonical rule and under norm + topk."""
    calls = []
    canonical = restate.hybrid_graph_canonical

    def both(x, k, mask, batch):
        got = canonical(x, k, mask, batch)
        assert torch.equal(got, restate.hybrid_graph(x, k, mask, batch))
        calls.append(k)
        return got
    monkeypatch.setattr(restate, 'hybrid_graph_canonical', both)
    b = synth.make_batch(3, 2, n_protein=60, ligand_sizes=[9, 7])
    pn, vu = synth.make_tape(5, 3, 16)
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    for cfgd in [c for c in pins_mod.OPTION_CONFIGS if c.get('cutoff_mode') == 'hybrid']:
        restate.sample_diffusion(synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd)), cfgd, *args, pn, vu, num_steps=3)
    for cfgd in [c for c in lfp.LAYER_FORM_CONFIGS if c.get('cutoff_mode') == 'hybrid']:
        b, pn, vu = lfp.chain_inputs()
        args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
        layer_forms.sample_diffusion(synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd)), cfgd, *args, pn, vu, num_steps=3)
        for nb in lfp.RETURN_ALL_BLOCKS:
            cb = dict(cfgd, num_blocks=nb)
            b, pp, lp = lfp.return_all_inputs()
            layer_forms.forward(synth.make_state_dict(1, cb, schedules=restate.make_schedules(cb)), cb, pp, b['protein_v'], b['batch_protein'],
                                lp, b['init_ligand_v'], b['batch_ligand'], return_all=True)
    assert len(calls) == 3 * 1 + 3 * 2 + 3 * 2 + 1 + 2, calls       # graphs: 3 steps x blocks per chain, one per block per forward


def test_lattice_pocket_ties_and_duplicates():
    """The lattice pocket's squared distances are exact (multiples of LATTICE^2 / 4), so rows tie at the k-th place; the duplicates
    repeat sites of smaller index; the tie ligand sits on sites, on half-lattice points and in coincident pairs."""
    p = synth.lattice_pocket(1, 120, n_dup=6)
    l = synth.tie_ligand(2, p)
    d2 = restate._d2_fp32(torch.from_numpy(p), torch.from_numpy(p))
    assert np.all(np.mod(d2, synth.LATTICE ** 2 / 4) == 0)
    s = np.sort(d2, axis=1)
    assert all((s[:, k] == s[:, k + 1]).mean() > 0.5 for k in (8, 32, 48))          # most rows tie across the k-th place
    for i in range(114, 120):
        assert (d2[i, :i] == 0).any()
    dl = restate._d2_fp32(torch.from_numpy(l), torch.from_numpy(p))
    assert (dl[:4].min(1) == 0).all() and (dl[4:].min(1) > 0).all()
    assert np.array_equal(l[-6::2], l[-5::2])


def test_near_tie_triples_flip_under_fma():
    """Each triple of the near-tie graph: a before b under the canonical fp32 key, b before a under both FMA contractions and exact d2;
    in the all-protein role a and b are q's two nearest atoms, so the pair is in q's cached protein keys."""
    rng = np.random.RandomState(0)
    for i in range(6):
        q, a, b = synth.near_tie_triple(rng, np.full(3, 20.0 + 7 * i))
        assert synth._d2_orders(q, a, b) == [True, False, False, False]
    p, l = synth.near_tie_graph(3)
    assert len(p) == 6 * 2 + 6 + 6 * 3 + 60 and len(l) == 6 + 6 * 2 + 6 * 3          # four roles of 6 triples each, 60 fill atoms
    d2 = synth.d2_fp32(p, p)
    q, a, b = len(p) - 60 - 3, len(p) - 60 - 2, len(p) - 60 - 1                    # the last all-protein triple
    assert list(np.argsort(d2[q], kind='stable')[1:3]) == [a, b]


def test_ragged_batch_layout():
    b = synth.make_ragged_batch(5, [300, 57, 30, 0, 120], [20, 1, 0, 7, 33])
    assert torch.bincount(b['batch_protein'], minlength=5).tolist() == [300, 57, 30, 0, 120]
    assert torch.bincount(b['batch_ligand'], minlength=5).tolist() == [20, 1, 0, 7, 33]
    assert b['protein_v'].shape == (507, synth.PROTEIN_FEATURE_DIM) and int(b['init_ligand_v'].max()) < synth.LIGAND_NUM_CLASSES
