"""The engine's neighbour lists where they are decided by ties, and batches whose graphs differ in protein count (run with -m gpu;
`pytest -s` prints what each check compared).

Every batch of the other GPU tests repeats one protein count, and their random coordinates never put two squared distances of a row
within an ulp.  Whenever a batch has protein atoms the engine builds its graph with `knn_protein_cache_kernel` (each protein atom's
k + 1 smallest protein keys, once per bound batch) and `knn_update_kernel` (those keys merged with the ligand keys by rank counting),
and hybrid ligand rows with `hybrid_ligand_row`; the full scan `knn_kernel` runs only under TDIFF_KNN_FULL=1 and in ops.knn_graph.
Geometry from oracle/synth.py:
* 'lattice': pockets on a cubic lattice of spacing 1.5 (squared distances exact, rows tie across the k-th place), ligand atoms on
  half-lattice points, and a graph of exactly k + 1 nodes with at most k protein atoms;
* 'coincident': lattice pockets with duplicated sites (a coincident protein atom precedes the query), ligand atoms on protein sites
  and in coincident pairs;
* 'near_tie': triples whose order under the canonical fp32 key differs from both FMA-contracted and exact d2, with q, a, b as
  ligand / protein / protein, protein / ligand / ligand, all ligand and all protein (the pair then in q's cached protein keys).
1. k-NN at ties, k = 1, 8, 32, 48, 64: the forward's edge_index bit-exact against restate.knn_graph_canonical on the incremental
   path and with TDIFF_KNN_FULL=1; ops.knn_graph the same.
2. Later blocks (num_blocks 2, 3): each block's graph equals the canonical graph of the engine's own return_all coordinates.
3. Hybrid, k = 8, 21, 32, on the same geometry and `synth.hybrid_norm_tie_graph`: the edge set equals
   restate.hybrid_graph_canonical bit for bit (and differs from the reference's norm + topk only at the constructed tie), degrees.
4. Ragged pockets, protein [300, 57, 30, 0, 120] / ligand [20, 1, 0, 7, 33]: forward and return_all, a 6-step chain and
   likelihood_estimation against the oracle; the chain bit-identical under TDIFF_KNN_FULL, TDIFF_NO_SLOT_KEEP and TDIFF_FREE_DEPTH=0
   (also with every graph above k protein atoms, where the ligand-free cache is on, and with ligand atoms beside fewer than k protein
   atoms in a later graph, where the bind gate turns it off), with the graphs in another order, and per graph run alone.
5. Coincident atoms (d = 0 edges into the gaussians, the gate and h2x's rel_x): forward finite and within tolerance of the oracle,
   all 9 layers within LAYER_TOL of float64.
6. Size edges: a 2800-node graph (224,000 B of k-NN shared memory), alone and beside small graphs, at k = 32 and 64; 2801 refused."""
import math
import time

import numpy as np
import pytest
import torch

from oracle import layer_forms, layerwise, restate, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')
POS_RTOL, POS_ATOL, LOGIT_ATOL = 1e-4, 1e-5, 1e-3          # against the fp32 oracle, as in the other GPU tests
RAGGED_P, RAGGED_L = [300, 57, 30, 0, 120], [20, 1, 0, 7, 33]
RAGGED_P_CACHED = [300, 57, 40, 45, 120]                    # every graph above k = 32 protein atoms: the ligand-free cache is on
RAGGED_FEW = ([300, 20, 30, 0, 120], [20, 6, 0, 7, 33])     # graph 1: ligand atoms beside fewer than k protein atoms: gate off


def _model(cfg, sd):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


def _weights(cfg, seed=0):
    return synth.make_state_dict(seed, cfg, schedules=restate.make_schedules(cfg))


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ARGS)


def _composed(b):
    """(x, mask_ligand, batch) of batch `b` in the engine's node order: per graph its protein atoms, then its ligand atoms."""
    z = lambda t: torch.zeros(len(t), 1)
    _, x, batch, mask = restate.compose_context(z(b['protein_pos']), z(b['init_ligand_pos']), b['protein_pos'], b['init_ligand_pos'],
                                                b['batch_protein'], b['batch_ligand'])
    return x, mask, batch


def _small_graph(k, seed):
    """k + 1 nodes, ceil((k + 1) / 2) <= k of them protein atoms on the lattice, the ligand atoms on half-lattice points."""
    n_p = (k + 2) // 2
    p = synth.lattice_pocket(seed, n_p)
    l = synth.lattice_pocket(seed + 1, k + 1 - n_p, origin=(3.75, -3.75, 2.25)) if k + 1 > n_p else np.zeros((0, 3), np.float32)
    return p, l


def tie_batch(kind, k):
    if kind == 'lattice':
        p0, p1 = synth.lattice_pocket(1, 150), synth.lattice_pocket(3, 60, origin=(-6.0, 0.0, 7.5))
        graphs = [(p0, synth.tie_ligand(2, p0, n_site=0, n_half=10, n_pairs=0)), _small_graph(k, 11),
                  (p1, synth.tie_ligand(4, p1, n_site=0, n_half=5, n_pairs=0, origin=(-6.0, 0.0, 7.5)))]
    elif kind == 'coincident':
        p0, p1 = synth.lattice_pocket(4, 120, n_dup=8), synth.lattice_pocket(6, 40, n_dup=4)
        ps = synth.lattice_pocket(12, (k + 2) // 2, n_dup=min(2, (k + 2) // 2 - 1))
        graphs = [(p0, synth.tie_ligand(5, p0, n_site=6, n_half=2, n_pairs=4)), (p1, synth.tie_ligand(7, p1, n_site=3, n_half=0, n_pairs=2)),
                  (ps, ps[:k + 1 - len(ps)])]                                     # k + 1 nodes, every ligand atom on a protein site
    else:
        graphs = [synth.near_tie_graph(3), _small_graph(k, 13), synth.near_tie_graph(4, n_triples=12, n_fill=20)]
    return synth.batch_from_graphs(graphs, seed=k)


TIE_KINDS = ('lattice', 'coincident', 'near_tie')


def _fixed_degree(ei, k):
    """The canonical graph as the engine's fixed-degree slot list holds it (DESIGN.md section 2): a node preceded by k + 1 or more
    coincident atoms, whose k + 1 smallest keys do not include itself, keeps the first k of them.  Returns (graph, such rows)."""
    deg = torch.bincount(ei[1])
    over = (deg > k).nonzero().view(-1)
    keep = torch.ones(ei.shape[1], dtype=torch.bool)
    for d in over.tolist():
        keep[(ei[1] == d).nonzero().view(-1)[k:]] = False
    return ei[:, keep], len(over)


# ------------------------------------------------------------------------------------------------ 1. k-NN at ties
@pytest.mark.parametrize('full', [False, True], ids=['incremental', 'full_scan'])
@pytest.mark.parametrize('k', [1, 8, 32, 48, 64])
def test_knn_at_ties_bit_exact(k, full, monkeypatch):
    """At k = 1 the coincident batch has nodes preceded by two coincident atoms: there the canonical k-NN (like PyG) keeps k + 1
    edges and the engine k, the first k of them."""
    from targetdiff_b200 import ops
    if full:
        monkeypatch.setenv('TDIFF_KNN_FULL', '1')
    cfg = {'knn': k, 'num_layers': 1}
    model = _model(cfg, _weights(cfg))
    for kind in TIE_KINDS:
        b = tie_batch(kind, k)
        x, mask, batch = _composed(b)
        want, n_over = _fixed_degree(restate.knn_graph_canonical(x, k, batch), k)
        got = model(*_args(b))['edge_index'].cpu()
        s = ops.knn_graph(x.to(DEV), k, batch.to(DEV)).cpu()
        print('k=%-2d %-11s %-10s %5d nodes %6d edges (%d rows cut to k): engine %s, ops.knn_graph %s' %
              (k, 'full scan' if full else 'incremental', kind, len(x), want.shape[1], n_over, torch.equal(got, want), torch.equal(s, want)))
        assert n_over == 0 or (k == 1 and kind == 'coincident')
        assert torch.equal(got, want), kind
        assert torch.equal(s, want), kind


# ------------------------------------------------------------------------------------------------ 2. later blocks
@pytest.mark.parametrize('k', [8, 32])
@pytest.mark.parametrize('blocks', [2, 3])
def test_later_block_graphs_from_return_all(blocks, k):
    """Block b's graph (edge_index of the b + 1-block network) equals the canonical graph of the coordinates the B-block network's
    return_all gives before block b: the cached protein keys merged with moved ligand atoms."""
    cfg = {'knn': k, 'num_layers': 1}
    sd = _weights(cfg, seed=2)
    for kind in ('coincident', 'lattice'):
        b = tie_batch(kind, k)
        x, mask, batch = _composed(b)
        full = _model(dict(cfg, num_blocks=blocks), sd)(*_args(b), return_all=True)
        for nb in range(1, blocks + 1):
            xb = x.clone()
            xb[mask] = full['layer_pred_ligand_pos'][nb - 1].cpu()
            got = _model(dict(cfg, num_blocks=nb), sd)(*_args(b))['edge_index'].cpu()
            assert torch.equal(got, restate.knn_graph_canonical(xb, k, batch)), (kind, nb)


# ------------------------------------------------------------------------------------------------ 3. hybrid
def _edges(ei):
    return set(map(tuple, ei.T.tolist()))


@pytest.mark.parametrize('full', [False, True], ids=['incremental', 'full_scan'])
@pytest.mark.parametrize('k', [8, 21, 32])
def test_hybrid_at_ties_bit_exact(k, full, monkeypatch):
    if full:
        monkeypatch.setenv('TDIFF_KNN_FULL', '1')
    p0 = synth.lattice_pocket(1, 120)
    p1 = synth.lattice_pocket(4, 100, n_dup=8)
    graphs = [(p0, synth.tie_ligand(2, p0)), (p1, synth.tie_ligand(5, p1, n_site=6, n_half=2, n_pairs=3)),
              synth.near_tie_graph(4, n_triples=12), synth.hybrid_norm_tie_graph(k)]
    b = synth.batch_from_graphs(graphs, seed=k)
    x, mask, batch = _composed(b)
    cfg = {'cutoff_mode': 'hybrid', 'knn': k, 'num_layers': 1}
    got = _model(cfg, _weights(cfg))(*_args(b))['edge_index'].cpu()
    want = restate.hybrid_graph_canonical(x, k, mask, batch)
    mirror = restate.hybrid_graph(x, k, mask, batch)
    assert got.shape == want.shape and _edges(got) == _edges(want)
    deg = torch.bincount(got[1], minlength=len(x))
    nl = torch.bincount(batch[mask], minlength=len(graphs))
    ng = torch.bincount(batch, minlength=len(graphs))
    assert torch.equal(deg[mask], nl[batch[mask]] - 1 + k)
    assert torch.equal(deg[~mask], torch.clamp(ng[batch[~mask]] - 1, max=k))
    # the reference's norm + topk keeps protein atom k instead of k - 1 of the last graph's tie row; nothing else differs
    base = int((batch < len(graphs) - 1).sum())
    q = base + int((~mask[batch == len(graphs) - 1]).sum())
    diff = {e for e in _edges(mirror) ^ _edges(want) if e[1] >= base}        # (exact ties of the lattice graphs topk orders freely)
    print('hybrid k=%d %s: %d edges, engine == canonical, differs from norm + topk at %s' %
          (k, 'full scan' if full else 'incremental', got.shape[1], sorted(diff)))
    assert diff == {(base + k, q), (base + k - 1, q)}


# ------------------------------------------------------------------------------------------------ 4. ragged pockets
def _ragged(p=RAGGED_P, l=RAGGED_L):
    return synth.make_ragged_batch(21, p, l)


def _chain(model, b, pn, vu):
    r = model.sample_diffusion(*_args(b), num_steps=pn.shape[0], center_pos_mode='protein', noise_tape=(pn, vu), stack_traj=True)
    return {k: r[k].cpu() for k in TRAJ}


def _differing(a, c):
    return [k for k in TRAJ if not torch.equal(a[k], c[k])]


def _rows(r, idx):
    return {k: (r[k][idx] if k in ('pos', 'v') else r[k][:, idx]) for k in TRAJ}


def _regroup(b, order):
    """The graphs `order` of batch `b` in that order, renumbered 0.., and the index of their ligand rows in `b`."""
    parts, lig = [], []
    for i, g in enumerate(order):
        sp, sl = b['batch_protein'] == g, b['batch_ligand'] == g
        parts.append({k: (torch.full((int(s.sum()),), i, dtype=torch.long) if k.startswith('batch') else b[k][s])
                      for k, s in (('protein_pos', sp), ('protein_v', sp), ('batch_protein', sp), ('init_ligand_pos', sl),
                                   ('init_ligand_v', sl), ('batch_ligand', sl))})
        lig.append(sl.nonzero().view(-1))
    return {k: torch.cat([p[k] for p in parts]) for k in ARGS}, torch.cat(lig)


def test_ragged_forward_and_return_all_vs_oracle():
    """Two blocks, so return_all has an entry between the blocks; edge_index is block 1's graph."""
    cfg = {'num_blocks': 2}
    sd = _weights(cfg, seed=3)
    b = _ragged()
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    b = dict(b, protein_pos=pp, init_ligand_pos=lp)
    tr = {}
    want = layer_forms.forward(sd, cfg, *_args(b, 'cpu'), trace=tr, return_all=True)
    out = _model(cfg, sd)(*_args(b), return_all=True)
    assert torch.equal(out['edge_index'].cpu(), tr['block_edge_index'][-1])
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=1e-4, atol=1e-4)
    assert len(out['layer_pred_ligand_pos']) == len(want['layer_pred_ligand_pos']) == 3
    for g, w in zip(out['layer_pred_ligand_pos'], want['layer_pred_ligand_pos']):
        torch.testing.assert_close(g.cpu(), w, rtol=POS_RTOL, atol=POS_ATOL)
    for g, w in zip(out['layer_pred_ligand_v'], want['layer_pred_ligand_v']):
        torch.testing.assert_close(g.cpu(), w, rtol=0, atol=LOGIT_ATOL)


@pytest.fixture(scope='module')
def ragged_chain():
    sd = _weights({}, seed=4)
    b = _ragged()
    pn, vu = synth.make_tape(8, 6, len(b['batch_ligand']))
    model = _model({}, sd)
    return sd, b, pn, vu, model, _chain(model, b, pn, vu)


def test_ragged_chain_vs_oracle(ragged_chain):
    sd, b, pn, vu, _, got = ragged_chain
    w = restate.sample_diffusion(sd, None, *_args(b, 'cpu'), pn, vu, num_steps=6)
    assert torch.equal(got['v_traj'], torch.stack(w['v_traj'])) and torch.equal(got['v'], w['v'])
    torch.testing.assert_close(got['pos_traj'], torch.stack(w['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['pos'], w['pos'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['v0_traj'], torch.stack(w['v0_traj']), rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(got['vt_traj'], torch.stack(w['vt_traj']), rtol=0, atol=LOGIT_ATOL)


def test_ragged_likelihood_vs_oracle():
    sd = _weights({}, seed=5)
    b = _ragged()
    model = _model({}, sd)
    pn, vu = synth.make_tape(9, 1, len(b['batch_ligand']))
    for t in (torch.tensor([0, 999, 417, 3, 500]), torch.full((5,), 1000)):
        want = restate.likelihood_estimation(sd, None, *_args(b, 'cpu'), t, pn[0], vu[0])
        got = model.likelihood_estimation(*_args(b), time_step=t.to(DEV), noise=(pn[0], vu[0]))
        for g, w in zip(got, want):
            assert g.shape == (5,) and float(g[2]) == 0.0                  # graph 2 has no ligand atom
            torch.testing.assert_close(g.cpu(), w, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize('proteins,ligands', [(RAGGED_P, RAGGED_L), (RAGGED_P_CACHED, RAGGED_L), RAGGED_FEW],
                         ids=['with_empty_pocket', 'all_above_k', 'ligand_beside_few_protein'])
def test_ragged_chain_bit_identical_under_switches(proteins, ligands, monkeypatch):
    sd = _weights({}, seed=4)
    b = _ragged(proteins, ligands)
    pn, vu = synth.make_tape(8, 6, len(b['batch_ligand']))
    base = _chain(_model({}, sd), b, pn, vu)
    for env in ('TDIFF_KNN_FULL', 'TDIFF_NO_SLOT_KEEP', 'TDIFF_FREE_DEPTH'):
        with monkeypatch.context() as mp:
            mp.setenv(env, '0' if env == 'TDIFF_FREE_DEPTH' else '1')
            bad = _differing(_chain(_model({}, sd), b, pn, vu), base)
        print('ragged %s, %s: outputs differing %s' % (proteins, env, bad))
        assert not bad, env


def test_ragged_reordered_and_single_graphs_bit_identical(ragged_chain):
    sd, b, pn, vu, model, r = ragged_chain
    perm = [4, 2, 0, 3, 1]                        # the graph without protein atoms stays before the last one
    bp, idx = _regroup(b, perm)
    bad = _differing(_chain(model, bp, pn[:, idx], vu[:, idx]), _rows(r, idx))
    assert not bad, bad
    fresh = _model({}, sd)
    for g in [g for g, n in enumerate(RAGGED_L) if n]:
        bg, idx = _regroup(b, [g])
        want = _rows(r, idx)
        same, new = _chain(model, bg, pn[:, idx], vu[:, idx]), _chain(fresh, bg, pn[:, idx], vu[:, idx])
        print('ragged graph %d (%d protein, %d ligand atoms) alone: differs %s (same model) / %s (fresh model)' %
              (g, RAGGED_P[g], RAGGED_L[g], _differing(same, want), _differing(new, want)))
        assert not _differing(same, want) and not _differing(new, want), g


# ------------------------------------------------------------------------------------------------ 5. coincident atoms
def test_coincident_atoms_forward_and_layers():
    k = 32
    b = tie_batch('coincident', k)
    sd = _weights({})
    x, mask, batch = _composed(b)
    assert (restate._d2_fp32(x[mask], x) == 0).sum() > int(mask.sum())       # d = 0 pairs besides each atom with itself
    want = restate.forward(sd, None, *_args(b, 'cpu'))
    out = _model({}, sd)(*_args(b))
    for key in ('pred_ligand_pos', 'pred_ligand_v', 'final_h'):
        assert torch.isfinite(out[key]).all(), key
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=LOGIT_ATOL)
    rows = layerwise.engine_layer_parity('coincident k=%d' % k, {}, sd, b, 9, _model, DEV, tag='tc3')
    for r in rows:
        assert all(math.isfinite(v) for v in r), r
    layerwise.check_layers(rows, 'tc3', k)


# ------------------------------------------------------------------------------------------------ 6. size edges
BIG = 2800


def _big_graphs(n_nodes, mixed):
    p, _ = synth.make_pocket(77, n_nodes - 40)
    g = torch.Generator().manual_seed(5)
    big = (p, p.mean(0, keepdim=True) + torch.randn(40, 3, generator=g))
    if not mixed:
        return synth.batch_from_graphs([big], seed=1)
    small = []
    for seed, n_p, n_l in ((78, 60, 10), (79, 30, 5)):
        q, _ = synth.make_pocket(seed, n_p)
        small.append((q, q.mean(0, keepdim=True) + torch.randn(n_l, 3, generator=g)))
    return synth.batch_from_graphs([small[0], big, small[1]], seed=1)


@pytest.mark.parametrize('k', [32, 64])
def test_largest_graph(k, monkeypatch):
    """A graph of 2800 nodes (the bind limit) alone and between two small graphs: edge_index against the canonical graph on both
    k-NN paths; beside the small graphs, layer 0 against float64."""
    cfg = {'knn': k}
    sd = _weights(cfg)
    for mixed in (False, True):
        b = _big_graphs(BIG, mixed)
        x, mask, batch = _composed(b)
        want = restate.knn_graph_canonical(x, k, batch)
        t0 = time.perf_counter()
        got = _model(dict(cfg, num_layers=1), layerwise.prefix_state_dict(sd, 1))(*_args(b))['edge_index'].cpu()
        print('%d-node graph%s, k=%d: %d edges, engine == canonical %s (%.1f s)' %
              (BIG, ' with two small graphs' if mixed else '', k, want.shape[1], torch.equal(got, want), time.perf_counter() - t0))
        assert torch.equal(got, want), mixed
    with monkeypatch.context() as mp:
        mp.setenv('TDIFF_KNN_FULL', '1')
        got = _model(dict(cfg, num_layers=1), layerwise.prefix_state_dict(sd, 1))(*_args(b))['edge_index'].cpu()
    assert torch.equal(got, want)
    rows = layerwise.engine_layer_parity('%d nodes k=%d' % (BIG, k), cfg, sd, b, 1, _model, DEV, tag='tc3')
    layerwise.check_layers(rows, 'tc3', k)


def test_graph_above_bind_limit_refused():
    from targetdiff_b200._lib import TdiffError
    cfg = {'num_layers': 1}
    b = _big_graphs(BIG + 1, False)
    with pytest.raises(TdiffError, match='graph with 2801 nodes exceeds'):
        _model(cfg, _weights(cfg))(*_args(b))
