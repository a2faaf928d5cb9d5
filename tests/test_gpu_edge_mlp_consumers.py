"""The edge-MLP launches at the tile counts where their consumer warpgroups differ (run with -m gpu; `pytest -s` prints the per-layer
error table).

The unfolded NOUT = 128 launches of edge_mlp_v4.cu run three consumer warpgroups per CTA, the folded key and the xv launch two, and
every launch covers one destination class (protein destinations, then ligand destinations) with that class's table resident.  A
consumer takes the CTA's tiles c, c + 3, ...; one without a tile in the CTA's last round only passes the MMA order on.  Here, at
k = 8, 16, 32, 48 and 64:

1. Each class launch with exactly 1, 2 and 3 tiles per CTA (2, 1 and 0 consumers without a tile in the last round), every layer
   against float64 (oracle.layerwise, LAYER_TOL).
2. Launches with fewer tiles than SMs on a batch with a protein-free graph and a graph without ligand atoms (layers against float64),
   and batches where one class is empty on the host: no protein atoms at all, no ligand atoms at all (forward against the fp32 oracle).
3. Short chains that must be bit-identical on the batch, on the same graphs in another order and on each graph alone: the ragged batch
   above (a protein-free graph alone has an empty protein class on the host), and a batch whose ligands lie far from their pockets,
   where the relevant-rows list of the last x2h and the ligand-free cache's dirty lists have an empty protein class in the device
   counts only."""
import math

import pytest
import torch

from oracle import layerwise, restate, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
CONS = 3                                      # consumer warpgroups of the unfolded NOUT = 128 launches
KS = [8, 16, 32, 48, 64]
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')


def _model(cfg, sd):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


def _weights(k):
    cfg = {'knn': k}
    return cfg, synth.make_state_dict(0, cfg, schedules=restate.make_schedules(cfg))


def _graph(seed, n_protein, n_ligand, shift=0.0):
    """One graph: a synthetic pocket of `n_protein` atoms (0: its atoms are dropped, the ligand stays where the pocket was) and a
    ligand of `n_ligand` atoms, moved by `shift` Angstrom along x."""
    b = synth.make_batch(seed, 1, n_protein=n_protein or 40, ligand_sizes=[n_ligand])
    if n_protein == 0:
        b.update(protein_pos=b['protein_pos'][:0], protein_v=b['protein_v'][:0], batch_protein=b['batch_protein'][:0])
    b['init_ligand_pos'] = b['init_ligand_pos'] + torch.tensor([shift, 0.0, 0.0])
    return b


def _batch(graphs):
    """Graphs given as (seed, n_protein, n_ligand[, shift]) concatenated into one batch."""
    parts = [_graph(*g) for g in graphs]
    for i, p in enumerate(parts):
        p['batch_protein'] = p['batch_protein'] + i
        p['batch_ligand'] = p['batch_ligand'] + i
    return {k: torch.cat([p[k] for p in parts]) for k in ARGS}


def _regroup(b, order):
    """The graphs `order` of batch `b`, in that order and renumbered 0.., and the index of their ligand rows in `b`."""
    parts, lig = [], []
    for i, g in enumerate(order):
        sp, sl = b['batch_protein'] == g, b['batch_ligand'] == g
        parts.append({k: (torch.full((int(s.sum()),), i, dtype=torch.long) if k.startswith('batch') else b[k][s])
                      for k, s in (('protein_pos', sp), ('protein_v', sp), ('batch_protein', sp), ('init_ligand_pos', sl),
                                   ('init_ligand_v', sl), ('batch_ligand', sl))})
        lig.append(sl.nonzero().view(-1))
    return {k: torch.cat([p[k] for p in parts]) for k in ARGS}, torch.cat(lig)


def _layers(label, k, b, n_layers):
    cfg, sd = _weights(k)
    rows = layerwise.engine_layer_parity(label, cfg, sd, b, n_layers, _model, DEV, tag='tc3')
    layerwise.check_layers(rows, 'tc3', k)


def _sm():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _idle(n_dst, k, sm):
    """Consumers without a tile in the last round, over the CTAs of a class launch of n_dst destinations (a multiple of the class
    padding, so n_dst * k is a multiple of the 64-row tile)."""
    tiles = n_dst * k // 64
    grid = min(tiles, sm)
    return {(-(tiles // grid + (1 if i < tiles % grid else 0))) % CONS for i in range(grid)}


# ------------------------------------------------------------------------------------------------ 1. tiles per CTA
def _rounds_batch(k, m, sm):
    """Both classes with sm * m tiles: sm * m * 64 / k protein and as many ligand atoms, in graphs of at most ~150 + 150 atoms."""
    n = sm * m * 64 // k
    G = -(-n // 150)
    q, r = divmod(n, G)
    return _batch([(100 + i, q + (i < r), q + (i < r)) for i in range(G)]), n


@pytest.mark.parametrize('m', [1, 2, 3])
@pytest.mark.parametrize('k', KS)
def test_tiles_per_cta_layers_vs_float64(k, m):
    sm = _sm()
    b, n = _rounds_batch(k, m, sm)
    pad = 128 // math.gcd(k, 128)
    assert n % pad == 0 and n * k == 64 * sm * m
    assert _idle(n, k, sm) == {(-m) % CONS}
    _layers('k=%d, %d tiles per CTA' % (k, m), k, b, 2)


# ------------------------------------------------------------------------------------------------ 2. fewer tiles than SMs, empty classes
RAGGED = [(3, 110, 20), (4, 0, 9), (5, 60, 1), (6, 70, 0)]      # a protein-free graph (not the last) and a graph without ligand atoms


@pytest.mark.parametrize('k', KS)
def test_small_ragged_batch_layers_vs_float64(k):
    b = _batch(RAGGED)
    pad = 128 // math.gcd(k, 128)
    up = lambda v: -(-v // pad) * pad
    assert up(len(b['batch_ligand'])) * k // 64 < _sm()              # the ligand-destination launches
    _layers('k=%d ragged' % k, k, b, 3)


@pytest.mark.parametrize('case', ['no_ligand', 'no_protein'])
@pytest.mark.parametrize('k', [8, 32, 48])
def test_empty_class_forward_vs_oracle(k, case):
    """One class empty on the host.  No ligand atoms: the x2h launches cover protein destinations only and the h2x launches do not
    run.  No protein atoms: every launch covers ligand destinations only.  (The float64 layer reference needs ligand rows and a
    pocket to centre on, so this compares the forward with the fp32 oracle, uncentred.)"""
    cfg, sd = _weights(k)
    b = _batch([(7, 90, 0), (8, 50, 0)] if case == 'no_ligand' else [(9, 0, 40), (10, 0, 12)])
    tr = {}
    want = restate.forward(sd, cfg, *(b[a] for a in ARGS), trace=tr)
    out = _model(cfg, sd)(*(b[a].to(DEV) for a in ARGS))
    assert torch.equal(out['edge_index'].cpu(), tr['edge_index'])
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=1e-3)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------ 3. chains: reordered and per graph
def _chain(model, b, pn, vu, center):
    r = model.sample_diffusion(*(b[k].to(DEV) for k in ARGS), num_steps=pn.shape[0], center_pos_mode=center, noise_tape=(pn, vu),
                               stack_traj=True)
    return {k: r[k].cpu() for k in TRAJ}


def _rows(r, idx):
    return {k: (r[k][idx] if k in ('pos', 'v') else r[k][:, idx]) for k in TRAJ}


def _differing(a, c):
    return [k for k in TRAJ if not torch.equal(a[k], c[k])]


def _far_batch(k):
    """Ligands of k + 4 atoms 80 Angstrom from pockets of more than k atoms: no edge joins a ligand and a protein atom, so no protein
    atom is relevant to the last x2h and none becomes dirty in the ligand-free cache."""
    return _batch([(20 + i, 2 * k + 10 * i, k + 4, 80.0) for i in range(3)])


@pytest.mark.parametrize('case', ['ragged', 'far'])
@pytest.mark.parametrize('k', KS)
def test_chain_reordered_and_per_graph_bit_identical(k, case):
    cfg, sd = _weights(k)
    b = _batch(RAGGED) if case == 'ragged' else _far_batch(k)
    center = 'none' if case == 'ragged' else 'protein'        # the ragged batch has a graph without pocket to centre on
    G = int(b['batch_ligand'].max()) + 1 if case == 'far' else len(RAGGED)
    S = 4
    pn, vu = synth.make_tape(11, S, len(b['batch_ligand']))
    model = _model(cfg, sd)
    r = _chain(model, b, pn, vu, center)
    perm = torch.randperm(G, generator=torch.Generator().manual_seed(k)).tolist()
    bp, idx = _regroup(b, perm)
    rp = _chain(model, bp, pn[:, idx], vu[:, idx], center)
    bad = _differing(rp, _rows(r, idx))
    print('k=%d %s: reordered %s differs in %s' % (k, case, perm, bad))
    assert not bad, bad
    for g in range(G):
        bg, idx = _regroup(b, [g])
        if len(idx) == 0:
            continue                                            # no ligand atoms: nothing to sample
        same = _chain(model, bg, pn[:, idx], vu[:, idx], center)
        bad = _differing(same, _rows(r, idx))
        print('k=%d %s: graph %d alone differs in %s' % (k, case, g, bad))
        assert not bad, (g, bad)
