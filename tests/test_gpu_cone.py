"""The backward cone of the sampling loop's last block (DESIGN.md section 4.3; run with -m gpu).

A sampling step reads only the ligand rows of the network's output, so x2h evaluation g of the last block runs only on the
destinations within G - 1 - g hops of the relevant nodes (ligand atoms and their neighbours), and its node GEMMs only on those rows
(A blocks, q) and one hop further (B blocks).  Rows are independent, so every chain must be bit-identical to the same chain computed
on every row (TDIFF_NO_RESTRICT=1), and the engine's lists must be the sets a host breadth-first search over its own edge_index gives.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import restate, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(cfgd):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfgd or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(synth.make_state_dict(3, cfgd, schedules=restate.make_schedules(cfgd)), strict=True)
    return m.to(DEV)


def _args(b):
    return tuple(b[k].to(DEV) for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))


def _pocket_1h36(n_graphs, n_ligand=25, wall=0.0, seed=2021):
    """The 1h36 pocket n_graphs times, each with n_ligand atoms at sigma = 1 A around the pocket centroid, moved towards the wall by
    the fraction `wall` of the pocket radius."""
    from targetdiff_b200.pocket import pdb_to_pocket_data
    data = pdb_to_pocket_data(os.path.join(ROOT, 'tests', 'golden', '1h36_pocket10.pdb'))
    p = data.protein_pos
    g = torch.Generator().manual_seed(seed)
    bl = torch.arange(n_graphs).repeat_interleave(n_ligand)
    centre = p.mean(0, keepdim=True) + torch.tensor([[wall, 0.0, 0.0]]) * float((p - p.mean(0)).norm(dim=1).max())
    return dict(protein_pos=p.repeat(n_graphs, 1), protein_v=data.protein_atom_feature.float().repeat(n_graphs, 1),
                batch_protein=torch.arange(n_graphs).repeat_interleave(p.shape[0]),
                init_ligand_pos=centre + torch.randn(len(bl), 3, generator=g),
                init_ligand_v=torch.randint(0, synth.LIGAND_NUM_CLASSES, (len(bl),), generator=g), batch_ligand=bl)


def _ragged_wall(seed=7):
    """Ragged pockets and ligands, each ligand moved most of the way to its pocket's wall."""
    b = synth.make_batch(seed, 4, n_protein=180, ligand_sizes=[9, 30, 3, 17])
    for gi in range(4):
        p = b['protein_pos'][b['batch_protein'] == gi]
        sel = b['batch_ligand'] == gi
        b['init_ligand_pos'][sel] = b['init_ligand_pos'][sel] - b['init_ligand_pos'][sel].mean(0) + p.mean(0) + \
            torch.tensor([0.8, 0.0, 0.0]) * float((p - p.mean(0)).norm(dim=1).max())
    return b


BATCHES = {
    'cfg3_subset': lambda: synth.make_batch(100, 8, n_protein=300, n_ligand=20, distinct_pockets=4),
    '1h36': lambda: _pocket_1h36(4),
    'cfg5_k48': lambda: synth.make_batch(101, 2, n_protein=1200, n_ligand=40),
    'ragged_wall': _ragged_wall,
    '1h36_wall': lambda: _pocket_1h36(3, n_ligand=12, wall=0.8),
}
CFG = {'cfg5_k48': {'knn': 48}}


def _sample(b, cfgd, restrict, **kw):
    if not restrict:
        os.environ['TDIFF_NO_RESTRICT'] = '1'
    try:
        model = _model(cfgd)
        r = model.sample_diffusion(*_args(b), center_pos_mode='protein', **kw)
    finally:
        os.environ.pop('TDIFF_NO_RESTRICT', None)
    return r, model


def _assert_same(a, r):
    assert torch.equal(a['pos'], r['pos']) and torch.equal(a['v'], r['v'])
    for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
        assert torch.equal(torch.stack(a[k]), torch.stack(r[k])), k


def _both(b, cfgd, **kw):
    ref, _ = _sample(b, cfgd, False, **kw)
    got, model = _sample(b, cfgd, True, **kw)
    _assert_same(ref, got)
    return model


def _tape(b, S, seed=11):
    return synth.make_tape(seed, S, int(b['init_ligand_pos'].shape[0]))


@pytest.mark.parametrize('name', list(BATCHES))
def test_cone_chain_bit_identical(name):
    b = BATCHES[name]()
    S = 5
    _both(b, CFG.get(name), num_steps=S, noise_tape=_tape(b, S))


@pytest.mark.parametrize('cfgd', [{'cutoff_mode': 'hybrid'}, {'num_blocks': 2}, {'num_x2h': 2}, {'sync_twoup': True},
                                  {'num_x2h': 2, 'num_h2x': 2, 'sync_twoup': True, 'ew_net_type': 'r'}, {'ew_net_type': 'm'}],
                         ids=lambda c: ','.join('%s=%s' % kv for kv in c.items()))
def test_cone_layer_forms_bit_identical(cfgd):
    b = _ragged_wall(9)
    S = 4
    _both(b, cfgd, num_steps=S, noise_tape=_tape(b, S))


def test_cone_seeded_fixed_respaced_start():
    """Seeded chains (device Philox), with fixed atoms, on a respaced time sequence and from a start ligand."""
    from targetdiff_b200.sampling import respaced_time_seq
    b = _pocket_1h36(3, n_ligand=14)
    n = int(b['init_ligand_pos'].shape[0])
    mask = torch.zeros(n, dtype=torch.bool)
    mask[::4] = True
    _both(b, None, num_steps=4, seed=1234)
    _both(b, None, num_steps=4, seed=99, fixed_mask=mask.to(DEV))
    _both(b, None, time_seq=respaced_time_seq(1000, 5), seed=5)
    _both(b, None, time_seq=[60, 40, 25, 10, 0], start_time=60, seed=7, fixed_mask=mask.to(DEV))


# ---- the lists themselves against a host restatement
def _host_cone(ei, is_lig, G, n_dirty):
    """Per evaluation g the protein nodes of (its destinations, its B-block rows), by breadth-first search from the relevant set along
    src."""
    src, dst = ei
    rel = is_lig.copy()
    rel[src[is_lig[dst]]] = True
    far = 1 << 30
    dist = np.where(rel, 0, far)
    for r in range(G):
        s = src[dist[dst] == r]
        dist[s[dist[s] > r + 1]] = r + 1
    touched = is_lig.copy()
    touched[dst[is_lig[src]]] = True
    dirty = [touched]
    while len(dirty) < n_dirty:
        d = dirty[-1].copy()
        d[dst[dirty[-1][src]]] = True
        dirty.append(d)
    out = []
    for g in range(G):
        a = ~is_lig & (dist <= G - 1 - g)
        if g < n_dirty:
            a &= dirty[g]
        out.append((set(np.nonzero(a)[0].tolist()), set(np.nonzero(~is_lig & (dist <= G - g))[0].tolist())))
    assert out[-1][0] == set(np.nonzero(rel & ~is_lig)[0].tolist())      # the last evaluation: the relevant nodes
    return out


@pytest.mark.parametrize('name,n_dirty', [('cfg3_subset', 2), ('1h36_wall', 2), ('cfg5_k48', 0), ('ragged_wall', 2)])
def test_cone_lists_match_host_bfs(name, n_dirty):
    from targetdiff_b200 import _lib
    b = BATCHES[name]()
    cfgd = CFG.get(name)
    S = 3
    _, model = _sample(b, cfgd, True, num_steps=S, noise_tape=_tape(b, S))
    lib = _lib.load()
    eng = model.engine(DEV)
    torch.cuda.synchronize()
    dims = (ctypes.c_int32 * 2)()
    _lib.check(lib.tdiff_get_cone(eng, dims, None, None))
    G, stride = dims
    assert G == 9
    counts = np.zeros((2 * G, 4), np.int32)
    rows = np.zeros((2 * G, stride), np.int32)
    _lib.check(lib.tdiff_get_cone(eng, dims, counts.ctypes.data_as(ctypes.c_void_p), rows.ctypes.data_as(ctypes.c_void_p)))
    st = torch.cuda.current_stream(torch.device(DEV)).cuda_stream
    E = lib.tdiff_num_edges(eng, ctypes.c_void_p(st))
    ei = torch.empty(2, E, dtype=torch.int64, device=DEV)
    _lib.check(lib.tdiff_get_edge_index(eng, ctypes.c_void_p(ei.data_ptr()), ctypes.c_void_p(st)))
    torch.cuda.synchronize()
    ei = ei.cpu().numpy()
    # composed node order: per graph its protein atoms, then its ligand atoms
    pc = torch.bincount(b['batch_protein']).tolist()
    lc = torch.bincount(b['batch_ligand'], minlength=len(pc)).tolist()
    is_lig = np.concatenate([np.r_[np.zeros(p, bool), np.ones(l, bool)] for p, l in zip(pc, lc)])
    N = is_lig.shape[0]
    lig = set(np.nonzero(is_lig)[0].tolist())
    want = _host_cone(ei, is_lig, G, n_dirty)
    sizes = []
    for t in range(2 * G):
        n_ent, split, n_p, _ = counts[t]
        prot = want[t // 2][t % 2]
        assert n_p == len(prot) and split >= n_p and split - n_p < 128 and n_ent - split >= len(lig), t
        assert set(rows[t, :n_p].tolist()) == prot and len(set(rows[t, :n_p].tolist())) == n_p, t      # no duplicates
        assert (rows[t, n_p:split] == -1).all(), t
        assert set(rows[t, split:n_ent].tolist()) - {-1} == lig, t
        sizes.append(int(n_p))
    print('%s: protein nodes of (R_g, R_g-1) per evaluation %s of %d protein nodes' % (name, list(zip(sizes[0::2], sizes[1::2])), N - len(lig)))
