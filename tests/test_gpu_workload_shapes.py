"""The sampling chain at the shapes bench.py measures -- cfg2, cfg3 and cfg5 (bench.WORKLOADS), the batches bench.make_workload
builds -- against itself on a reordered batch, against single-graph runs, the fp32 oracle and float64 (run with -m gpu; `pytest -s`
prints every comparison).

The other GPU tests run graphs one to three orders of magnitude smaller than these: tens of edge-MLP tiles per CTA instead of
hundreds, a few thousand ligand atoms at most, a handful of ragged ligand sizes.  A fault that needs the full size (a tile counter
past 65,536, a barrier phase after hundreds of tiles per CTA, the class-list padding of one particular mix of ragged sizes, a launch
cap past some node count) would pass all of them.  Per workload, with synthetic weights at the workload's k and a noise tape:

1. Reorder invariance.  The chain (graph-replayed, all four trajectories) on the batch and on the same graphs in a fixed random
   order, the tape rows permuted with the ligand atoms: after undoing the permutation every trajectory and the final state are
   bit-identical.  The permutation moves graphs across CTAs, tiles and, for cfg2, the padding of the ragged ligand class.
2. Single-graph anchors (first, last, and the middle graph or the largest and smallest ligand): each graph alone on the same model
   (re-bound after the batch: its buffers still hold the batch's data) and on a fresh model equals its rows of the batch bit for
   bit, and its chain matches `restate.sample_diffusion` at the chain tolerances of the other tests.
3. One anchor against float64: all 9 layers (oracle.layerwise, LAYER_TOL) and every chain step (oracle.stepwise, STEP_TOL; pocket
   at the origin, center_pos_mode='none').  For cfg5 this is the k = 48 network on a 1240-atom graph.
4. cfg3 with a seed: the device stream equals `philox.engine_tape` on all 12,800 ligand atoms.

Also here, a value edge rather than a shape edge: 5. attention logits of |logit| >= 100 (q scaled up), where exp overflows fp32
without the softmax's max shift, layer by layer against float64 at k = 8, 32, 48 and 64."""
import math
import time
from types import SimpleNamespace

import pytest
import torch

import bench
from oracle import layerwise, philox, restate, stepwise, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K = synth.LIGAND_NUM_CLASSES
POS_RTOL, POS_ATOL, LOGIT_ATOL = 1e-4, 1e-5, 1e-3      # chain against the fp32 oracle, as in the other GPU tests
STEPS = {'cfg2': 4, 'cfg3': 4, 'cfg5': 3}               # the caches are built at step 0 and reused from step 1 on
TRAJ = ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj', 'pos', 'v')
ARGS = ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand')


def _model(cfg, sd):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


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


def _chain(model, b, pn, vu):
    r = model.sample_diffusion(*(b[k].to(DEV) for k in ARGS), num_steps=pn.shape[0], center_pos_mode='protein', noise_tape=(pn, vu),
                               stack_traj=True)
    return {k: r[k].cpu() for k in TRAJ}


def _rows(r, idx):
    """The ligand rows `idx` of every trajectory (atoms are dim 1 of a trajectory, dim 0 of the final state)."""
    return {k: (r[k][idx] if k in ('pos', 'v') else r[k][:, idx]) for k in TRAJ}


def _differing(a, c):
    """Names of the outputs that are not bit-identical."""
    return [k for k in TRAJ if not torch.equal(a[k], c[k])]


def _device_mem_gb():
    free, total = torch.cuda.mem_get_info(DEV)
    return (total - free) / 1e9


@pytest.fixture(scope='module', params=['cfg2', 'cfg3', 'cfg5'])
def workload(request):
    """One bench workload: weights, batch, tape, and the chain on the batch.  One workload at a time is alive on the device."""
    w = request.param
    t0 = time.perf_counter()
    a = SimpleNamespace(workload=w, **bench.WORKLOADS[w])
    b, G, N, Nl = bench.make_workload(a, 0)
    cfg = {'knn': a.knn}
    sd = synth.make_state_dict(0, cfg, schedules=restate.make_schedules())
    S = STEPS[w]
    pn, vu = synth.make_tape(77, S, Nl)
    model = _model(cfg, sd)
    r = _chain(model, b, pn, vu)
    sizes = torch.bincount(b['batch_ligand'], minlength=G)
    print('\n%s: %d graphs, %d nodes, %d ligand atoms (sizes %d..%d), k=%d, %d steps; batch chain + set-up %.1f s, device memory in use '
          '%.2f GB' % (w, G, N, Nl, int(sizes.min()), int(sizes.max()), a.knn, S, time.perf_counter() - t0, _device_mem_gb()))
    yield SimpleNamespace(name=w, cfg=cfg, sd=sd, b=b, G=G, sizes=sizes, pn=pn, vu=vu, model=model, r=r, S=S)
    del model, r
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _anchors(wl):
    G = wl.G
    if wl.name == 'cfg2':
        extra = [int(torch.argmax(wl.sizes)), int(torch.argmin(wl.sizes))]     # the largest and the smallest prior size
    else:
        extra = [G // 2 + 1]                                                   # from the middle of the batch
    return list(dict.fromkeys([0, G - 1] + extra))


# ------------------------------------------------------------------------------------------------ 1. reorder invariance
def test_reordered_batch_is_bit_identical(workload):
    wl = workload
    perm = torch.randperm(wl.G, generator=torch.Generator().manual_seed(5)).tolist()
    bp, idx = _regroup(wl.b, perm)
    rp = _chain(wl.model, bp, wl.pn[:, idx], wl.vu[:, idx])
    bad = _differing(rp, _rows(wl.r, idx))
    n_diff = int((rp['pos_traj'] != wl.r['pos_traj'][:, idx]).any(-1).any(0).sum())
    print('%s reordered batch: outputs differing %s, ligand atoms with another position trajectory %d of %d' %
          (wl.name, bad, n_diff, len(idx)))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ 2. single-graph anchors
def _max_abs(a, c):
    return float((a.double() - c.double()).abs().max())


def test_single_graph_anchors(workload):
    wl = workload
    fresh = _model(wl.cfg, wl.sd)
    for g in _anchors(wl):
        bg, idx = _regroup(wl.b, [g])
        pn, vu = wl.pn[:, idx], wl.vu[:, idx]
        want = _rows(wl.r, idx)
        same = _chain(wl.model, bg, pn, vu)          # re-bound after the batch
        new = _chain(fresh, bg, pn, vu)
        ref = restate.sample_diffusion(wl.sd, wl.cfg, *(bg[k] for k in ARGS), pn, vu, num_steps=wl.S)
        ref = {k: (torch.stack(ref[k]) if isinstance(ref[k], list) else ref[k]) for k in TRAJ}
        e_pos = _max_abs(same['pos_traj'], ref['pos_traj'])
        e_v0, e_vt = _max_abs(same['v0_traj'], ref['v0_traj']), _max_abs(same['vt_traj'], ref['vt_traj'])
        v_flips = int((same['v_traj'] != ref['v_traj']).sum())
        print('%s graph %3d (%d ligand atoms): differs from its batch rows in %s (same model) / %s (fresh model);  vs fp32 oracle: '
              'pos %.2e  v0 %.2e  vt %.2e  type flips %d  (limits pos %.0e + %.0e |pos|, logits %.0e)' %
              (wl.name, g, len(idx), _differing(same, want), _differing(new, want), e_pos, e_v0, e_vt, v_flips, POS_ATOL, POS_RTOL,
               LOGIT_ATOL))
        assert not _differing(same, want) and not _differing(new, want), g
        assert v_flips == 0 and torch.equal(same['v'], ref['v']), g
        torch.testing.assert_close(same['pos_traj'], ref['pos_traj'], rtol=POS_RTOL, atol=POS_ATOL)
        torch.testing.assert_close(same['pos'], ref['pos'], rtol=POS_RTOL, atol=POS_ATOL)
        torch.testing.assert_close(same['v0_traj'], ref['v0_traj'], rtol=0, atol=LOGIT_ATOL)
        torch.testing.assert_close(same['vt_traj'], ref['vt_traj'], rtol=0, atol=LOGIT_ATOL)
    del fresh


# ------------------------------------------------------------------------------------------------ 3. one anchor vs float64
def test_anchor_layers_vs_float64(workload):
    wl = workload
    g = _anchors(wl)[-1]
    bg, _ = _regroup(wl.b, [g])
    rows = layerwise.engine_layer_parity('%s graph %d' % (wl.name, g), wl.cfg, wl.sd, bg, 9, _model, DEV, tag='tc3')
    layerwise.check_layers(rows, 'tc3', wl.cfg['knn'])


def test_anchor_steps_vs_float64(workload):
    wl = workload
    g = _anchors(wl)[-1]
    bg, idx = _regroup(wl.b, [g])
    shift = bg['protein_pos'].mean(0, keepdim=True)              # the pocket at the origin: 'none' then sees the centred frame
    bg = dict(bg, protein_pos=bg['protein_pos'] - shift, init_ligand_pos=bg['init_ligand_pos'] - shift)
    label = '%s graph %d' % (wl.name, g)
    rows = stepwise.engine_steps_vs_float64(label, wl.model, wl.sd, wl.cfg, bg, wl.pn[:, idx], wl.vu[:, idx], range(wl.S), DEV)
    stepwise.check_steps(label, rows)


# ------------------------------------------------------------------------------------------------ 4. the seeded stream at cfg3 size
@pytest.mark.parametrize('workload', ['cfg3'], indirect=True)
def test_cfg3_seeded_stream_is_engine_tape(workload):
    wl = workload
    seed = 2 ** 33 + 2024
    n = wl.b['batch_ligand'].numel()
    args = tuple(wl.b[k].to(DEV) for k in ARGS)
    kw = dict(num_steps=wl.S, center_pos_mode='protein', stack_traj=True)
    dev = wl.model.sample_diffusion(*args, seed=seed, **kw)
    pn, vu = philox.engine_tape(seed, n, wl.S, K)
    tape = wl.model.sample_diffusion(*args, noise_tape=(pn, vu), **kw)
    T = wl.sd['betas'].shape[0]
    sigma = math.exp(0.5 * float(wl.sd['posterior_logvar'][T - 1]))
    offset = restate.center_pos(wl.b['protein_pos'], wl.b['init_ligand_pos'], wl.b['batch_protein'], wl.b['batch_ligand'])[2]
    offset = offset[wl.b['batch_ligand']]
    ulps, later = philox.stream_errors(dev['pos_traj'], tape['pos_traj'], pn[0], sigma, offset)
    flips = int((dev['v_traj'] != tape['v_traj']).sum())
    # the same without the centred frame in the scale: large where a coordinate nearly cancels its graph's offset
    ulps_uncentred = philox.stream_errors(dev['pos_traj'][:1], tape['pos_traj'][:1], pn[0], sigma)[0]
    print('cfg3 seeded stream, %d atoms x %d steps: type flips %d  step 0: %.2f ulp (%.2f ulp of |pos| + sigma |noise| alone)  '
          'later steps: %.2e rel  (limits %.0f ulp, %.0e)' %
          (n, wl.S, flips, ulps, ulps_uncentred, later, philox.STREAM_ULPS, philox.STREAM_LATER_REL))
    assert flips == 0
    assert torch.equal(dev['v0_traj'][0], tape['v0_traj'][0]) and torch.equal(dev['vt_traj'][0], tape['vt_traj'][0])
    assert ulps <= philox.STREAM_ULPS and later <= philox.STREAM_LATER_REL, (ulps, later)


# ------------------------------------------------------------------------------------------------ 5. logits that overflow exp unshifted
# The last Linear of every hq_func / xq_func is scaled by Q_SCALE, so that the float64 reference's attention logits reach
# |logit| >= LOGIT_MIN (exp(100) is 1e43, past fp32's 3.4e38: a softmax without the max shift gives inf / NaN).
Q_SCALE, LOGIT_MIN = 200.0, 100.0
# Largest per-row error of one layer against float64 allowed (h, x), about 3-4x the maxima measured on one NVIDIA H100 80GB HBM3 at a
# 400 W power limit: h 1.71e-4, x 1.42e-3 (k = 8, 32, 48, 64; largest |logit| 164 - 248 per layer).  The fp32 oracle's own error is up
# to 1.0e-5 in h and 5.6e-5 in x.  A softmax weight moves by its logit's absolute rounding, which grows with the logit: both are
# 10-20x the small-logit cases' (oracle.layerwise.LAYER_TOL), and the engine's q and k keep ~16 mantissa bits (bf16 splits).
OVERFLOW_TOL = (6e-4, 5e-3)


def _overflow_state_dict(cfg):
    sd = synth.make_state_dict(3, cfg, schedules=restate.make_schedules(cfg))
    n = 0
    for key in list(sd):
        if key.startswith('refine_net.base_block.') and ('.hq_func.net.3.' in key or '.xq_func.net.3.' in key):
            sd[key] = sd[key] * Q_SCALE
            n += 1
    assert n == 9 * 2 * 2
    return sd


@pytest.mark.parametrize('k', [8, 32, 48, 64])
def test_layer_parity_logits_past_exp_overflow(k, monkeypatch):
    """k = 32: folded key launch, softmax fused into its epilogue; k = 48: keys through HBM, aggregate_*_logits; k = 64: folded key
    launch, unfused aggregation; k = 8: the unfolded key launch."""
    cfg = {'knn': k}
    sd = _overflow_state_dict(cfg)
    b = synth.make_batch(61, 3, n_protein=110, ligand_sizes=[20, 1, 33])
    seen = []
    softmax = restate.scatter_softmax_rows

    def recording(src, index, n):
        if src.dtype == torch.float64:
            seen.append(float(src.abs().max()))
        return softmax(src, index, n)
    monkeypatch.setattr(restate, 'scatter_softmax_rows', recording)
    rows = layerwise.engine_layer_parity('q x%g knn=%d' % (Q_SCALE, k), cfg, sd, b, 3, _model, DEV, tag='tc3')
    print('q x%g knn=%d: largest |logit| of the float64 reference per layer %s; limits h %.0e x %.0e' %
          (Q_SCALE, k, ' '.join('%.0f' % max(seen[2 * i:2 * i + 2]) for i in range(len(rows))), *OVERFLOW_TOL))
    assert len(seen) == 2 * len(rows) and min(max(seen[2 * i:2 * i + 2]) for i in range(len(rows))) >= LOGIT_MIN, seen
    for r in rows:
        assert all(math.isfinite(v) for v in r), r
        assert r[1] <= OVERFLOW_TOL[0] and r[3] <= OVERFLOW_TOL[1], r
