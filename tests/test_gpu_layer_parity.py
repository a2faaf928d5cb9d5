"""Each attention layer of the engine against float64, and the k values and engine switches the other GPU tests do not reach
(run with -m gpu; `pytest -s` prints the per-layer error table).

The end-to-end tests compare 9 chained layers with the fp32 oracle at 1e-4, so they cannot tell how far one layer of the engine is
from exact arithmetic.  Here the network is cut after l = 1, 2, ... layers (the state dict without the later layers' keys loads
strictly into a ScorePosNet3D with num_layers = l): the engine's output of l layers is compared with `restate.att_layer` evaluated
in float64 (oracle/layerwise.py) on the engine's own output of l - 1 layers, on the oracle's graph.  So each comparison measures the
rounding of that one layer.  Per row,

    err[r] = |out[r] - ref64[r]|_inf / max(|ref64[r] - in[r]|_inf, 0.01 * median_r |ref64 - in|_inf)

for h over all rows and for x over the ligand rows; the fp32 oracle's error on the same inputs is printed beside it.

Also here: forwards and short chains against the oracle at k = 1, 7, 8, 9, 64 (a 64-row tile of the default edge kernel spans more
than the 8 destinations whose P rows it stages only for k <= 7, and exactly 8 at k = 8), the incremental k-NN at such k,
TDIFF_NO_FUSED_AGG and TDIFF_NO_SLOT_KEEP, and the stand-alone aggregation ops against float64."""
import math

import pytest
import torch

from oracle import layerwise, restate, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
MODE_ID = {'simt': 0, 'tc3v2': 2, 'tc6': 3, 'tc3': 5}
POS_RTOL, POS_ATOL, LOGIT_ATOL, H_RTOL, H_ATOL = 1e-4, 1e-5, 1e-3, 1e-4, 1e-4
# per-layer limits against float64 (LAYER_TOL, X_TOL_K1) and the measured maxima behind them: oracle/layerwise.py

EDGE_MLPS = ('.hk_func.', '.hv_func.', '.xk_func.', '.xv_func.')


def _signed_gain_state_dict(seed):
    """Synthetic weights with about half of every edge MLP's LayerNorm gains negated, one zero gain and one subnormal gain (the
    packer's sign and constant-feature branches, engine.cu pack_edge_mlp)."""
    sd = synth.make_state_dict(seed, schedules=restate.make_schedules())
    g = torch.Generator().manual_seed(seed + 1000)
    n = 0
    for key in list(sd):
        if key.endswith('.net.1.weight') and any(m in key for m in EDGE_MLPS):
            w, b = sd[key].clone(), sd[key[:-len('weight')] + 'bias'].clone()
            w[torch.rand(w.shape, generator=g) < 0.5] *= -1.0
            w[5], b[5] = 0.0, 0.3              # constant feature relu(0.3)
            w[77], b[77] = -1e-40, 0.2         # bias / |gain| overflows fp32: also a constant feature
            sd[key], sd[key[:-len('weight')] + 'bias'] = w, b
            n += 1
    assert n == 2 + 9 * 4                      # hk, hv of the (unused) init layer; hk, hv, xk, xv of the 9 layers
    return sd


def _weights(kind, cfg=None):
    if kind == 'signed':
        return _signed_gain_state_dict(1)
    return synth.make_state_dict(0, cfg, schedules=restate.make_schedules(cfg), gain=3.0 if kind == 'gain3' else 1.0)


def _batch(seed, parts):
    """A batch of graphs with different pocket sizes: parts = [(n_protein, [ligand sizes of its graphs]), ...]."""
    out, g0 = [], 0
    for i, (n_protein, sizes) in enumerate(parts):
        b = synth.make_batch(seed * 10 + i, len(sizes), n_protein=n_protein, ligand_sizes=sizes)
        b['batch_protein'] = b['batch_protein'] + g0
        b['batch_ligand'] = b['batch_ligand'] + g0
        g0 += len(sizes)
        out.append(b)
    return {k: torch.cat([b[k] for b in out]) for k in out[0]}


# ragged graphs with a single-atom ligand; the last graph (36 atoms) is smaller than k + 1 for k >= 48, the others larger
MIXED = [(110, [20, 1, 33]), (30, [6])]
THREE = [(110, [20, 1]), (30, [6])]                   # 3 graphs (time_emb runs with t = [999, 500, 3])
HYBRID = [(70, [12, 1, 9])]                            # >= k protein atoms per graph, k + n_ligand - 1 <= 64 slots


def _model(cfg, sd):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfg or {})
    m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


def _args(b, dev=DEV):
    return tuple(b[k].to(dev) for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))


# ------------------------------------------------------------------------------------------------ 1. layer by layer vs float64
def _layer_parity(label, cfg, sd, b, n_layers, mode='tc3', time_step=None):
    """Runs prefixes of 1..n_layers layers (oracle.layerwise.engine_layer_parity), each in edge-MLP mode `mode`; returns
    [(layer, h err max, h p99.9, x err max, x p99.9, fp32 oracle's 4 values)]."""
    def make(c, s):
        from targetdiff_b200 import _lib
        model = _model(c, s)
        assert _lib.load().tdiff_edge_mlp_mode(model.engine(DEV)) == MODE_ID[mode]
        return model
    return layerwise.engine_layer_parity(label, cfg, sd, b, n_layers, make, DEV, time_step=time_step, tag=mode)


_check_layers = layerwise.check_layers


@pytest.mark.parametrize('k', [1, 2, 7, 8, 9, 10, 16, 31, 32, 33, 48, 63, 64])
def test_layer_parity_k_sweep(k):
    cfg = {'knn': k}
    rows = _layer_parity('knn=%d' % k, cfg, _weights('synthetic', cfg), _batch(3, MIXED), 3)
    _check_layers(rows, 'tc3', k)


@pytest.mark.parametrize('k', [32, 48])
@pytest.mark.parametrize('weights', ['synthetic', 'gain3', 'signed'])
def test_layer_parity_all_layers(weights, k):
    cfg = {'knn': k}
    rows = _layer_parity('%s knn=%d' % (weights, k), cfg, _weights(weights), _batch(4, MIXED), 9)
    _check_layers(rows, 'tc3')


@pytest.mark.parametrize('k', [8, 32, 48])
@pytest.mark.parametrize('mode', ['simt', 'tc3v2', 'tc6', 'tc3'])
def test_layer_parity_every_mode(mode, k, monkeypatch):
    monkeypatch.setenv('TDIFF_EDGE_MLP', mode)
    cfg = {'knn': k}
    rows = _layer_parity('mode knn=%d' % k, cfg, _weights('synthetic', cfg), _batch(5, MIXED), 3, mode=mode)
    _check_layers(rows, mode)


OPTIONS = [{'ew_net_type': 'r'}, {'ew_net_type': 'm'}, {'ew_net_type': 'none'}, {'x2h_out_fc': True},
           {'time_emb_dim': 1, 'time_emb_mode': 'simple'},
           {'cutoff_mode': 'hybrid', 'knn': 8}, {'cutoff_mode': 'hybrid', 'knn': 21}, {'cutoff_mode': 'hybrid', 'knn': 32}]


@pytest.mark.parametrize('cfg', OPTIONS, ids=lambda c: ','.join('%s=%s' % kv for kv in c.items()))
def test_layer_parity_options(cfg):
    t = torch.tensor([999, 500, 3]) if cfg.get('time_emb_dim') else None
    parts = HYBRID if cfg.get('cutoff_mode') == 'hybrid' else THREE
    rows = _layer_parity(','.join('%s=%s' % kv for kv in cfg.items()), cfg, _weights('synthetic', cfg), _batch(6, parts), 3, time_step=t)
    _check_layers(rows, 'tc3')


def test_layer_parity_no_fused_aggregation(monkeypatch):
    """TDIFF_NO_FUSED_AGG=1 at k = 32: keys and values go through HBM and the stand-alone aggregation kernel."""
    monkeypatch.setenv('TDIFF_NO_FUSED_AGG', '1')
    rows = _layer_parity('no fused agg knn=32', {}, _weights('synthetic'), _batch(7, MIXED), 3)
    _check_layers(rows, 'tc3')


def _tiles_per_cta(n_dst, k, sm):
    tiles = -(-n_dst * k // 64)
    grid = min(tiles, sm)
    return [tiles // grid + (1 if i < tiles % grid else 0) for i in range(grid)]


def test_layer_parity_large_batch():
    """About 40 graphs of 90 + 40 atoms at k = 32: every CTA of both edge-kernel instantiations (NOUT = 128 over all destinations
    and over ligand destinations, NOUT = 16 over ligand destinations) runs >= 3 tiles, and some CTAs get an odd count, so one of
    their two consumer warpgroups has a tile less."""
    G, n_p, n_l, k = 40, 90, 40, 32
    sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    pad = 128 // math.gcd(k, 128)                       # each class of the destination list ends on a 128-row boundary (engine.cu)
    up = lambda n: -(-n // pad) * pad
    for n_dst in (up(G * n_p) + up(G * n_l), up(G * n_l)):
        per = _tiles_per_cta(n_dst, k, sm)
        assert min(per) >= 3 and any(c % 2 for c in per), (n_dst, sm, sorted(set(per)))
    rows = _layer_parity('large 40x(90+40) knn=32', {}, _weights('synthetic'), synth.make_batch(8, G, n_protein=n_p, n_ligand=n_l), 3)
    _check_layers(rows, 'tc3')


# ------------------------------------------------------------------------------------------------ 2. end to end where nothing else runs
def _forward_vs_oracle(cfg, sd, b):
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    want = restate.forward(sd, cfg, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    model = _model(cfg, sd)
    out = model(pp.to(DEV), b['protein_v'].to(DEV), b['batch_protein'].to(DEV), lp.to(DEV), b['init_ligand_v'].to(DEV), b['batch_ligand'].to(DEV))
    assert torch.equal(out['edge_index'].cpu(), tr['edge_index'])
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=H_RTOL, atol=H_ATOL)
    return model


@pytest.mark.parametrize('k,mode', [(1, 'tc3'), (7, 'tc3'), (9, 'tc3'), (64, 'tc3'), (8, 'simt'), (8, 'tc3v2'), (8, 'tc6'), (8, 'tc3')])
def test_forward_small_k_vs_oracle(k, mode, monkeypatch):
    monkeypatch.setenv('TDIFF_EDGE_MLP', mode)
    cfg = {'knn': k}
    model = _forward_vs_oracle(cfg, _weights('synthetic', cfg), _batch(9, MIXED))
    from targetdiff_b200 import _lib
    assert _lib.load().tdiff_edge_mlp_mode(model.engine(DEV)) == MODE_ID[mode]


@pytest.mark.parametrize('k', [7, 64])
def test_chain_small_and_large_k_vs_oracle(k):
    cfg = {'knn': k}
    sd = _weights('synthetic', cfg)
    b = _batch(10, MIXED)
    S = 6
    pn, vu = synth.make_tape(4, S, len(b['batch_ligand']))
    want = restate.sample_diffusion(sd, cfg, *_args(b, 'cpu'), pn, vu, num_steps=S)
    got = _model(cfg, sd).sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', noise_tape=(pn, vu))
    assert torch.equal(torch.stack(got['v_traj']), torch.stack(want['v_traj']))
    torch.testing.assert_close(torch.stack(got['pos_traj']), torch.stack(want['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(torch.stack(got['v0_traj']), torch.stack(want['v0_traj']), rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(torch.stack(got['vt_traj']), torch.stack(want['vt_traj']), rtol=0, atol=LOGIT_ATOL)


def _chain_pair(cfg, b, env, monkeypatch, S=8):
    """The same chain without and with the switch `env` set; both results."""
    pn, vu = synth.make_tape(3, S, int(b['init_ligand_pos'].shape[0]))
    sd = _weights('synthetic', cfg)
    res = []
    for on in (False, True):
        if on:
            monkeypatch.setenv(env, '1')
        model = _model(cfg, sd)
        out = model.sample_diffusion(*_args(b), num_steps=S, center_pos_mode='protein', noise_tape=(pn, vu))
        res.append((out, model(*_args(b))['edge_index']))
    return res


def _assert_same_chain(res):
    (a, ea), (c, ec) = res
    assert torch.equal(ea, ec)
    assert torch.equal(a['pos'], c['pos']) and torch.equal(a['v'], c['v'])
    assert torch.equal(torch.stack(a['pos_traj']), torch.stack(c['pos_traj']))
    assert torch.equal(torch.stack(a['v0_traj']), torch.stack(c['v0_traj']))


@pytest.mark.parametrize('k', [1, 9, 64])
def test_incremental_knn_equals_full_scan_small_and_large_k(k, monkeypatch):
    """Cached protein keys + per-step ligand merge (knn_update_kernel) against the full per-step scan (TDIFF_KNN_FULL=1), bit for
    bit, with a graph smaller than k + 1 atoms at k = 64."""
    _assert_same_chain(_chain_pair({'knn': k}, _batch(12, [(90, [20, 1, 33, 7]), (30, [6])]), 'TDIFF_KNN_FULL', monkeypatch))


@pytest.mark.parametrize('k', [32, 9])
def test_no_slot_keep_equals_default(k, monkeypatch):
    """TDIFF_NO_SLOT_KEEP=1 recomputes every edge's gate each step instead of keeping those of unchanged neighbour slots: the chain
    must be bit-identical."""
    _assert_same_chain(_chain_pair({'knn': k}, _batch(13, MIXED), 'TDIFF_NO_SLOT_KEEP', monkeypatch))


# ------------------------------------------------------------------------------------------------ 3. stand-alone aggregation vs float64
def _agg_problem(n, kk, seed):
    """Slot lists with ragged degrees (several rows of degree 0), logits of about +-60 on some destinations, and zero gates."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (n, kk), generator=g, dtype=torch.int32)
    deg = torch.randint(0, kk + 1, (n,), generator=g)
    deg[::7] = 0
    deg[1] = kk
    src[torch.arange(kk)[None, :] >= deg[:, None]] = -1
    k = torch.randn(n * kk, 128, generator=g)
    q = torch.randn(n, 128, generator=g)
    q[2::5] *= 60.0                                    # logits q.k / sqrt(8) of order +-60: exp overflows fp32 without the max shift
    e_w = torch.rand(n * kk, generator=g)
    e_w[torch.rand(n * kk, generator=g) < 0.2] = 0.0
    return src, k, q, e_w, g


def _softmax(q, k, dst, n):
    return restate.scatter_softmax_rows((q.view(-1, 16, 8)[dst] * k.view(-1, 16, 8) / math.sqrt(8)).sum(-1), dst, n)


def _max_err(got, want):
    return float((got.double() - want).abs().max())


@pytest.mark.parametrize('kk', [1, 7, 8, 9, 33, 48, 64])
def test_attn_aggregate_h_vs_float64(kk):
    from targetdiff_b200 import ops
    n = 90
    src, k, q, e_w, g = _agg_problem(n, kk, 20 + kk)
    v = torch.randn(n * kk, 128, generator=g)
    h = torch.randn(n, 128, generator=g)
    valid = src.view(-1) >= 0
    dst = torch.arange(n).repeat_interleave(kk)[valid]
    want = {}
    for dt in (torch.float64, torch.float32):
        with layerwise.default_dtype(dt):
            alpha = _softmax(q.to(dt), k[valid].to(dt), dst, n)
            m = alpha.unsqueeze(-1) * (v[valid].to(dt) * e_w[valid].to(dt)[:, None]).view(-1, 16, 8)
            want[dt] = restate.scatter_sum_rows(m, dst, n).view(n, 128) + h.to(dt)
    got = ops.attn_aggregate_h(k.to(DEV), v.to(DEV), e_w.to(DEV), src.to(DEV), q.to(DEV), h.to(DEV)).cpu()
    assert torch.isfinite(got).all()
    zero = (src < 0).all(1)
    assert torch.equal(got[zero], h[zero])                                   # degree 0: h unchanged
    e_gpu, e_32 = _max_err(got, want[torch.float64]), _max_err(want[torch.float32], want[torch.float64])
    print('aggregate_h kk=%d  max |err| %.2e  (fp32 oracle %.2e)' % (kk, e_gpu, e_32))
    assert e_gpu <= 4 * e_32 + 1e-6


@pytest.mark.parametrize('kk', [1, 7, 8, 9, 33, 48, 64])
def test_attn_aggregate_x_vs_float64(kk):
    from targetdiff_b200 import ops
    n = 70
    src, k, q, e_w, g = _agg_problem(n, kk, 40 + kk)
    self_loop = src == torch.arange(n, dtype=torch.int32)[:, None]
    src[self_loop] = (src[self_loop] + 1) % n
    v16 = torch.randn(n * kk, 16, generator=g)
    x = torch.randn(n, 3, generator=g) * 4
    mask = torch.rand(n, generator=g) < 0.6
    valid = src.view(-1) >= 0
    dst = torch.arange(n).repeat_interleave(kk)[valid]
    s = src.view(-1)[valid].long()
    want = {}
    for dt in (torch.float64, torch.float32):
        with layerwise.default_dtype(dt):
            xd = x.to(dt)
            alpha = _softmax(q.to(dt), k[valid].to(dt), dst, n)
            rel = xd[dst] - xd[s]
            m = alpha.unsqueeze(-1) * ((v16[valid].to(dt) * e_w[valid].to(dt)[:, None]).unsqueeze(-1) * rel.unsqueeze(1))
            want[dt] = xd + restate.scatter_sum_rows(m, dst, n).mean(1) * mask[:, None]
    got = ops.attn_aggregate_x(k.to(DEV), v16.to(DEV), e_w.to(DEV), src.to(DEV), q.to(DEV), x.to(DEV), mask.to(DEV)).cpu()
    assert torch.isfinite(got).all()
    still = (src < 0).all(1) | ~mask
    assert torch.equal(got[still], x[still])                                 # degree 0 or not a ligand row: x unchanged
    e_gpu, e_32 = _max_err(got, want[torch.float64]), _max_err(want[torch.float32], want[torch.float64])
    print('aggregate_x kk=%d  max |err| %.2e  (fp32 oracle %.2e)' % (kk, e_gpu, e_32))
    assert e_gpu <= 4 * e_32 + 1e-6
