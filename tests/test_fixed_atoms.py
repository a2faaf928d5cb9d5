"""Fixed atoms (fragment-conditioned sampling, DESIGN.md section 1) on the CPU: the oracle's semantics against closed forms in
float64, the fixed atoms' Philox domains, and the driver's sizes, row layout and CPU generator order.  The engine side is
tests/test_gpu_fixed_atoms.py."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import fixed_atoms, philox, restate, synth

K = synth.LIGAND_NUM_CLASSES
T20 = {'num_diffusion_timesteps': 20}
EPS32 = 2.0 ** -23
MARGIN = 1e-4
Z_MAX, P_MIN = 5.0, 1e-6


def _setup(S=20, cfg=T20, seed=5, sizes=(6, 9)):
    sd = synth.make_state_dict(seed, cfg, schedules=restate.make_schedules(cfg))
    b = synth.make_batch(seed + 1, len(sizes), n_protein=30, ligand_sizes=list(sizes))
    n = len(b['batch_ligand'])
    pn, vu = synth.make_tape(seed + 2, S, n)
    g = torch.Generator().manual_seed(seed + 3)
    fixed_tape = (torch.randn(S + 1, n, 3, generator=g), torch.rand(S + 1, n, K, generator=g))
    mask = torch.zeros(n, dtype=torch.bool)
    mask[[0, 1, 2, sizes[0], sizes[0] + 4]] = True           # rows in both graphs, not all leading
    return sd, b, pn, vu, fixed_tape, mask


def _run(sd, cfg, b, pn, vu, S, fixed_mask=None, fixed_tape=None, **kw):
    args = (sd, cfg, b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'],
            pn, vu)
    if fixed_mask is None:
        return restate.sample_diffusion(*args, num_steps=S, **kw)
    return fixed_atoms.sample_diffusion(*args, fixed_mask, fixed_tape, num_steps=S, **kw)


def _same(r1, r2):
    for k in ('pos', 'v'):
        assert torch.equal(r1[k], r2[k]), k
    for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
        assert len(r1[k]) == len(r2[k]) and all(torch.equal(x, y) for x, y in zip(r1[k], r2[k])), k


# ------------------------------------------------------------------------------------------------ oracle semantics
def test_oracle_empty_mask_is_no_mask():
    """oracle.fixed_atoms.sample_diffusion with nothing fixed is restate.sample_diffusion (pinned against the reference) bit for bit,
    also with pos_only and the noise mean type."""
    for cfg, pos_only in ((T20, False), (T20, True), (dict(T20, model_mean_type='noise'), False)):
        S = 6
        sd, b, pn, vu, ft, mask = _setup(S, cfg)
        plain = _run(sd, cfg, b, pn, vu, S, pos_only=pos_only)
        _same(plain, _run(sd, cfg, b, pn, vu, S, fixed_mask=torch.zeros_like(mask), fixed_tape=ft, pos_only=pos_only))


def _closed_form(sd, x0c, off, v0, tm, eps, u):
    """float64 q(x_tm | x0) + offset and the Gumbel-max class with its margin (None where the draw is exact, tm < 0)."""
    if tm < 0:
        return x0c.double() + off.double(), v0, None
    ac = float(sd['alphas_cumprod'][tm])
    x = math.sqrt(ac) * x0c.double() + math.sqrt(1.0 - ac) * eps.double() + off.double()
    lca, l1 = float(sd['log_alphas_cumprod_v'][tm]), float(sd['log_one_minus_alphas_cumprod_v'][tm]) - math.log(K)
    log_x = torch.full((len(v0), K), math.log(1e-30), dtype=torch.float64)
    log_x[torch.arange(len(v0)), v0] = 0.0
    a, c = log_x + lca, torch.full_like(log_x, l1)
    m = torch.maximum(a, c)
    lp = m + torch.log(torch.exp(a - m) + torch.exp(c - m))
    sc = -torch.log(-torch.log(u.double() + 1e-30) + 1e-30) + lp
    top = sc.topk(2, dim=1).values
    return x, sc.argmax(1), top[:, 0] - top[:, 1]


@pytest.mark.parametrize('pos_only', [False, True])
def test_oracle_fixed_rows_are_the_forward_process(pos_only):
    """Fixed rows of pos_traj[s] = sqrt(ac[t-1]) x0 + sqrt(1 - ac[t-1]) eps[s+1] + offset in float64 within fp32 rounding; types
    the float64 Gumbel-max wherever its margin exceeds 1e-4; x0 and v0 themselves after t = 0."""
    S = 20
    sd, b, pn, vu, ft, mask = _setup(S)
    r = _run(sd, T20, b, pn, vu, S, fixed_mask=mask, fixed_tape=ft, pos_only=pos_only)
    _, x0c, off = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    x0c, off, v0 = x0c[mask], off[b['batch_ligand'][mask]], b['init_ligand_v'][mask]
    worst, exempt = 0.0, 0
    for s in range(S):
        tm = 20 - 1 - s - 1
        x, v, margin = _closed_form(sd, x0c, off, v0, tm, ft[0][s + 1][mask], ft[1][s + 1][mask])
        got = r['pos_traj'][s][mask].double()
        scale = x.abs() + x0c.double().abs() + ft[0][s + 1][mask].double().abs() + off.double().abs()
        worst = max(worst, float(((got - x).abs() / (EPS32 * scale)).max()))
        if pos_only:
            assert torch.equal(r['v_traj'][s][mask], v0)
        else:
            ok = margin > MARGIN if margin is not None else torch.ones(len(v), dtype=torch.bool)
            exempt += int((~ok).sum())
            assert torch.equal(r['v_traj'][s][mask][ok], v[ok]), s
    print('oracle fixed rows vs float64: %.2f ulp, %d exempt type draws' % (worst, exempt))
    assert worst <= 4.0 and exempt <= 1
    # after t = 0: the lab-frame target (one rounding of the centring and one of the offset) and its classes exactly
    final = r['pos'][mask].double()
    assert float(((final - b['init_ligand_pos'][mask].double()).abs() / (EPS32 * b['init_ligand_pos'][mask].double().abs() + 1e-30)).max()) <= 1.0 + 1e-9
    assert torch.equal(r['pos_traj'][-1][mask], r['pos'][mask])
    assert torch.equal(r['v'][mask], v0)


def test_oracle_v0_traj_is_the_networks():
    """v0_traj stays the network's output for every row, fixed ones included (the overwrite comes after it)."""
    S = 3
    sd, b, pn, vu, ft, mask = _setup(S)
    seen = []
    r = _run(sd, T20, b, pn, vu, S, fixed_mask=mask, fixed_tape=ft, step_callback=lambda s, t, preds, pos, v: seen.append(preds))
    for s in range(S):
        assert torch.equal(r['v0_traj'][s], torch.log_softmax(seen[s]['pred_ligand_v'], -1))


# ------------------------------------------------------------------------------------------------ Philox domains
def test_fixed_tape_layout():
    """fixed_tape is the kernel's layout: draw d of atom a from counters (a, d, 0, 'fxps') and (a, d, 1 + c // 4, 'fxtv'), the same
    key and transforms as the sampler's stream, S + 1 draws."""
    seed, S, n = 2 ** 40 + 99, 3, 7
    pn, vu = fixed_atoms.fixed_tape(seed, n, S, K)
    assert pn.shape == (S + 1, n, 3) and vu.shape == (S + 1, n, K) and pn.dtype == vu.dtype == torch.float32
    a, d = 5, 3
    k0, k1 = seed & 0xffffffff, seed >> 32
    x, y, z, w = (int(v) for v in philox.philox4x32_10(a, d, 0, 0x66787073, k0, k1))
    u = lambda word: (word >> 8) / 2.0 ** 24
    r0, r2 = math.sqrt(-2 * math.log(1 - u(x))), math.sqrt(-2 * math.log(1 - u(z)))
    want = [r0 * math.cos(2 * math.pi * u(y)), r0 * math.sin(2 * math.pi * u(y)), r2 * math.cos(2 * math.pi * u(w))]
    assert pn[d, a].tolist() == [float(np.float32(v)) for v in want]
    for c in range(K):
        assert float(vu[d, a, c]) == u(int(philox.philox4x32_10(a, d, 1 + c // 4, 0x66787476, k0, k1)[c % 4]))
    pn2, vu2 = fixed_atoms.fixed_tape(seed, n, S, K, pos_only=True)
    assert torch.equal(pn2, pn) and not vu2.any()


def test_fixed_domains_share_no_counter_with_the_sampler():
    """Every counter carries its domain in word 3, and the four domain words differ, so no counter of the fixed stream is one of the
    sampler's; the values at the same (atom, step) are unrelated."""
    doms = {philox.POS_DOMAIN, philox.TYPE_DOMAIN, fixed_atoms.FIX_POS_DOMAIN, fixed_atoms.FIX_TYPE_DOMAIN}
    assert len(doms) == 4
    seed, n, S = 12345, 512, 64
    pa, va = philox.engine_tape(seed, n, S, K)
    pb, vb = fixed_atoms.fixed_tape(seed, n, S, K)
    assert float((va == vb[:S]).double().mean()) < 1e-4
    for dd in range(3):
        assert abs(float(np.corrcoef(pa[..., dd].numpy().ravel(), pb[:S, ..., dd].numpy().ravel())[0, 1])) * math.sqrt(n * S) <= Z_MAX
    assert abs(float(np.corrcoef(va.numpy().ravel(), vb[:S].numpy().ravel())[0, 1])) * math.sqrt(va.numel()) <= Z_MAX


@pytest.mark.parametrize('seed', [12345, 0x0123456789ABCDEF])
def test_fixed_stream_distribution(seed):
    """The checks tests/test_oracle_sampler.py makes of the sampler's stream, on the fixed domains."""
    pn, vu = fixed_atoms.fixed_tape(seed, 4096, 255, K)
    pn, vu = pn.double().numpy(), vu.double().numpy()
    for d in range(3):
        x = pn[..., d].ravel()
        n = x.size
        assert abs(x.mean()) * math.sqrt(n) <= Z_MAX and abs(x.var() - 1.0) / math.sqrt(2.0 / n) <= Z_MAX, d
        assert stats.kstest(x, 'norm').pvalue >= P_MIN, d
    corr = lambda a, b: float(np.corrcoef(a.ravel(), b.ravel())[0, 1]) * math.sqrt(a.size)
    for i, j in ((0, 1), (0, 2), (1, 2)):
        assert abs(corr(pn[..., i], pn[..., j])) <= Z_MAX and abs(corr(pn[..., i] ** 2, pn[..., j] ** 2)) <= Z_MAX
    assert vu.min() >= 0.0 and vu.max() <= 1.0 - 2.0 ** -24
    for c in range(K):
        x = vu[..., c].ravel()
        assert stats.kstest(x, 'uniform').pvalue >= P_MIN, c
        assert stats.chisquare(np.bincount((x * 64).astype(np.int64), minlength=64)).pvalue >= P_MIN, c
    for c in range(K - 1):
        assert abs(corr(vu[..., c], vu[..., c + 1])) <= Z_MAX, c


# ------------------------------------------------------------------------------------------------ driver
class _Recorder:
    """Stands in for ScorePosNet3D in sample_diffusion_ligand: records what the driver hands to sample_diffusion."""
    num_classes, num_timesteps = K, 20

    def __init__(self):
        self.calls = []

    def sample_diffusion(self, **kw):
        self.calls.append(kw)
        n, S = len(kw['batch_ligand']), kw['num_steps']
        return {'pos': kw['init_ligand_pos'].clone(), 'v': kw['init_ligand_v'].clone(), 'pos_traj': torch.zeros(S, n, 3),
                'v_traj': torch.zeros(S, n, dtype=torch.long), 'v0_traj': torch.zeros(S, n, K), 'vt_traj': torch.zeros(S, n, K)}


def _pocket(n=40):
    from targetdiff_b200.data import ProteinLigandData
    b = synth.make_batch(9, 1, n_protein=n, ligand_sizes=[1])
    return ProteinLigandData(protein_pos=b['protein_pos'], protein_atom_feature=b['protein_v'])


def test_driver_sizes_rows_and_cpu_draw_order():
    from targetdiff_b200.sampling import sample_diffusion_ligand
    data = _pocket()
    frag = (torch.randn(3, 3) + 10.0, torch.tensor([1, 4, 7]))
    S, n_f = 4, 3
    model = _Recorder()
    torch.manual_seed(77)
    out = sample_diffusion_ligand(model, data, 6, batch_size=6, device='cpu', num_steps=S, sample_num_atoms='range', rng='cpu',
                                  fixed_ligand=frag)
    kw = model.calls[0]
    sizes = [max(n, n_f + 1) for n in range(1, 7)]                              # 'range' gives 1..6, raised to 4
    assert [len(p) for p in out[0]] == sizes
    assert torch.equal(torch.bincount(kw['batch_ligand']), torch.tensor(sizes))
    starts = np.cumsum([0] + sizes[:-1])
    rows = torch.from_numpy((starts[:, None] + np.arange(n_f)).reshape(-1))
    want_mask = torch.zeros(sum(sizes), dtype=torch.bool)
    want_mask[rows] = True
    assert torch.equal(kw['fixed_mask'], want_mask)
    assert torch.equal(kw['init_ligand_pos'][rows], frag[0].repeat(6, 1))
    assert torch.equal(kw['init_ligand_v'][rows], frag[1].repeat(6))
    # the CPU generator: init draws over every row, the interleaved per-step draws, then the fixed tape
    n = sum(sizes)
    torch.manual_seed(77)
    init_pos = torch.randn(n, 3)
    init_u = torch.rand(n, K)
    pn, vu = torch.empty(S, n, 3), torch.empty(S, n, K)
    for s in range(S):
        pn[s], vu[s] = torch.randn(n, 3), torch.rand(n, K)
    fpn, fvu = torch.randn(S + 1, n, 3), torch.rand(S + 1, n, K)
    assert torch.equal(kw['noise_tape'][0], pn) and torch.equal(kw['noise_tape'][1], vu)
    assert torch.equal(kw['fixed_noise_tape'][0], fpn) and torch.equal(kw['fixed_noise_tape'][1], fvu)
    free = ~want_mask
    center = data.protein_pos.float().sum(0, keepdim=True) / data.protein_pos.shape[0]
    assert torch.allclose(kw['init_ligand_pos'][free], (center + init_pos)[free], rtol=0, atol=1e-5)
    gumbel = -torch.log(-torch.log(init_u + 1e-30) + 1e-30)
    assert torch.equal(kw['init_ligand_v'][free], gumbel.argmax(-1)[free])
    # and the oracle's driver consumes the generator the same way
    seen = []
    real = fixed_atoms.sample_diffusion
    try:
        fixed_atoms.sample_diffusion = lambda *a, **k: seen.append(a) or real(*a, **k)
        sd = synth.make_state_dict(0, T20, schedules=restate.make_schedules(T20))
        torch.manual_seed(77)
        fixed_atoms.sample_diffusion_ligand(sd, T20, data.protein_pos, data.protein_atom_feature, 6, None, frag, batch_size=6,
                                            num_steps=S, sample_num_atoms='range')
    finally:
        fixed_atoms.sample_diffusion = real
    a = seen[0]
    assert torch.equal(a[10], want_mask)
    assert torch.equal(a[8], pn) and torch.equal(a[9], vu)
    assert torch.equal(a[11][0], fpn) and torch.equal(a[11][1], fvu)
    assert torch.equal(a[6], kw['init_ligand_v'])


def test_driver_without_fragment_draws_as_before():
    """No fragment: the same calls and draws as the driver without the feature (no fixed keywords at all)."""
    from targetdiff_b200.sampling import sample_diffusion_ligand
    model = _Recorder()
    torch.manual_seed(3)
    sample_diffusion_ligand(model, _pocket(), 3, batch_size=3, device='cpu', num_steps=2, sample_num_atoms='range', rng='cpu')
    assert 'fixed_mask' not in model.calls[0] and 'fixed_noise_tape' not in model.calls[0]
    assert [int(c) for c in torch.bincount(model.calls[0]['batch_ligand'])] == [1, 2, 3]


def test_driver_refusals():
    from targetdiff_b200.sampling import sample_diffusion_ligand
    data = _pocket()
    with pytest.raises(ValueError, match='pos_only'):
        sample_diffusion_ligand(_Recorder(), data, 2, device='cpu', num_steps=2, sample_num_atoms='range', pos_only=True,
                                fixed_ligand=(torch.zeros(2, 3), torch.tensor([0, 1])))
    with pytest.raises(ValueError, match='classes'):
        sample_diffusion_ligand(_Recorder(), data, 2, device='cpu', num_steps=2, sample_num_atoms='range',
                                fixed_ligand=(torch.zeros(2, 3), torch.tensor([0, K])))
    with pytest.raises(ValueError, match='fixed_ligand'):
        sample_diffusion_ligand(_Recorder(), data, 2, device='cpu', num_steps=2, sample_num_atoms='range',
                                fixed_ligand=(torch.zeros(2, 2), torch.tensor([0, 1])))


def test_cli_fragment_files(tmp_path):
    from targetdiff_b200.cli import load_fragment
    pos, v = np.arange(9, dtype=np.float32).reshape(3, 3), np.array([2, 0, 5])
    np.savez(tmp_path / 'f.npz', pos=pos, v=v)
    torch.save({'pos': torch.from_numpy(pos), 'v': torch.from_numpy(v)}, tmp_path / 'f.pt')
    for name in ('f.npz', 'f.pt'):
        p, c = load_fragment(str(tmp_path / name))
        assert p.dtype == torch.float32 and c.dtype == torch.int64
        assert torch.equal(p, torch.from_numpy(pos)) and torch.equal(c, torch.from_numpy(v))
    np.savez(tmp_path / 'bad.npz', pos=pos[:, :2], v=v)
    with pytest.raises(ValueError):
        load_fragment(str(tmp_path / 'bad.npz'))
    np.savez(tmp_path / 'float_v.npz', pos=pos, v=v.astype(np.float32))
    with pytest.raises(ValueError):
        load_fragment(str(tmp_path / 'float_v.npz'))
    with pytest.raises(ValueError):
        load_fragment(str(tmp_path / 'f.sdf'))
