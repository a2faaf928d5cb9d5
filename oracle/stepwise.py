"""One sampling step at any floating-point precision (TEST INFRASTRUCTURE, CPU only).

`restate.sample_diffusion` chains the network and the step update in fp32, so comparing the engine with it after a chain measures
everything at once.  `step` evaluates only the update after the network -- the loop body of `restate.sample_diffusion`
(reference models/molopt_score_model.py:663-693), from the same helpers -- on given network outputs and noise.  At fp32 it is that
loop body bit for bit; with `dtype=torch.float64` the same fp32 schedule tables are read in float64, so comparing the engine's
`step_epilogue_kernel` with it measures the rounding of the epilogue alone (the float64 counterpart of oracle/layerwise.py).
`engine_steps_vs_float64` runs that comparison on an engine chain; it is shared by tests/test_gpu_sampler.py and
tests/test_gpu_workload_shapes.py, with the limits `STEP_TOL`.
"""
import torch
import torch.nn.functional as F

from . import restate
from .layerwise import default_dtype
from .synth import DEFAULT_MODEL_CONFIG

TABLES = ('posterior_mean_c0_coef', 'posterior_mean_ct_coef', 'posterior_logvar', 'log_alphas_v', 'log_one_minus_alphas_v',
          'log_alphas_cumprod_v', 'log_one_minus_alphas_cumprod_v', 'sqrt_recip_alphas_cumprod', 'sqrt_recipm1_alphas_cumprod')


def step(sd, cfg, t, xt, vt, x0, logits, pos_noise, v_uniform, pos_only=False, dtype=torch.float32):
    """The step at time `t` (int) from the state (xt [Nl,3], vt [Nl] int64), given the network's outputs for that state
    (x0 [Nl,3]: pred_ligand_pos; logits [Nl,K]: pred_ligand_v) and the step's noise (pos_noise [Nl,3], v_uniform [Nl,K]).
    Centred frame, every atom at the same t.  Returns a dict of dtype tensors:
      pos     the next positions [Nl,3]
      scale   |c0 x0| + |ct xt| + |sigma noise| per coordinate [Nl,3], the size of the terms `pos` sums (x0 after the 'noise'
              mean type's conversion): position errors are measured relative to it
      v      the next atom types [Nl] (vt itself with pos_only)
      v0, vt  log_softmax(logits) and the log posterior [Nl,K] (None with pos_only)
      margin  the Gumbel score of the chosen class minus the runner-up's [Nl] (None with pos_only)."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    assert cfg['model_mean_type'] in ('C0', 'noise')
    sdd = {k: sd[k].to(dtype) for k in TABLES}
    n = xt.shape[0]
    K = logits.shape[1]
    tt = torch.full((1,), int(t), dtype=torch.long)
    batch = torch.zeros(n, dtype=torch.long)
    with default_dtype(dtype):
        xt, x0, nz = xt.to(dtype), x0.to(dtype), pos_noise.to(dtype)
        pos0 = x0
        if cfg['model_mean_type'] == 'noise':                                            # :663-666 with :419-422
            eps = x0 - xt
            pos0 = restate.extract(sdd['sqrt_recip_alphas_cumprod'], tt, batch) * xt - \
                restate.extract(sdd['sqrt_recipm1_alphas_cumprod'], tt, batch) * eps
        pos_mean = restate.q_pos_posterior(sdd, pos0, xt, tt, batch)                     # :673
        logvar = restate.extract(sdd['posterior_logvar'], tt, batch)                     # :674
        nonzero = (1 - (tt == 0).to(dtype))[batch].unsqueeze(-1)                         # :676
        pos = pos_mean + nonzero * (0.5 * logvar).exp() * nz                             # :677-679
        scale = (restate.extract(sdd['posterior_mean_c0_coef'], tt, batch) * pos0).abs() + \
            (restate.extract(sdd['posterior_mean_ct_coef'], tt, batch) * xt).abs() + (nonzero * (0.5 * logvar).exp() * nz).abs()
        out = {'pos': pos, 'scale': scale, 'v': vt.clone(), 'v0': None, 'vt': None, 'margin': None}
        if pos_only:                                                                     # :681
            return out
        log_v_recon = F.log_softmax(logits.to(dtype), dim=-1)                            # :682
        log_v = restate.index_to_log_onehot(vt, K)                                       # :683
        log_prob = restate.q_v_posterior(sdd, log_v_recon, log_v, tt, batch, K)          # :684
        u = v_uniform.to(dtype)
        out['v'] = restate.log_sample_categorical_from_uniform(log_prob, u)              # :685
        score = -torch.log(-torch.log(u + 1e-30) + 1e-30) + log_prob                     # :160-166
        top2 = score.topk(2, dim=-1).values
        out.update(v0=log_v_recon, vt=log_prob, margin=top2[:, 0] - top2[:, 1])
    return out


def errors(pos, v, v0, vt, ref, margin=1e-4):
    """A step's outputs (any dtype; v0 / vt None with pos_only) against the float64 `ref = step(..., dtype=torch.float64)`:
    {'pos': max |pos - ref| / ref scale, 'v0', 'vt': max absolute error, 'exempt': atoms whose Gumbel margin is <= `margin`,
     'v_diff': atoms with another type than ref's among the others}."""
    out = {'pos': float(((pos.double() - ref['pos']).abs() / ref['scale'].clamp(min=1e-30)).max())}
    if ref['v0'] is None:
        out.update(v0=0.0, vt=0.0, exempt=0, v_diff=int((v != ref['v']).sum()))
        return out
    close = ref['margin'] <= margin
    out.update(v0=float((v0.double() - ref['v0']).abs().max()), vt=float((vt.double() - ref['vt']).abs().max()),
               exempt=int(close.sum()), v_diff=int((v != ref['v'])[~close].sum()))
    return out


# Per-step errors against float64 allowed, about 3-4x the largest value measured on one NVIDIA H100 80GB HBM3 at a 400 W power limit
# (the kernels are deterministic), or of the fp32 oracle's own error where that is larger.  Measured maxima, engine / fp32 oracle:
# position (relative) 1.39e-7 / 1.65e-7, v0 (absolute) 4.1e-7 / 3.8e-7, vt (absolute) 1.94e-6 / 1.70e-6.  The position error is 0
# at t = 0 for both (sigma = 0 and x0 enters exactly).
STEP_TOL = {'pos': 6e-7, 'v0': 1.5e-6, 'vt': 6e-6}
# atoms whose float64 Gumbel margin (best score minus runner-up) is at most MARGIN are not compared; none occurred in any case
MARGIN, MAX_EXEMPT = 1e-4, 2


def engine_steps_vs_float64(label, model, sd, cfg, b, pn, vu, check, dev, pos_only=False):
    """A chain of the engine `model` on batch `b` (pockets at the origin) and noise tape (pn, vu), center_pos_mode='none', so that
    pos_traj[s] is the state itself.  For each step s in `check`, x0 and the logits come from a stand-alone forward on that step's
    input state, and `step` in float64 on the same inputs is the reference.  Returns [(s, t, engine errors, fp32 oracle errors)]."""
    T = sd['betas'].shape[0]
    B = int(b['batch_protein'].max()) + 1
    args = tuple(b[k].to(dev) for k in ('protein_pos', 'protein_v', 'batch_protein', 'init_ligand_pos', 'init_ligand_v', 'batch_ligand'))
    r = model.sample_diffusion(*args, num_steps=pn.shape[0], center_pos_mode='none', pos_only=pos_only, noise_tape=(pn, vu),
                               stack_traj=True)
    time_emb = (cfg or {}).get('time_emb_dim', 0) > 0
    rows = []
    for s in check:
        t = T - 1 - s
        xt = b['init_ligand_pos'] if s == 0 else r['pos_traj'][s - 1]
        vt = b['init_ligand_v'] if s == 0 else r['v_traj'][s - 1]
        kw = {'time_step': torch.full((B,), t, dtype=torch.long, device=dev)} if time_emb else {}
        out = model(args[0], args[1], args[2], xt.to(dev), vt.to(dev), args[5], **kw)
        x0, logits = out['pred_ligand_pos'].cpu(), out['pred_ligand_v'].cpu()
        a = (sd, cfg, t, xt, vt, x0, logits, pn[s], vu[s])
        ref = step(*a, pos_only=pos_only, dtype=torch.float64)
        f32 = step(*a, pos_only=pos_only)
        e = errors(r['pos_traj'][s], r['v_traj'][s], None if pos_only else r['v0_traj'][s],
                   None if pos_only else r['vt_traj'][s], ref, MARGIN)
        o = errors(f32['pos'], f32['v'], f32['v0'], f32['vt'], ref, MARGIN)
        rows.append((s, t, e, o))
        print('%-22s s=%4d t=%4d  pos %.2e  v0 %.2e  vt %.2e  exempt %d   fp32 oracle: pos %.2e  v0 %.2e  vt %.2e' %
              (label, s, t, e['pos'], e['v0'], e['vt'], e['exempt'], o['pos'], o['v0'], o['vt']))
    return rows


def check_steps(label, rows):
    for s, t, e, o in rows:
        assert e['v_diff'] == 0, (label, s, t, e)
        for k, lim in STEP_TOL.items():
            assert e[k] <= lim, (label, s, t, k, e[k], lim)
    assert sum(e['exempt'] for _, _, e, _ in rows) <= MAX_EXEMPT
