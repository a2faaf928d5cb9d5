"""One sampling step at any floating-point precision (TEST INFRASTRUCTURE, CPU only).

`restate.sample_diffusion` chains the network and the step update in fp32, so comparing the engine with it after a chain measures
everything at once.  `step` evaluates only the update after the network -- the loop body of `restate.sample_diffusion`
(reference models/molopt_score_model.py:663-693), from the same helpers -- on given network outputs and noise.  At fp32 it is that
loop body bit for bit; with `dtype=torch.float64` the same fp32 schedule tables are read in float64, so comparing the engine's
`step_epilogue_kernel` with it measures the rounding of the epilogue alone (the float64 counterpart of oracle/layerwise.py).
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
