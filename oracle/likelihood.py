"""Likelihood scoring restated on the CPU (TEST INFRASTRUCTURE): the per-atom variational-bound terms of tdiff_likelihood_terms, the
own-type prior, and the driver of scripts/likelihood_est_diffusion.py.

    atom_terms        the per-atom position and type terms at t (models/molopt_score_model.py:588-617), on oracle.restate's pieces,
                      in fp32 or float64.  In fp32 their per-graph means are restate.likelihood_estimation's, bit for bit.
    prior_atom_terms  kl_pos_prior / kl_v_prior (:411-438) per atom with the ligand's own types.  The reference's script passes graph
                      indices as types (:573); the type prior is class-symmetric (q(v_T | onehot(c)) is one vector up to a permutation),
                      so both agree in exact arithmetic and, in fp32, up to the order of the class sum.
    terms             the engine's [B] outputs: forward on x_t, then the means of atom_terms and prior_atom_terms.
    likelihood_tape   the engine's likelihood random stream (tdiff_likelihood_terms without a tape), restated on oracle.philox's
                      Philox4x32-10, Box-Muller and u01, with the counter layout below.
    data_likelihood_estimation   the reference driver (scripts/likelihood_est_diffusion.py:18-64) restated, graph-id prior included,
                      drawing randn(Nl, 3) then rand(Nl, K) per batch from torch's global CPU generator as the unmodified script does.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import fixed_atoms, philox, restate, start_ligand

# Likelihood scoring (tdiff_likelihood_terms, DESIGN.md section 1): graph g is noised at t_g with its own draw key k_g, and atom j of
# the graph (its index within the graph) draws on counters (j, k_g, t_g << 8, "lkps") for positions and (j, k_g, t_g << 8 | (1 + c/4),
# "lktv") for class c, with the sampler's key, Box-Muller and u01 (oracle/philox.py).  Nothing in a counter says where the graph sits in
# the batch.
LK_POS_DOMAIN, LK_TYPE_DOMAIN = 0x6c6b7073, 0x6c6b7476
# every Philox domain word of the engine: the sampler's, the fixed set's, the start's and the likelihood stream's
DOMAINS = {'sampler_pos': philox.POS_DOMAIN, 'sampler_type': philox.TYPE_DOMAIN,
           'fixed_pos': fixed_atoms.FIX_POS_DOMAIN, 'fixed_type': fixed_atoms.FIX_TYPE_DOMAIN,
           'start_pos': start_ligand.START_POS_DOMAIN, 'start_type': start_ligand.START_TYPE_DOMAIN,
           'likelihood_pos': LK_POS_DOMAIN, 'likelihood_type': LK_TYPE_DOMAIN}


def likelihood_counters(time_steps, keys, batch_ligand):
    """(j, k_g, t_g << 8) per ligand atom, as uint32 numpy arrays, for graph arrays `time_steps`, `keys` [B] and a sorted `batch_ligand`."""
    b = np.asarray(batch_ligand, dtype=np.int64)
    t = np.asarray(time_steps, dtype=np.int64)
    if t.size and (t.min() < 0 or t.max() >= 1 << 24):
        raise ValueError('likelihood stream: time steps must lie in 0..2^24 - 1')
    first = np.searchsorted(b, b, side='left')
    j = np.arange(len(b), dtype=np.int64) - first
    k = np.asarray(keys, dtype=np.int64)[b] & 0xFFFFFFFF
    return j.astype(np.uint32), k.astype(np.uint32), (t[b] << 8).astype(np.uint32)


def likelihood_normals(seed, time_steps, keys, batch_ligand):
    """float64 normals [Nl, 3] of the likelihood stream (before the kernel's fp32 rounding)."""
    k0, k1 = philox.split_key(seed)
    j, k, tw = likelihood_counters(time_steps, keys, batch_ligand)
    x, y, z, w = philox.philox4x32_10(j, k, tw, LK_POS_DOMAIN, k0, k1)
    u0, u1, u2, u3 = 1.0 - philox.u01(x), philox.u01(y), 1.0 - philox.u01(z), philox.u01(w)
    ra, rb = np.sqrt(-2.0 * np.log(u0)), np.sqrt(-2.0 * np.log(u2))
    return np.stack([ra * np.cos(2 * np.pi * u1), ra * np.sin(2 * np.pi * u1), rb * np.cos(2 * np.pi * u3)], -1)


def likelihood_uniforms(seed, time_steps, keys, batch_ligand, K):
    """float64 uniforms [Nl, K] of the likelihood stream's Gumbel-max draw (exact in fp32)."""
    k0, k1 = philox.split_key(seed)
    j, k, tw = likelihood_counters(time_steps, keys, batch_ligand)
    lanes = []
    for blk in range((K + 3) // 4):
        lanes += philox.philox4x32_10(j, k, tw | np.uint32(1 + blk), LK_TYPE_DOMAIN, k0, k1)
    return np.stack([philox.u01(w) for w in lanes[:K]], -1)


def likelihood_tape(seed, time_steps, keys, batch_ligand, K):
    """The noise tdiff_likelihood_terms draws for `seed`, as its tape (pos_noise [Nl, 3], v_uniform [Nl, K]) in fp32 torch tensors;
    `keys` None means k_g = g, as the engine's default."""
    b = np.asarray(batch_ligand, dtype=np.int64)
    t = np.asarray(time_steps, dtype=np.int64)
    if keys is None:
        keys = np.arange(len(t))
    pn = likelihood_normals(seed, t, keys, b).astype(np.float32).reshape(-1, 3)
    vu = likelihood_uniforms(seed, t, keys, b, K).astype(np.float32).reshape(-1, K)
    return torch.from_numpy(pn), torch.from_numpy(vu)


_TABLES = ('alphas_cumprod', 'posterior_mean_c0_coef', 'posterior_mean_ct_coef', 'posterior_logvar', 'log_alphas_v',
           'log_one_minus_alphas_v', 'log_alphas_cumprod_v', 'log_one_minus_alphas_cumprod_v')


def _tables(sd, dtype):
    return {k: sd[k].to(dtype) for k in _TABLES}


def _log_onehot(v, K, dtype):
    return torch.log(F.one_hot(v, K).to(dtype).clamp(min=1e-30))        # index_to_log_onehot, :124-130


def atom_terms(sd, x0, v0, xt, vt, pred_pos, pred_logits, t_atom, K, dtype=torch.float32, return_scale=False):
    """Per-atom (position term, type term) [Nl] at the per-atom times `t_atom` (< T) for the clean ligand (x0, v0), its noised state
    (xt, vt) and the network's outputs at it, centred frame.  Positions: normal_kl(q_pos_posterior(x0), logvar, q_pos_posterior(pred),
    logvar) / log 2 for t > 0, -log_normal(x0, q_pos_posterior(pred), logvar / 2) at t = 0 (compute_pos_Lt, :470-482).  Types:
    categorical_kl(log_true, log_model) for t > 0, -log_categorical(log_onehot(v0), log_model) at t = 0 (compute_v_Lt, :484-489)."""
    sd = _tables(sd, dtype)
    x0, xt, pred_pos, pred_logits = (a.to(dtype) for a in (x0, xt, pred_pos, pred_logits))
    t = torch.as_tensor(t_atom, dtype=torch.long)
    idx = torch.arange(len(t))
    mean_model = restate.q_pos_posterior(sd, pred_pos, xt, t, idx)
    log_v0, log_vt = _log_onehot(v0, K, dtype), _log_onehot(vt, K, dtype)
    log_recon = F.log_softmax(pred_logits, dim=-1)
    log_model = restate.q_v_posterior(sd, log_recon, log_vt, t, idx, K)
    log_true = restate.q_v_posterior(sd, log_v0, log_vt, t, idx, K)
    mask = (t == 0).to(dtype)
    logvar = restate.extract(sd['posterior_logvar'], t, idx)
    mean_true = restate.q_pos_posterior(sd, x0, xt, t, idx)
    kl_p = restate._normal_kl(mean_true, logvar, mean_model, logvar) / np.log(2.)
    ls = 0.5 * logvar
    nll_p = -((-((x0 - mean_model) ** 2) / (2 * torch.exp(ls * 2)) - ls - np.log(np.sqrt(2 * np.pi))).sum(-1))
    kl_c = (log_true.exp() * (log_true - log_model)).sum(1)
    nll_c = -(log_v0.exp() * log_model).sum(1)
    tp, tv = mask * nll_p + (1. - mask) * kl_p, mask * nll_c + (1. - mask) * kl_c
    if not return_scale:
        return tp, tv
    # the type term is a small sum of products with cancellation: its rounding is of the size of the magnitudes it is computed from,
    # the unnormalised log posteriors, their logsumexp and log_softmax(logits), weighted as the products are
    tm1 = torch.where(t - 1 < 0, torch.zeros_like(t), t - 1)
    one = restate.q_v_pred_one_timestep(sd, log_vt, t, idx, K)
    un_m = restate.q_v_pred(sd, log_recon, tm1, idx, K) + one
    un_t = restate.q_v_pred(sd, log_v0, tm1, idx, K) + one
    mag_m = un_m.abs() + torch.logsumexp(un_m, -1, keepdim=True).abs() + log_recon.abs()
    mag_t = un_t.abs() + torch.logsumexp(un_t, -1, keepdim=True).abs()
    s_kl = (log_true.exp() * (mag_t + mag_m)).sum(1)
    s_nll = (log_v0.exp() * mag_m).sum(1)
    return tp, tv, mask * s_nll + (1. - mask) * s_kl


def prior_atom_terms(sd, x0, v_types, K, dtype=torch.float32, return_scale=False):
    """Per-atom (kl_pos_prior, kl_v_prior) terms [Nl] at T - 1 (:411-438) with the types `v_types` ([Nl] class indices: the ligand's own
    types, or the graph ids the reference's script passes)."""
    T = sd['alphas_cumprod'].shape[0]
    sd = _tables(sd, dtype)
    x0 = x0.to(dtype)
    last = torch.full((x0.shape[0],), T - 1, dtype=torch.long)
    idx = torch.arange(x0.shape[0])
    a_pos = restate.extract(sd['alphas_cumprod'], last, idx)
    mean = a_pos.sqrt() * x0
    logvar = torch.log((1.0 - a_pos).sqrt())
    kl_pos = restate._normal_kl(torch.zeros_like(mean), torch.zeros_like(logvar), mean, logvar)
    log_qT = restate.q_v_pred(sd, _log_onehot(v_types, K, dtype), last, idx, K)
    log_half = -torch.log(K * torch.ones_like(log_qT))
    kl_v = (log_qT.exp() * (log_qT - log_half)).sum(1)
    if not return_scale:
        return kl_pos, kl_v
    return kl_pos, kl_v, (log_qT.exp() * (log_qT.abs() + log_half.abs())).sum(1)


def terms(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step, pos_noise, v_uniform,
          return_atoms=False):
    """tdiff_likelihood_terms restated in fp32 on a tape: dict of kl_pos, kl_v, prior_pos, prior_v [B] (and, with `return_atoms`,
    atom_kl_pos, atom_kl_v [Nl], xt [Nl,3] centred, vt [Nl]).  Lab-frame inputs, centred on the protein."""
    K = sd['v_inference.2.weight'].shape[0]
    B = int(batch_protein.max()) + 1
    time_step = torch.as_tensor(time_step, dtype=torch.long)
    protein_pos, x0, _ = restate.center_pos(protein_pos, ligand_pos, batch_protein, batch_ligand, 'protein')
    a_pos = sd['alphas_cumprod'].index_select(0, time_step)[batch_ligand].unsqueeze(-1)            # :578-583
    xt = a_pos.sqrt() * x0 + (1.0 - a_pos).sqrt() * pos_noise
    vt = restate.log_sample_categorical_from_uniform(restate.q_v_pred(sd, restate.index_to_log_onehot(ligand_v, K), time_step,
                                                                      batch_ligand, K), v_uniform)
    out = restate.forward(sd, cfg, protein_pos, protein_v, batch_protein, xt, vt, batch_ligand, time_step=time_step)
    tp, tv = atom_terms(sd, x0, ligand_v, xt, vt, out['pred_ligand_pos'], out['pred_ligand_v'], time_step[batch_ligand], K)
    pp, pv = prior_atom_terms(sd, x0, ligand_v, K)
    mean = lambda v: restate._scatter_mean_rows(v, batch_ligand, B)
    r = {'kl_pos': mean(tp), 'kl_v': mean(tv), 'prior_pos': mean(pp), 'prior_v': mean(pv)}
    if return_atoms:
        r.update(atom_kl_pos=tp, atom_kl_v=tv, xt=xt, vt=vt)
    return r


def _clones(data, n):
    """Batch.from_data_list of n clones of `data` (protein_pos, protein_atom_feature, ligand_pos, ligand_atom_feature_full)."""
    n_p, n_l = data['protein_pos'].shape[0], data['ligand_pos'].shape[0]
    return (data['protein_pos'].repeat(n, 1), data['protein_atom_feature'].float().repeat(n, 1),
            torch.repeat_interleave(torch.arange(n), n_p), data['ligand_pos'].repeat(n, 1),
            data['ligand_atom_feature_full'].repeat(n), torch.repeat_interleave(torch.arange(n), n_l))


def data_likelihood_estimation(sd, cfg, data, time_steps, batch_size=1):
    """scripts/likelihood_est_diffusion.py:18-64 on CPU: per batch of up to `batch_size` timesteps, the noise drawn from torch's global
    CPU generator as the script's `normal_()` then `rand_like` (randn(Nl, 3), rand(Nl, K)); then the graph-id prior of one clone.
    Returns the script's 4-tuple (all_kl_pos, all_kl_v [n_t + 1], sum_kl_pos, sum_kl_v)."""
    K = sd['v_inference.2.weight'].shape[0]
    T = sd['betas'].shape[0]
    time_steps = torch.as_tensor(time_steps, dtype=torch.long)
    n_t = len(time_steps)
    num_batch = int(np.ceil(n_t / batch_size))
    kp, kv = [], []
    cur = 0
    for i in range(num_batch):
        n = batch_size if i < num_batch - 1 else n_t - batch_size * (num_batch - 1)
        pp, pf, bp, lp, lv, bl = _clones(data, n)
        pn = torch.randn(len(bl), 3)
        vu = torch.rand(len(bl), K)
        a, b = restate.likelihood_estimation(sd, cfg, pp, pf, bp, lp, lv, bl, time_steps[cur:cur + n], pos_noise=pn, v_uniform=vu)
        kp.append(a)
        kv.append(b)
        cur += n
    pp, pf, bp, lp, lv, bl = _clones(data, 1)
    prior_p, prior_v = restate.likelihood_estimation(sd, cfg, pp, pf, bp, lp, lv, bl, torch.tensor([T]))
    kp, kv = torch.cat(kp), torch.cat(kv)
    sum_p, sum_v = T * torch.mean(kp), T * torch.mean(kv)
    kp, kv = torch.cat([kp, prior_p]), torch.cat([kv, prior_v])
    sum_p += prior_p[0]
    sum_v += prior_v[0]
    return kp, kv, sum_p.item(), sum_v.item()


def nll_sums(kl_pos, kl_v, T):
    """The script's sums of one ligand's terms [n_t + 1] (the last entry the prior): T * mean over t + prior, each in fp32 torch."""
    kl_pos, kl_v = torch.as_tensor(kl_pos), torch.as_tensor(kl_v)
    sp, sv = T * torch.mean(kl_pos[:-1]), T * torch.mean(kl_v[:-1])
    sp += kl_pos[-1]
    sv += kl_v[-1]
    return sp.item(), sv.item()

