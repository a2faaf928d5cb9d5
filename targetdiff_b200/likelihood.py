"""Likelihood scoring of ligands in a pocket: the variational bound of scripts/likelihood_est_diffusion.py, the unsupervised affinity
score of the TargetDiff paper (DESIGN.md section 1).

    likelihood_time_steps(T, n)      the n timesteps i * T // n (n = 10: the script's 0, 100, ..., 900 at T = 1000; n = T: every t)
    data_likelihood_estimation(...)  the script's driver with its signature and 4-tuple: batches of up to `batch_size` clones of `data`
                                     at successive timesteps through ScorePosNet3D.likelihood_estimation, then the prior of one clone,
                                     summed as T * mean + prior.  rng='device' draws on torch's generator of the device, as the script;
                                     rng='cpu' draws randn(Nl, 3) then rand(Nl, K) per batch from torch's global CPU generator, the
                                     numbers the unmodified script consumes on CPU after the same seeding.
    ligand_nll(...)                  many ligands in one pocket: every (ligand, t) pair is a graph of one engine batch
                                     (ScorePosNet3D.likelihood_terms), packed ligand-major into batches of up to `batch_size` graphs,
                                     keyed by the ligand's index.  A ligand's result is the same bits whatever the batch size and
                                     whatever else is scored with it.
"""
import numpy as np
import torch


def likelihood_time_steps(T, n=10):
    """[i * T // n for i in range(n)]: n evenly spaced timesteps from 0 (n = T gives every timestep, an exact sum over t)."""
    T, n = int(T), int(n)
    if not 1 <= n <= T:
        raise ValueError('the number of timesteps must lie in 1..T = %d, got %d' % (T, n))
    return [i * T // n for i in range(n)]


def _clones(data, n, device):
    """Batch.from_data_list of n clones of `data`, as the likelihood arrays on `device`."""
    ppos, pfeat = torch.as_tensor(data['protein_pos']).float(), torch.as_tensor(data['protein_atom_feature']).float()
    lpos, lv = torch.as_tensor(data['ligand_pos']).float(), torch.as_tensor(data['ligand_atom_feature_full']).long()
    n_p, n_l = ppos.shape[0], lpos.shape[0]
    out = (ppos.repeat(n, 1), pfeat.repeat(n, 1), torch.repeat_interleave(torch.arange(n), n_p), lpos.repeat(n, 1), lv.repeat(n),
           torch.repeat_interleave(torch.arange(n), n_l))
    return tuple(x.to(device) for x in out)


def data_likelihood_estimation(model, data, time_steps, batch_size=1, device='cuda:0', rng='device'):
    """scripts/likelihood_est_diffusion.py:18-64: (all_kl_pos [n_t + 1] CPU, all_kl_v [n_t + 1] CPU, sum_kl_pos, sum_kl_v); the last
    entries are the prior, computed as the script does (its graph ids as types, DESIGN.md section 1)."""
    if rng not in ('device', 'cpu'):
        raise ValueError("rng must be 'device' or 'cpu', got %r" % (rng,))
    T, K = model.num_timesteps, model.num_classes
    time_steps = torch.as_tensor(time_steps, dtype=torch.long)
    n_t = len(time_steps)
    num_batch = int(np.ceil(n_t / batch_size))
    all_kl_pos, all_kl_v = [], []
    cur = 0
    for i in range(num_batch):
        n = batch_size if i < num_batch - 1 else n_t - batch_size * (num_batch - 1)
        pp, pf, bp, lp, lv, bl = _clones(data, n, device)
        noise = None
        if rng == 'cpu':
            pn = torch.randn(len(bl), 3)
            noise = (pn, torch.rand(len(bl), K))
        kl_pos, kl_v = model.likelihood_estimation(pp, pf, bp, lp, lv, bl, time_steps[cur:cur + n].to(device), noise=noise)
        all_kl_pos.append(kl_pos)
        all_kl_v.append(kl_v)
        cur += n
    pp, pf, bp, lp, lv, bl = _clones(data, 1, device)
    kl_pos_prior, kl_v_prior = model.likelihood_estimation(pp, pf, bp, lp, lv, bl, torch.tensor([T], device=device))
    all_kl_pos, all_kl_v = torch.cat(all_kl_pos), torch.cat(all_kl_v)
    sum_kl_pos, sum_kl_v = T * torch.mean(all_kl_pos), T * torch.mean(all_kl_v)
    all_kl_pos, all_kl_v = torch.cat([all_kl_pos, kl_pos_prior]), torch.cat([all_kl_v, kl_v_prior])
    sum_kl_pos += kl_pos_prior[0]
    sum_kl_v += kl_v_prior[0]
    return all_kl_pos.cpu(), all_kl_v.cpu(), sum_kl_pos.item(), sum_kl_v.item()


def _ligand_arrays(ligands):
    out = []
    for i, (pos, v) in enumerate(ligands):
        pos = torch.as_tensor(np.asarray(pos) if not torch.is_tensor(pos) else pos).float().cpu()
        v = torch.as_tensor(np.asarray(v) if not torch.is_tensor(v) else v).cpu()
        if v.is_floating_point() or pos.dim() != 2 or pos.shape[1] != 3 or v.dim() != 1 or v.shape[0] != pos.shape[0] or v.shape[0] < 1:
            raise ValueError('ligand %d: pos must be [n,3] and v [n] integer class indices (n >= 1), got %s and %s'
                             % (i, tuple(pos.shape), tuple(v.shape)))
        out.append((pos, v.long()))
    return out


def ligand_nll(model, data, ligands, time_steps=None, batch_size=640, device='cuda:0', seed=None, embedding=False):
    """Score every ligand (pos [n,3] lab frame, v [n] class indices) of `ligands` in the pocket `data` (protein_pos,
    protein_atom_feature).  Returns one dict per ligand: kl_pos, kl_v [n_t + 1] (the last entry the prior, with the ligand's own types),
    sum_kl_pos, sum_kl_v (T * mean over t + prior, as the script) and nll = sum_kl_pos + sum_kl_v; with `embedding`, also the script's
    pred_ligand_v, final_h and final_ligand_h of a fix_x forward on the clean ligand.  `seed` keys the likelihood stream (default:
    drawn from torch's CPU generator); graph (i, t) draws with key i."""
    T = model.num_timesteps
    if embedding and model.time_emb_dim > 0:
        raise ValueError('embedding=True needs a checkpoint without a time embedding: its fix_x forward has no time step '
                         '(the reference fetch_embedding cannot run either)')
    if model.model_mean_type != 'C0':
        raise ValueError('likelihood scoring needs model_mean_type C0, got %r' % (model.model_mean_type,))
    time_steps = likelihood_time_steps(T) if time_steps is None else [int(t) for t in time_steps]
    if not time_steps or any(not 0 <= t <= T - 1 for t in time_steps):
        raise ValueError('time_steps must be a non-empty list in 0..T-1 = %d' % (T - 1))
    batch_size = int(batch_size)
    if batch_size < 1:
        raise ValueError('batch_size must be >= 1')
    ligands = _ligand_arrays(ligands)
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    ppos = torch.as_tensor(data['protein_pos']).float()
    pfeat = torch.as_tensor(data['protein_atom_feature']).float()
    n_p, n_t = ppos.shape[0], len(time_steps)
    graphs = [(i, t) for i in range(len(ligands)) for t in time_steps]            # ligand-major
    res = {k: torch.empty(len(graphs)) for k in ('kl_pos', 'kl_v', 'prior_pos', 'prior_v')}
    for b0 in range(0, len(graphs), batch_size):
        part = graphs[b0:b0 + batch_size]
        n = len(part)
        sizes = torch.tensor([ligands[i][1].shape[0] for i, _ in part])
        lpos = torch.cat([ligands[i][0] for i, _ in part])
        lv = torch.cat([ligands[i][1] for i, _ in part])
        out = model.likelihood_terms(ppos.repeat(n, 1).to(device), pfeat.repeat(n, 1).to(device),
                                     torch.repeat_interleave(torch.arange(n), n_p).to(device), lpos.to(device), lv.to(device),
                                     torch.repeat_interleave(torch.arange(n), sizes).to(device), [t for _, t in part],
                                     keys=[i for i, _ in part], seed=seed)
        for k in res:
            res[k][b0:b0 + n] = out[k].cpu()
    results = []
    for i in range(len(ligands)):
        sl = slice(i * n_t, (i + 1) * n_t)
        kl_pos = torch.cat([res['kl_pos'][sl], res['prior_pos'][sl][:1]])
        kl_v = torch.cat([res['kl_v'][sl], res['prior_v'][sl][:1]])
        sum_kl_pos, sum_kl_v = T * torch.mean(kl_pos[:-1]), T * torch.mean(kl_v[:-1])
        sum_kl_pos += kl_pos[-1]
        sum_kl_v += kl_v[-1]
        results.append({'kl_pos': kl_pos, 'kl_v': kl_v, 'sum_kl_pos': sum_kl_pos.item(), 'sum_kl_v': sum_kl_v.item(),
                        'nll': sum_kl_pos.item() + sum_kl_v.item()})
    if embedding:
        for b0 in range(0, len(ligands), batch_size):
            part = list(range(b0, min(b0 + batch_size, len(ligands))))
            n = len(part)
            sizes = [ligands[i][1].shape[0] for i in part]
            pr = model.fetch_embedding(ppos.repeat(n, 1).to(device), pfeat.repeat(n, 1).to(device),
                                       torch.repeat_interleave(torch.arange(n), n_p).to(device),
                                       torch.cat([ligands[i][0] for i in part]).to(device), torch.cat([ligands[i][1] for i in part]).to(device),
                                       torch.repeat_interleave(torch.arange(n), torch.tensor(sizes)).to(device))
            pv, fh, flh = pr['pred_ligand_v'].cpu(), pr['final_h'].cpu(), pr['final_ligand_h'].cpu()
            a = node = 0
            for i, s in zip(part, sizes):
                results[i].update(pred_ligand_v=pv[a:a + s], final_h=fh[node:node + n_p + s], final_ligand_h=flh[a:a + s])
                a += s
                node += n_p + s
    return results
