"""Connectivity guidance restated on the CPU (TEST INFRASTRUCTURE, torch-CPU in float64 for closed forms and float32 for the engine's
decisions and chains).

An extension beyond the reference (DESIGN.md section 1, "Connectivity guidance").  At every denoising step each graph's ligand x0
predictions y (centred frame, after clash guidance when that is on) are moved so that the molecule's separate pieces come closer:

1. Row i sits at q_i: the target x0_f of a held row (a fixed or kept atom), y_i otherwise.  Rows i, c are bonded when |q_i - q_c| < rho.
2. One connected component: every row keeps y exactly.
3. Each component C takes its closest outside pair (i in C, j not in C): the smallest d^2 = |q_i - q_j|^2, ties to the lowest (i, j) in
   within-graph indices; d = sqrt(d^2) >= rho > b.
4. A component with a held row stays.  Every other one moves rigidly: each of its rows gets y + f (q_j - q_i), f = (lambda w (d - b)) / d,
   w = 1 when j's component has a held row and 1/2 otherwise.  Every shift is computed from the unshifted predictions.

At float32 every operation is one rounded torch op in the engine's order, d^2 = (dx dx + dy dy) + dz dz with dx = q_j - q_i, so the
bond and closest-pair decisions are the engine's and the guided rows agree to the bit.  For a free component whose partner is free
the shift is -(lambda / 4) grad_t E_C(t) at t = 0, E_C = max(0, |q_i + t - q_j| - b)^2 with the pair held (`pair_energy`).

`guide` is the rule, `hook` a `guidance` hook for oracle.clash_guidance.sample_diffusion / sample_diffusion_ligand that runs after an
optional clash-guidance hook and captures the held mask and the centred targets.  The existing oracle modules are left as they are.
"""
import numpy as np
import torch

from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components


def _scalar(x, dtype):
    return torch.tensor(float(x), dtype=dtype)


def graph_decisions(q, radius, dtype=torch.float64):
    """One graph's decisions on its positions q [n,3]: (labels [n] numpy int, the component count, d2 [n,n] at `dtype`)."""
    q = q.to(dtype)
    dx = q[None, :, 0] - q[:, None, 0]
    dy = q[None, :, 1] - q[:, None, 1]
    dz = q[None, :, 2] - q[:, None, 2]
    d2 = (dx * dx + dy * dy) + dz * dz
    bonded = torch.sqrt(d2) < _scalar(radius, dtype)
    n_comp, labels = connected_components(csr_matrix(bonded.numpy()), directed=False)
    return labels, int(n_comp), d2


def closest_pair(labels, d2, c):
    """(i, j) of component label c: the smallest d2[i, j] over i in c, j outside it, ties to the lowest (i, j)."""
    inside = labels == c
    m = d2.clone()
    m[~torch.from_numpy(inside)] = float('inf')
    m[:, torch.from_numpy(inside)] = float('inf')
    flat = int(torch.argmin(m.reshape(-1)))       # torch.argmin returns the first minimum in row-major order: the lowest (i, j)
    n = d2.shape[0]
    return flat // n, flat % n


def guide(y, batch_ligand, radius, length, strength, held=None, targets=None, dtype=torch.float64, info=None):
    """The guided predictions [Nl,3] at `dtype` of y [Nl,3]; held [Nl] bool and targets [Nl,3] the held rows and their positions (None:
    no held row).  strength == 0: y itself.  `info`, a list, receives one dict per graph with its labels, component count and the
    closest pair of each moved component."""
    y = y.to(dtype)
    out = y.clone()
    if float(strength) == 0.0:
        return out
    lam, b = _scalar(strength, dtype), _scalar(length, dtype)
    half, one = _scalar(0.5, dtype), _scalar(1.0, dtype)
    hm = torch.zeros(len(y), dtype=torch.bool) if held is None else torch.as_tensor(held, dtype=torch.bool)
    q_all = y.clone()
    if bool(hm.any()):
        q_all[hm] = targets.to(dtype)[hm]
    for g in torch.unique(batch_ligand).tolist():
        rows = (batch_ligand == g).nonzero().reshape(-1)
        q, h = q_all[rows], hm[rows].numpy()
        labels, n_comp, d2 = graph_decisions(q, radius, dtype)
        rec = {'labels': labels, 'n_comp': n_comp, 'pairs': {}}
        if info is not None:
            info.append(rec)
        if n_comp == 1:
            continue
        comp_held = np.zeros(n_comp, dtype=bool)
        np.logical_or.at(comp_held, labels, h)
        for c in range(n_comp):
            if comp_held[c]:
                continue
            i, j = closest_pair(labels, d2, c)
            rec['pairs'][c] = (i, j)
            d = torch.sqrt(d2[i, j])
            w = one if comp_held[labels[j]] else half
            f = ((lam * w) * (d - b)) / d
            sel = rows[torch.from_numpy(labels == c)]
            out[sel] = y[sel] + f * (q[j] - q[i])
    return out


def pair_energy(qi, qj, length, t):
    """E_C(t) = max(0, |q_i + t - q_j| - b)^2 in float64: the term of component C, its closest pair (i, j) held, C translated by t."""
    d = torch.linalg.norm(qi.double() + t.double() - qj.double())
    return float(torch.clamp(d - float(length), min=0.0) ** 2)


def hook(radius, length, strength, held=None, targets=None, clash=None, dtype=torch.float32):
    """A `guidance` hook (y, protein_pos, batch_ligand, batch_protein) -> y_hat for oracle.clash_guidance's chains: `clash` (a hook of
    oracle.clash_guidance.hook, or None) first, then `guide` at `dtype` with the held rows `held` [Nl] at `targets` [Nl,3], the
    chain's centred x0 (its init_ligand_pos with center_pos_mode 'none')."""
    def fn(y, pp, bl, bp):
        if clash is not None:
            y = clash(y, pp, bl, bp)
        return guide(y, bl, radius, length, strength, held=held, targets=targets, dtype=dtype)
    return fn
