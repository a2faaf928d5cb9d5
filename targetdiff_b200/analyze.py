"""Stability screen of generated molecules on the GPU (reference utils/evaluation/analyze.py:106-143 `check_stability`;
caller scripts/evaluate_diffusion.py:78-84).  `check_stability` keeps the reference's signature and return tuple for one molecule;
`check_stability_batch` screens a whole result set in one launch (one warp per molecule)."""
import ctypes

import numpy as np
import torch

from . import _lib


def check_stability_batch(positions, atom_types, hs=False, device='cuda:0'):
    """positions: list of [n_i,3] arrays (or one [sum n_i,3] tensor with `atom_types` a list of arrays); atom_types: atomic numbers.
    Every coordinate must be an fp32 value (the sampler's positions, fp32 widened to float64, are): the screen computes in float64
    on exactly those values, as the reference does, and refuses others with ValueError rather than rounding them.
    Returns (molecule_stable [M] bool, nr_stable_atoms [M] int, n_atoms [M] int, nr_bonds [sum n_i] int) as numpy arrays."""
    counts = [len(a) for a in atom_types]
    as64 = lambda p: np.asarray(p, dtype=np.float64).reshape(0, 3) if np.size(p) == 0 else np.asarray(p, dtype=np.float64)   # zero atoms
    pos64 = np.concatenate([as64(p) for p in positions]) if isinstance(positions, (list, tuple)) else np.asarray(positions, dtype=np.float64)
    pos = torch.from_numpy(pos64.astype(np.float32))
    if not np.array_equal(pos.numpy().astype(np.float64), pos64, equal_nan=True):
        # the kernel reads fp32 coordinates: rounding others would screen different atoms from the ones the reference would
        raise ValueError('positions must be fp32 values (as the sampler returns them, widened or not): %d coordinates are not'
                         % int((pos.numpy().astype(np.float64) != pos64).sum()))
    z = torch.as_tensor(np.concatenate([np.asarray(a).astype(np.int64) for a in atom_types])).to(torch.int32)
    if pos.shape[0] != sum(counts) or pos.dim() != 2 or pos.shape[1] != 3:
        raise ValueError('positions must be [n,3] per molecule')
    dev = torch.device(device)
    pos, z = pos.to(dev).contiguous(), z.to(dev).contiguous()
    M = len(counts)
    nr_bonds = torch.zeros(max(1, pos.shape[0]), dtype=torch.int32, device=dev)
    stable_atoms = torch.zeros(max(1, M), dtype=torch.int32, device=dev)
    mol_stable = torch.zeros(max(1, M), dtype=torch.uint8, device=dev)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    with torch.cuda.device(dev):
        _lib.check(_lib.load().tdiff_check_stability(P(pos), P(z), _lib.i32_array(counts), M, int(bool(hs)), P(nr_bonds), P(stable_atoms), P(mol_stable),
                                                     ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return (mol_stable[:M].cpu().numpy().astype(bool), stable_atoms[:M].cpu().numpy().astype(np.int64), np.asarray(counts, dtype=np.int64),
            nr_bonds[:pos.shape[0]].cpu().numpy().astype(np.int64))


def check_stability(positions, atom_type, debug=False, hs=False, return_nr_bonds=False, device='cuda:0'):
    """One molecule, the reference's signature: (molecule_stable, nr_stable_bonds, n_atoms[, nr_bonds])."""
    positions = np.asarray(positions)
    assert len(positions.shape) == 2 and positions.shape[1] == 3
    ms, ns, n, nb = check_stability_batch([positions], [np.asarray(atom_type)], hs=hs, device=device)
    if return_nr_bonds:
        return bool(ms[0]), int(ns[0]), int(n[0]), nb
    return bool(ms[0]), int(ns[0]), int(n[0])


def protein_contacts(ligand_pos, protein_pos, batch_ligand, batch_protein, radius):
    """Per molecule g: (number of ligand atoms of g with a protein atom of g closer than `radius`, the smallest ligand-protein
    distance within g, inf without pairs) as (int64 [B], float64 [B]) tensors on the CPU, B = the number of molecules.  Computed in
    torch in float64 on the CPU, for the clash-guidance tests and timing tool; it counts contacts, it is not a quality metric."""
    lp, pp = torch.as_tensor(ligand_pos).detach().cpu().double(), torch.as_tensor(protein_pos).detach().cpu().double()
    bl, bp = torch.as_tensor(batch_ligand).detach().cpu().long(), torch.as_tensor(batch_protein).detach().cpu().long()
    B = int(max(int(bl.max()) if bl.numel() else -1, int(bp.max()) if bp.numel() else -1)) + 1
    n_close = torch.zeros(B, dtype=torch.int64)
    d_min = torch.full((B,), float('inf'), dtype=torch.float64)
    for g in range(B):
        a, p = lp[bl == g], pp[bp == g]
        if len(a) == 0 or len(p) == 0:
            continue
        d = torch.cdist(a, p, compute_mode='donot_use_mm_for_euclid_dist').min(dim=1).values
        n_close[g] = int((d < radius).sum())
        d_min[g] = float(d.min())
    return n_close, d_min


def type_violations(v, allowed):
    """Atoms whose class is outside the allowed set.  v: class indices [n] (array or tensor, or a list of per-molecule arrays);
    allowed: class indices, a [K] bool mask, or a per-atom [n,K] bool mask.  Returns the count as an int (element constraints,
    DESIGN.md section 1)."""
    if isinstance(v, (list, tuple)):
        v = np.concatenate([np.asarray(x).reshape(-1) for x in v]) if len(v) else np.zeros(0, np.int64)
    v = torch.as_tensor(np.asarray(v)).long().reshape(-1)
    a = torch.as_tensor(np.asarray(allowed.cpu() if torch.is_tensor(allowed) else allowed))
    if a.dtype == torch.bool and a.dim() == 2:
        if a.shape[0] != len(v):
            raise ValueError('a per-atom mask needs one row per atom: %d rows, %d atoms' % (a.shape[0], len(v)))
        ok = a[torch.arange(len(v)), v]
    elif a.dtype == torch.bool:
        ok = a[v]
    else:
        ok = torch.isin(v, a.long().reshape(-1))
    return int((~ok).sum())


def ligand_components(pos, batch_ligand, radius):
    """Per molecule g: the number of connected components of its atoms when atoms closer than `radius` are bonded, as an int64 [B]
    tensor on the CPU (0 for a molecule without atoms), B = the number of molecules.  Computed in float64 on the CPU, for the
    connectivity-guidance tests and timing tool; a distance criterion, not a chemical bond perception."""
    p = torch.as_tensor(pos).detach().cpu().double()
    bl = torch.as_tensor(batch_ligand).detach().cpu().long()
    B = int(bl.max()) + 1 if bl.numel() else 0
    out = torch.zeros(B, dtype=torch.int64)
    for g in range(B):
        x = p[bl == g]
        n = len(x)
        if n == 0:
            continue
        adj = (torch.cdist(x, x, compute_mode='donot_use_mm_for_euclid_dist') < float(radius)).numpy()
        seen = np.zeros(n, dtype=bool)
        for r in range(n):
            if seen[r]:
                continue
            out[g] += 1
            seen[r] = True
            stack = [r]
            while stack:
                i = stack.pop()
                nxt = np.nonzero(adj[i] & ~seen)[0]
                seen[nxt] = True
                stack.extend(nxt.tolist())
    return out
