"""The engine's device random stream restated on the CPU (TEST INFRASTRUCTURE, numpy).

With a `seed` and no noise tape, `step_epilogue_kernel` (targetdiff_b200/csrc/sampler.cu) draws its own noise from a
counter-based Philox4x32-10 (Salmon et al., SC'11; the Random123 constants).  Every draw is a pure function of
(seed, atom, step), so the stream can be rebuilt here and handed to the oracle as a noise tape:

    key           (seed & 0xffffffff, seed >> 32)
    positions     counter (a, s, 0, 0x70737400)       -> words x, y, z, w
                  u0 = 1 - u01(x), u1 = u01(y), u2 = 1 - u01(z), u3 = u01(w)          (u0, u2 in (0, 1])
                  n0 = sqrt(-2 ln u0) cos(2 pi u1), n1 = sqrt(-2 ln u0) sin(2 pi u1), n2 = sqrt(-2 ln u2) cos(2 pi u3)
    class c       word c % 4 of counter (a, s, 1 + c // 4, 0x76756e69), u = u01(word)
    u01(x)        (x >> 8) * 2^-24, in [0, 1 - 2^-24]

`a` is the ligand atom's index in the batch and `s` the number of steps already taken (0 for the first step, at t = T - 1).
The uniforms are exact in fp32; the normals are computed here in float64 and rounded once, so they are within a few fp32 ulps
of the kernel's logf / sqrtf / cospif / sinpif.
"""
import numpy as np
import torch

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
POS_DOMAIN, TYPE_DOMAIN = 0x70737400, 0x76756e69
_MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 over broadcastable uint32 arrays: counter words c0..c3, key words k0, k1 -> the four output words."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint32) for c in (c0, c1, c2, c3))
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = np.uint32(k0), np.uint32(k1)
    with np.errstate(over='ignore'):
        for _ in range(10):
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _MASK32).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _MASK32).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0, k1 = k0 + W0, k1 + W1
    return c0, c1, c2, c3


def u01(x):
    """The kernel's uniform: the top 24 bits of a word, times 2^-24 (exact in fp32), as float64."""
    return (np.asarray(x, dtype=np.uint32) >> np.uint32(8)).astype(np.float64) * 2.0 ** -24


def split_key(seed):
    seed = int(seed)
    if not 0 <= seed < 2 ** 64:
        raise ValueError('seed must fit in 64 bits')
    return seed & 0xFFFFFFFF, seed >> 32


def position_normals(seed, atoms, steps):
    """float64 normals [..., 3] for broadcastable integer arrays `atoms`, `steps` (before the kernel's fp32 rounding)."""
    k0, k1 = split_key(seed)
    x, y, z, w = philox4x32_10(atoms, steps, 0, POS_DOMAIN, k0, k1)
    u0, u1, u2, u3 = 1.0 - u01(x), u01(y), 1.0 - u01(z), u01(w)
    ra, rb = np.sqrt(-2.0 * np.log(u0)), np.sqrt(-2.0 * np.log(u2))
    return np.stack([ra * np.cos(2 * np.pi * u1), ra * np.sin(2 * np.pi * u1), rb * np.cos(2 * np.pi * u3)], -1)


def type_uniforms(seed, atoms, steps, K):
    """float64 uniforms [..., K] of the Gumbel-max draw, for broadcastable integer arrays `atoms`, `steps`."""
    k0, k1 = split_key(seed)
    lanes = []
    for blk in range((K + 3) // 4):
        lanes += philox4x32_10(atoms, steps, 1 + blk, TYPE_DOMAIN, k0, k1)
    return np.stack([u01(w) for w in lanes[:K]], -1)


def engine_tape(seed, n_lig, num_steps, K, pos_only=False):
    """The noise the engine draws for `seed` over a chain of `num_steps` steps on `n_lig` ligand atoms, as a noise tape
    (pos_noise [S, Nl, 3], v_uniform [S, Nl, K]) in fp32 torch tensors.  With `pos_only` the kernel draws no type uniforms; the
    tape then carries zeros there."""
    s = np.arange(num_steps, dtype=np.uint32)[:, None]
    a = np.arange(n_lig, dtype=np.uint32)[None, :]
    pn = position_normals(seed, a, s).astype(np.float32)
    if pos_only:
        vu = np.zeros((num_steps, n_lig, K), np.float32)
    else:
        vu = type_uniforms(seed, a, s, K).astype(np.float32)
    return torch.from_numpy(pn), torch.from_numpy(vu)


# A chain run with `seed=` against the same chain on `engine_tape(seed, ...)`, limits about 3-4x the largest value measured on one
# NVIDIA H100 80GB HBM3 at a 400 W power limit.  First step: |pos_seed - pos_tape| in fp32 ulps of (|pos| + sigma |noise|), measured
# at most 0.83.  Later steps: max |pos_seed - pos_tape| relative to the largest coordinate of the step (the network carries the first
# step's ulps forward), measured at most 7.5e-8.
STREAM_ULPS, STREAM_LATER_REL = 3.0, 3e-7


def stream_errors(pos_seed, pos_tape, pos_noise0, sigma0, offset=None):
    """(first-step error in ulps, later steps' relative error) of the position trajectories [S, Nl, 3] of a seeded chain and of the
    same chain on its engine_tape, whose first step has the noise `pos_noise0` [Nl, 3] and sigma `sigma0`.  With the centring
    `offset` [Nl, 3] (center_pos_mode='protein'), the step's position is a sum in the centred frame to which the offset is added, so
    the ulps are of |pos| + |pos - offset| + sigma |noise|: where pos nearly cancels the offset, the centred sum's rounding is
    larger than an ulp of pos."""
    eps32 = 2.0 ** -23
    p0 = pos_tape[0].double()
    d0 = (pos_seed[0].double() - p0).abs()
    scale = p0.abs() + sigma0 * pos_noise0.double().abs()
    if offset is not None:
        scale = scale + (p0 - offset.double()).abs()
    ulps = float((d0 / (eps32 * scale)).max())
    later = 0.0
    if pos_seed.shape[0] > 1:
        dl = (pos_seed[1:] - pos_tape[1:]).abs().flatten(1).amax(1)
        later = float((dl / pos_tape[1:].abs().flatten(1).amax(1)).max())
    return ulps, later
