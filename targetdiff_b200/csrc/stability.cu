// stability.cu -- bond-count stability screen of generated molecules on the device (SURVEY.md 8(f) n4).
//
// Replaces the O(n^2) Python double loop of the reference's utils/evaluation/analyze.py:106-143 (`check_stability`, called once per
// generated molecule by scripts/evaluate_diffusion.py:78-84) and its helper `get_bond_order` (:90-103): for every atom pair the
// distance in picometres is compared with the single / double / triple bond-length tables (+ margins 10 / 5 / 3 pm), the bond orders
// are summed per atom, and an atom is stable when 0 < bonds <= its allowed valence (== with `hs`).
// One warp per molecule; arithmetic in fp64 rounded op by op as numpy does on the float64 positions the sampler returns (fp32 values):
// difference, each square, ((a + b) + c), sqrt, * 100.  The squared distance is written with __dmul_rn / __dadd_rn, which nvcc never
// contracts: with plain operators it fuses two of the products into DFMAs, and pairs within an ulp of a threshold then get another
// bond order than the reference's (DESIGN.md section 2, stability screen).  Double sqrt and the product are correctly rounded.
#include "tdiff_common.cuh"

namespace {
// element order of the reference's tables: H C N O F P S Cl (analyze.py:6,10-41)
__constant__ short c_bonds1[8][8] = {{74, 109, 101, 96, 92, 144, 134, 127},   {109, 154, 147, 143, 135, 184, 182, 177},
                                     {101, 147, 145, 140, 136, 177, 168, 175}, {96, 143, 140, 148, 142, 163, 151, 164},
                                     {92, 135, 136, 142, 142, 156, 158, 166},  {144, 184, 177, 163, 156, 221, 210, 203},
                                     {134, 182, 168, 151, 158, 210, 204, 207}, {127, 177, 175, 164, 166, 203, 207, 199}};
__constant__ short c_bonds2[8][8] = {{-1, -1, -1, -1, -1, -1, -1, -1},   {-1, 134, 129, 120, -1, -1, 160, -1}, {-1, 129, 125, 121, -1, -1, -1, -1},
                                     {-1, 120, 121, 121, -1, 150, -1, -1}, {-1, -1, -1, -1, -1, -1, -1, -1},     {-1, -1, -1, 150, -1, -1, 186, -1},
                                     {-1, 160, -1, -1, -1, 186, -1, -1}, {-1, -1, -1, -1, -1, -1, -1, -1}};
__constant__ short c_bonds3[8][8] = {{-1, -1, -1, -1, -1, -1, -1, -1}, {-1, 120, 116, 113, -1, -1, -1, -1}, {-1, 116, 110, -1, -1, -1, -1, -1},
                                     {-1, 113, -1, -1, -1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1, -1, -1},   {-1, -1, -1, -1, -1, -1, -1, -1},
                                     {-1, -1, -1, -1, -1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1, -1, -1}};
__constant__ short c_allowed[8] = {1, 4, 3, 2, 1, 5, 4, 1};       // analyze.py:44

__device__ __forceinline__ int element_index(int z) {             // atom_decoder (analyze.py:6-7); -1: not in the table (KeyError there)
  switch (z) {
    case 1: return 0; case 6: return 1; case 7: return 2; case 8: return 3; case 9: return 4; case 15: return 5; case 16: return 6; case 17: return 7;
    default: return -1;
  }
}

__global__ void __launch_bounds__(256)
check_stability_kernel(const float* __restrict__ pos, const int* __restrict__ atomic_num, const int* __restrict__ mol_ptr, int n_mol, int hs,
                       int* __restrict__ nr_bonds_out, int* __restrict__ stable_atoms, unsigned char* __restrict__ mol_stable, int* __restrict__ err) {
  const int lane = threadIdx.x & 31;
  const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= n_mol) return;
  const int b = mol_ptr[m], n = mol_ptr[m + 1] - b;
  int n_stable = 0;
  for (int i = lane; i < n; i += 32) {
    const int ei = element_index(atomic_num[b + i]);
    if (ei < 0) { atomicExch(err, 1); continue; }
    const double xi = pos[3 * (b + i)], yi = pos[3 * (b + i) + 1], zi = pos[3 * (b + i) + 2];
    int bonds = 0;
    for (int j = 0; j < n; ++j) {
      if (j == i) continue;
      const int ej = element_index(atomic_num[b + j]);
      if (ej < 0) continue;
      // the reference always evaluates the pair with the smaller index first: p1 - p2 and bonds[atom1][atom2] of (min, max); the tables
      // are symmetric and (-d)^2 == d^2, so the order does not matter
      const double dx = xi - (double)pos[3 * (b + j)], dy = yi - (double)pos[3 * (b + j) + 1], dz = zi - (double)pos[3 * (b + j) + 2];
      const double dist = 100.0 * sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));  // analyze.py:91,119
      int order = 0;
      if (dist < (double)(c_bonds1[ei][ej] + 10)) {                                          // margin1
        order = 1;
        if (dist < (double)(c_bonds2[ei][ej] + 5)) {                                         // margin2
          order = 2;
          if (dist < (double)(c_bonds3[ei][ej] + 3)) order = 3;                              // margin3
        }
      }
      bonds += order;
    }
    if (nr_bonds_out) nr_bonds_out[b + i] = bonds;
    const int allowed = c_allowed[ei];
    n_stable += hs ? (allowed == bonds) : (allowed >= bonds && bonds > 0);                   // analyze.py:130-133
  }
  n_stable = __reduce_add_sync(0xffffffffu, n_stable);
  if (lane == 0) {
    stable_atoms[m] = n_stable;
    mol_stable[m] = (n_stable == n) ? 1 : 0;                                                 // analyze.py:138
  }
}
}  // namespace

void td_launch_check_stability(const float* pos, const int* atomic_num, const int* mol_ptr, int n_mol, int hs, int* nr_bonds, int* stable_atoms,
                               unsigned char* mol_stable, int* err, cudaStream_t st) {
  if (n_mol > 0) check_stability_kernel<<<(n_mol + 7) / 8, 256, 0, st>>>(pos, atomic_num, mol_ptr, n_mol, hs, nr_bonds, stable_atoms, mol_stable, err);
}
