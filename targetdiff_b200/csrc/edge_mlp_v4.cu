// edge_mlp_v4.cu -- per-edge MLP, fourth generation (default): both Linear layers and every edge type's gaussian block on the Hopper
// tensor cores (wgmma), fp32-faithful through bf16 operand splitting.
//
// Math (reference models/uni_transformer.py:45-56,111-120, models/common.py:60-80 after the exact first-layer split, SURVEY App. B):
//   pre[e]  = P[dst, offA:+128] + P[src, offB:+128] + tab[type][20] + sum_j g_j(dist_e) * tab[type][j]
//   hid     = relu(LN(pre) * ln_g + ln_b)
//   out[e]  = hid . W2^T + b2
//
//   * rows are visited through a CLASS-SORTED destination list (protein destinations, padded to a tile multiple, then ligand
//     destinations): a tile holds destinations of one class, hence at most two edge types -- protein destination: P->P (3) or
//     L->P (1); ligand destination: P->L (2) or L->L (0).  The gaussian/type block of BOTH is one small MMA
//         Dpre[64 x 128] = G[64 x 64] . TabClass^T,   G row = (g_0..g_19, 1, 0..) in the 32-slot half of the row's own type;
//   * both MMAs run on one warpgroup (wgmma, operands in shared memory, fp32 accumulators in registers); it hands Dpre and D to the
//     CUDA-core roles as row-major fp32 tiles in shared memory, so those roles keep thread = row;
//   * LayerNorm statistics are exchanged through two slot sets (2 named barriers per tile).
//
// CTA = 16 warps (512 threads), one CTA per SM, persistent over tiles of 64 edge rows (one wgmma M):
//   warps  0-3   MMA warpgroup  Dpre and D wgmma, accumulator fragments -> shared memory
//   warps  4-7   epilogue       D -> +b2 -> logits / softmax weights / fused attention aggregation / plain rows
//   warps  8-15  row threads    warp 8+q+2*qq: rows 32q..32q+31, feature quarter qq; gathers P[src] / P[dst] straight from L2
// Shared memory (212 KB): W2 pieces 64 KB | class table pieces 32 KB | G pieces 16 KB | A pieces 32 KB | Dpre 33 KB | D 33 KB | exchange 2 KB.
// bf16 split: 2 pieces / 3 products (a1b1 + a1b2 + a2b1).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "tdiff_common.cuh"
#include "hopper_mma.cuh"

namespace v4 {

constexpr int kThreads = 16 * 32;
constexpr int kTile = 64;                  // rows per tile
constexpr int kMmaWarps = 4, kEpiWarp0 = 4, kEpiWarps = 4, kRowWarp0 = 8, kRowWarps = 8;
constexpr int kGAtom = kTile * 128;        // one SWIZZLE_128B K-block (64 bf16) of a 64-row operand
constexpr int kTabClassBytes = 2 * 128 * 128;   // one class table: 2 bf16 pieces of [128 x 64]
constexpr int kDRow = 132;                 // fp32 row stride of the Dpre / D tiles (conflict-free 16-byte thread-per-row reads)
// shared-memory map (bytes from the 1024-aligned base)
constexpr int oW = 0, oT = oW + 4 * 128 * 128, oG = oT + kTabClassBytes, oA = oG + 2 * kGAtom, oDp = oA + 4 * kGAtom,
              oD = oDp + kTile * kDRow * 4, oX = oD + kTile * kDRow * 4, oBar = oX + 2 * 4 * kTile * 4, kSmem = oBar + 16 * 8;
enum { B_G_FULL = 0, B_DPRE_FULL, B_A_FULL, B_A_EMPTY, B_D_FULL, B_D_EMPTY, B_LOAD, B_TAB };

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_LOOP:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra WAIT_DONE;\n\tbra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (true) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) break;
    __nanosleep(100);
  }
}
// TMA bulk copy (1-D): global -> shared, completion counted in bytes on an mbarrier
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst), "l"(gsrc), "r"(bytes),
               "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

__device__ __forceinline__ uint32_t cvt_bf16x2(float hi, float lo) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void sts64f(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts32f(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
__device__ __forceinline__ float lds32f(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}
// N consecutive fp32 of a Dpre / D row as raw bits
template <int N>
__device__ __forceinline__ void lds_row(uint32_t addr, uint32_t (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; i += 4) {
    const float4 v = lds128(addr + 4u * (uint32_t)i);
    r[i] = __float_as_uint(v.x); r[i + 1] = __float_as_uint(v.y); r[i + 2] = __float_as_uint(v.z); r[i + 3] = __float_as_uint(v.w);
  }
}
__device__ __forceinline__ void lds16(uint32_t addr, uint32_t (&r)[16]) { lds_row<16>(addr, r); }
__device__ __forceinline__ void lds32(uint32_t addr, uint32_t (&r)[32]) { lds_row<32>(addr, r); }
__device__ __forceinline__ void stg256(float* p, float a, float b, float c, float d, float e, float f, float g, float h) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p + 4), "f"(e), "f"(f), "f"(g), "f"(h) : "memory");
}
// fp32 pairs, each lane of the pair rounded on its own (the order of operations is the kernel's, not the compiler's)
typedef float2 f2;
__device__ __forceinline__ f2 pk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void upk2(f2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// accumulator fragment of one m64nNk16 warpgroup MMA -> row-major fp32 tile (row stride kDRow)
template <int N>
__device__ __forceinline__ void store_frag(uint32_t tile, const float (&d)[N / 2], int wq, int lane) {
  const uint32_t r0 = (uint32_t)(16 * wq + (lane >> 2));
#pragma unroll
  for (int i = 0; i < N / 8; ++i) {
    const uint32_t c = (uint32_t)(8 * i + 2 * (lane & 3));
    sts64f(tile + 4u * (r0 * kDRow + c), d[4 * i], d[4 * i + 1]);
    sts64f(tile + 4u * ((r0 + 8u) * kDRow + c), d[4 * i + 2], d[4 * i + 3]);
  }
}

// LayerNorm affine parameters and the output bias travel as a kernel argument (constant bank, read with 128-bit loads)
struct LnParams { float4 g4[32]; float4 b4[32]; float b2[128]; float mu[20]; };
// Fused attention in the epilogues (k == 32: the 32 rows of an epilogue warp are exactly the edges of one destination), reference
// models/uni_transformer.py:73-83:  key launch writes softmax_e(q.k/sqrt 8) * e_w, value launch does h[dst] += sum_e w * v.
struct AggArgs {
  const float* logits;   // [rows,16] written by the key launch; NULL = plain value output
  const float* e_w;      // [N*k]
  float* h;              // [N,128] node features, updated in place (a destination's row is touched by one warp only)
  int key_softmax;       // key launch (k == 32): write softmax weights * e_w instead of raw logits
};

// Reduce N (8 or 16) per-lane values over the 32 lanes of a warp with a transposing butterfly: N - 1 + log2(32 / N) shuffles instead
// of 5 N.  On return lane l holds the total (sum or max) of element (l & (N - 1)).
template <int N, bool MAX>
__device__ __forceinline__ float warp_transpose_reduce(float (&t)[N], int lane) {
  auto op = [](float a, float b) { return MAX ? fmaxf(a, b) : a + b; };
#pragma unroll
  for (int h = N / 2; h >= 1; h >>= 1) {
    const bool up = lane & h;
#pragma unroll
    for (int i = 0; i < h; ++i) {
      const float send = up ? t[i] : t[i + h];
      const float keep = up ? t[i + h] : t[i];
      t[i] = op(keep, __shfl_xor_sync(0xffffffffu, send, h));
    }
  }
  float r = t[0];
#pragma unroll
  for (int m = N; m < 32; m <<= 1) r = op(r, __shfl_xor_sync(0xffffffffu, r, m));
  return r;
}
// two fp32 values -> packed bf16 high pieces and packed bf16 residuals (the residual of the first piece is exact in fp32)
__device__ __forceinline__ void split2(float y0, float y1, uint32_t& hi, uint32_t& lo) {
  hi = cvt_bf16x2(y1, y0);
  float r0, r1;
  upk2(sub2(pk2(y0, y1), pk2(__uint_as_float(hi << 16), __uint_as_float(hi & 0xffff0000u))), r0, r1);
  lo = cvt_bf16x2(r1, r0);
}

}  // namespace v4

using namespace v4;

// NOUT = 128: key / value MLPs (hk, hv, xk);  NOUT = 16: the per-head scalar value MLP of h2x (xv).
// Rows: idx = a * k + j over the destination list `row_nodes` (a < n_dst; entries < 0 are padding), edge slot e = row_nodes[a] * k + j.
// Tiles below `split` destinations are protein-destination tiles (class table 0), the others ligand-destination tiles (table 1).
template <int NOUT>
__global__ void __launch_bounds__(kThreads, 1)
edge_mlp_v4_kernel(const float* __restrict__ P, int zero_row, const int* __restrict__ src, const unsigned char* __restrict__ etype,
                   const float* __restrict__ dist_arr, const int* __restrict__ row_nodes, long long n_dst, long long split_dst,
                   const int* __restrict__ d_counts, int k, int offA, int offB, const unsigned char* __restrict__ w2_image,
                   const unsigned char* __restrict__ tab_image, float coeff, const float* __restrict__ qnode, float* __restrict__ out, int out_by_slot, AggArgs agg, const __grid_constant__ LnParams lp) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const uint32_t sbase = smem_u32(smem_raw);
  const uint32_t sW = sbase + oW, sG = sbase + oG, sT = sbase + oT, sA = sbase + oA, sDp = sbase + oDp, sD = sbase + oD, sX = sbase + oX,
                 sBar = sbase + oBar;
  // the warp index is broadcast from lane 0 so that the compiler knows it is warp-uniform (role branches are uniform branches)
  const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  auto bar = [&](int i) { return sBar + 8u * (uint32_t)i; };
  // row -> (destination slot, neighbour slot): k is a power of two for every shipped configuration but 48
  const int kshift = (k & (k - 1)) == 0 ? __ffs(k) - 1 : -1;
  auto row_dst = [&](long long idx, int& j) -> unsigned {
    const unsigned a = kshift >= 0 ? (unsigned)idx >> kshift : (unsigned)idx / (unsigned)k;
    j = (int)((unsigned)idx - a * (unsigned)k);
    return a;
  };

  if ((sbase & 1023u) != 0) __trap();            // SWIZZLE_128B atoms need a 1024-byte aligned window
  if (d_counts) { n_dst = d_counts[0]; split_dst = d_counts[1]; }      // destination subset compacted on the device
  const long long n_rows = n_dst * k, split_rows = split_dst * k;      // both multiples of 128 by construction of the lists
  const long long n_tiles = (n_rows + kTile - 1) / kTile;
  const long long my_tiles = (n_tiles > blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  auto tile_class = [&](long long t) -> int { return ((long long)(blockIdx.x + t * (long long)gridDim.x) * kTile >= split_rows) ? 1 : 0; };

  // ---- one-time setup: weight image and the first tile's class table -> smem (TMA bulk copies), barriers
  constexpr int kWAtom = NOUT * 128;            // one K-half of a weight piece: NOUT rows x 128 B
  constexpr int kWPiece = 2 * kWAtom;
  if (tid == 0) {
    mbar_init(bar(B_LOAD), 1);
    mbar_init(bar(B_TAB), 1);
    mbar_init(bar(B_G_FULL), kRowWarps);
    mbar_init(bar(B_DPRE_FULL), kMmaWarps);
    mbar_init(bar(B_A_FULL), kRowWarps);
    mbar_init(bar(B_A_EMPTY), kMmaWarps);
    mbar_init(bar(B_D_FULL), kMmaWarps);
    mbar_init(bar(B_D_EMPTY), kEpiWarps);
    fence_barrier_init();
    mbar_expect_tx(bar(B_LOAD), 2u * kWPiece + (uint32_t)kTabClassBytes);
    bulk_g2s(sW, w2_image, 2u * kWPiece, bar(B_LOAD));
    bulk_g2s(sT, tab_image + (size_t)tile_class(0) * kTabClassBytes, (uint32_t)kTabClassBytes, bar(B_LOAD));
  }
  __syncthreads();

  if (warp >= kRowWarp0) {
    // ================================================================= row threads (thread = edge row x 32 features)
    const int rwp = warp - kRowWarp0, q = rwp & 1, qq = rwp >> 1;
    const int r = 32 * q + lane;                    // row of the tile
    float mu[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) mu[i] = lp.mu[5 * qq + i];
    const float coeff2 = coeff * 1.4426950408889634f;
    const uint32_t g_row = sG + (uint32_t)r * 128u;
    const uint32_t dp_row = sDp + 4u * ((uint32_t)r * kDRow + 32u * (uint32_t)qq);
    const uint32_t a_row = sA + (uint32_t)(qq >> 1) * kGAtom + (uint32_t)r * 128u;     // K-half qq / 2 of piece 0; piece 1 at + 2 kGAtom
    const uint32_t xslot = sX + (uint32_t)r * 4u;          // exchange slots of this row: set 0 (sums) / set 1 at +1024, quarter qq at + qq*256
    // metadata of this thread's row in tile `t` (s < 0: absent edge / padding destination / beyond the end)
    auto load_md = [&](long long t, int& s_, int& ty_, int& dst_, float& dist_) {
      s_ = -1; ty_ = 3; dst_ = 0; dist_ = 0.f;
      if (t < my_tiles) {
        const long long idx = (blockIdx.x + t * (long long)gridDim.x) * kTile + r;
        if (idx < n_rows) {
          int j;
          const unsigned a = row_dst(idx, j);
          const int d = row_nodes[a];
          if (d >= 0) {
            dst_ = d;
            const size_t e = (size_t)d * k + j;
            s_ = src[e]; ty_ = etype[e]; dist_ = dist_arr[e];
          }
        }
      }
    };
    // this quarter's chunk of the G row of one tile.  K slots of a 32-slot half: 8*qq + i = gaussian 5*qq + i (i < 5), slot 29 = 1
    // (constant row: type column + bias); half 0 = edge from a protein atom (types 3 / 2), half 1 = from a ligand atom (types 1 / 0).
    auto write_g = [&](int s_, int ty_, float dist_) {
      const bool ok = s_ >= 0;
      float gv[8];
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const float t = dist_ - mu[i];
        gv[i] = ok ? ex2_approx(coeff2 * (t * t)) : 0.0f;          // exp(coeff t^2); the bf16 split below keeps 16 bits of it
      }
      gv[5] = (ok && qq == 3) ? 1.0f : 0.0f;
      uint32_t hi[4], lo[4];
      split2(gv[0], gv[1], hi[0], lo[0]);
      split2(gv[2], gv[3], hi[1], lo[1]);
      split2(gv[4], gv[5], hi[2], lo[2]);
      hi[3] = lo[3] = 0u;
      const uint32_t half = (ty_ < 2) ? 4u : 0u;
      const uint32_t sw = (uint32_t)(r & 7);
      const uint32_t a_own = g_row + ((((uint32_t)qq + half) ^ sw) << 4), a_other = g_row + ((((uint32_t)qq + (half ^ 4u)) ^ sw) << 4);
      sts128(a_own, hi[0], hi[1], hi[2], hi[3]);
      sts128(a_own + kGAtom, lo[0], lo[1], lo[2], lo[3]);
      sts128(a_other, 0u, 0u, 0u, 0u);
      sts128(a_other + kGAtom, 0u, 0u, 0u, 0u);
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_G_FULL));
    };
    int s0, t0, d0, s1, t1, d1;
    float dist0, dist1;
    load_md(0, s0, t0, d0, dist0);
    if (my_tiles > 0) write_g(s0, t0, dist0);
    load_md(1, s1, t1, d1, dist1);
    for (long long it = 0; it < my_tiles; ++it) {
      const uint32_t ph = (uint32_t)(it & 1);
      const bool valid = s0 >= 0;
      // ---- P[src, offB + 32*qq ..] (absent slots read the all-zero row `zero_row` kept by the engine) + P[dst, offA + 32*qq ..]
      //      (rows of a warp usually share the destination: broadcast loads); both stay in flight while we wait for Dpre
      const float* ps = P + (size_t)(valid ? s0 : zero_row) * TD_NPROJ + offB + 32 * qq;
      float4 av[8], bv[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        bv[c] = __ldg(reinterpret_cast<const float4*>(ps + 4 * c));
        av[c] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (valid) av[c] = __ldg(reinterpret_cast<const float4*>(P + (size_t)d0 * TD_NPROJ + offA + 32 * qq + 4 * c));
      }
      f2 x[16];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        x[2 * c] = add2(pk2(bv[c].x, bv[c].y), pk2(av[c].x, av[c].y)); x[2 * c + 1] = add2(pk2(bv[c].z, bv[c].w), pk2(av[c].z, av[c].w));
      }
      // ---- + gaussian/type block from the tensor core
      mbar_wait(bar(B_DPRE_FULL), ph);
      {
        uint32_t v0[16], v1[16];
        lds16(dp_row, v0);
        lds16(dp_row + 64u, v1);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          x[i] = add2(x[i], pk2(__uint_as_float(v0[2 * i]), __uint_as_float(v0[2 * i + 1])));
          x[8 + i] = add2(x[8 + i], pk2(__uint_as_float(v1[2 * i]), __uint_as_float(v1[2 * i + 1])));
        }
      }
      // ---- gaussians of the NEXT tile now (the small MMA overlaps this tile's LayerNorm), metadata two ahead.  Writing G(it+1)
      //      also tells the MMA warpgroup that this warp has read Dpre(it).
      if (it + 1 < my_tiles) write_g(s1, t1, dist1);
      s0 = s1; t0 = t1; d0 = d1; dist0 = dist1;
      load_md(it + 2, s1, t1, d1, dist1);
      if (s0 >= 0) prefetch_l1(P + (size_t)d0 * TD_NPROJ + offA + 32 * qq);      // next tile's destination row quarter -> L1
      // ---- LayerNorm over the 128 features of the row: 4 threads (feature quarters) exchange partial sums through smem.
      //      Slot set 0 is rewritten only after every thread passed this tile's second barrier, set 1 only after the next tile's first.
      f2 sa = add2(x[0], x[1]), sb = add2(x[2], x[3]), sc = add2(x[4], x[5]), sd = add2(x[6], x[7]);
      sa = add2(sa, add2(x[8], x[9])); sb = add2(sb, add2(x[10], x[11])); sc = add2(sc, add2(x[12], x[13])); sd = add2(sd, add2(x[14], x[15]));
      float p0, p1;
      upk2(add2(add2(sa, sb), add2(sc, sd)), p0, p1);
      sts32f(xslot + (uint32_t)qq * 256u, p0 + p1);
      named_bar_sync(1 + q, 128);
      const float mean = ((lds32f(xslot) + lds32f(xslot + 256u)) + (lds32f(xslot + 512u) + lds32f(xslot + 768u))) * (1.0f / 128.0f);
      const f2 mean2 = pk2(mean, mean);
      f2 qa = pk2(0.f, 0.f), qb = qa, qc = qa, qd = qa;
#pragma unroll
      for (int i = 0; i < 16; i += 4) {
        x[i] = sub2(x[i], mean2); x[i + 1] = sub2(x[i + 1], mean2); x[i + 2] = sub2(x[i + 2], mean2); x[i + 3] = sub2(x[i + 3], mean2);
        qa = fma2(x[i], x[i], qa); qb = fma2(x[i + 1], x[i + 1], qb); qc = fma2(x[i + 2], x[i + 2], qc); qd = fma2(x[i + 3], x[i + 3], qd);
      }
      upk2(add2(add2(qa, qb), add2(qc, qd)), p0, p1);
      sts32f(xslot + 1024u + (uint32_t)qq * 256u, p0 + p1);
      named_bar_sync(1 + q, 128);
      const float var = ((lds32f(xslot + 1024u) + lds32f(xslot + 1280u)) + (lds32f(xslot + 1536u) + lds32f(xslot + 1792u))) * (1.0f / 128.0f);
      const float rstd = rsqrtf(var + 1e-5f);
      // ---- affine + ReLU, bf16 split -> this row's 32 features of both A pieces (K-major SWIZZLE_128B: 4 chunks of 16 B).
      //      Absent rows carry x = 0: their (finite) outputs are never consumed.
      uint32_t hi[16], lo[16];
      {
        const f2 rstd2 = pk2(rstd, rstd);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float4 g = lp.g4[8 * qq + c], b = lp.b4[8 * qq + c];
          float y0, y1, y2, y3;
          upk2(fma2(x[2 * c], mul2(rstd2, pk2(g.x, g.y)), pk2(b.x, b.y)), y0, y1);
          upk2(fma2(x[2 * c + 1], mul2(rstd2, pk2(g.z, g.w)), pk2(b.z, b.w)), y2, y3);
          split2(fmaxf(y0, 0.f), fmaxf(y1, 0.f), hi[2 * c], lo[2 * c]);
          split2(fmaxf(y2, 0.f), fmaxf(y3, 0.f), hi[2 * c + 1], lo[2 * c + 1]);
        }
      }
      mbar_wait(bar(B_A_EMPTY), ph ^ 1u);         // the previous tile's MMAs have read A
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const uint32_t a = a_row + ((((uint32_t)(4 * (qq & 1) + c)) ^ (uint32_t)(r & 7)) << 4);
        sts128(a, hi[4 * c], hi[4 * c + 1], hi[4 * c + 2], hi[4 * c + 3]);
        sts128(a + 2u * kGAtom, lo[4 * c], lo[4 * c + 1], lo[4 * c + 2], lo[4 * c + 3]);
      }
      fence_proxy_async();                        // A -> visible to the tensor-core (async) proxy
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_A_FULL));
    }
  } else if (warp < kMmaWarps) {
    // ================================================================= MMA warpgroup
    int cur_class = tile_class(0);
    for (long long t = 0; t < my_tiles; ++t) {
      const uint32_t ph = (uint32_t)(t & 1);
      // ---- Dpre = G(t) . TabClass^T   (K = 64: four K=16 instructions per product term)
      mbar_wait(bar(B_G_FULL), ph);               // every row warp has written G(t), i.e. has also read Dpre(t-1)
      if (t == 0) mbar_wait(bar(B_LOAD), 0);      // W2 pieces and the first class table have landed
      const int cls = tile_class(t);
      if (cls != cur_class) {                     // at most once per CTA and launch (tiles are class-sorted): swap the table by TMA
        if (tid == 0) {
          mbar_expect_tx(bar(B_TAB), (uint32_t)kTabClassBytes);
          bulk_g2s(sT, tab_image + (size_t)cls * kTabClassBytes, (uint32_t)kTabClassBytes, bar(B_TAB));
        }
        mbar_wait(bar(B_TAB), 0);
        cur_class = cls;
      }
      {
        float d[64];
        wgmma_fence();
        uint32_t accum = 0;
#pragma unroll
        for (int term = 0; term < 3; ++term) {
          const int pa_ = (term == 2) ? 1 : 0, pb_ = (term == 1) ? 1 : 0;      // a1b1, a1b2, a2b1
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            wgmma_n128(d, gmma_desc_sw128(sG + pa_ * kGAtom + kk * 32), gmma_desc_sw128(sT + pb_ * (kTabClassBytes / 2) + kk * 32), accum);
            accum = 1;
          }
        }
        wgmma_commit();
        wgmma_wait_all();
        store_frag<128>(sDp, d, warp, lane);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_DPRE_FULL));
      // ---- D = A(t) . W2^T
      mbar_wait(bar(B_A_FULL), ph);
      {
        float d[NOUT / 2];
        wgmma_fence();
        uint32_t accum = 0;
#pragma unroll
        for (int term = 0; term < 3; ++term) {
          const int pa_ = (term == 2) ? 1 : 0, pb_ = (term == 1) ? 1 : 0;
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) {
            const uint32_t aoff = (uint32_t)(pa_ * 2 * kGAtom + (kk >> 2) * kGAtom + (kk & 3) * 32);
            const uint32_t woff = (uint32_t)(pb_ * kWPiece + (kk >> 2) * kWAtom + (kk & 3) * 32);
            if constexpr (NOUT == 128) wgmma_n128(d, gmma_desc_sw128(sA + aoff), gmma_desc_sw128(sW + woff), accum);
            else wgmma_n16(d, gmma_desc_sw128(sA + aoff), gmma_desc_sw128(sW + woff), accum);
            accum = 1;
          }
        }
        wgmma_commit();
        wgmma_wait_all();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(B_A_EMPTY));
        mbar_wait(bar(B_D_EMPTY), ph ^ 1u);       // the epilogue is done with D(t-1)
        store_frag<NOUT>(sD, d, warp, lane);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_D_FULL));
    }
  } else {
    // ================================================================= epilogue: warp 4+w <-> rows 32 (w%2) .., columns 64 (w/2) ..
    const int eq = (warp - kEpiWarp0) & 1;
    const int HALF = (warp - kEpiWarp0) >> 1;      // one code copy for both column halves (b2 through indexed constant loads)
    const uint32_t drow = sD + 4u * ((uint32_t)(eq * 32 + lane) * kDRow + (uint32_t)(64 * HALF));
    for (long long it = 0; it < my_tiles; ++it) {
      const long long tile = blockIdx.x + it * gridDim.x;
      const uint32_t ph = (uint32_t)(it & 1);
      // fused aggregation (value launch, k == 32): everything that does not depend on the accumulator is fetched before waiting for it
      const bool do_agg = NOUT == 128 && qnode == nullptr && agg.logits != nullptr;
      const bool key_sm = NOUT == 128 && qnode != nullptr && agg.key_softmax;    // key launch, k == 32: softmax in this epilogue
      const long long idx = tile * kTile + eq * 32 + lane;
      const long long dslot = tile * 2 + eq;                          // k == 32: destination index of this warp's 32 rows
      const int dnode = (do_agg && dslot < n_dst) ? row_nodes[dslot] : -1;
      const bool active = dnode >= 0;                                 // warp-uniform
      float w[8], hin[4], ew = 0.f;
      bool valid_e = false;
      int dst = -1, jj = 0;
      if (do_agg) {
        // attention weights alpha * e_w of this destination's 32 edges, heads 8 HALF .. (written by the key launch's epilogue)
        if (active) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float4 t4 = __ldg(reinterpret_cast<const float4*>(agg.logits + (size_t)idx * TD_HEADS + 8 * HALF + 4 * i));
            w[4 * i] = t4.x; w[4 * i + 1] = t4.y; w[4 * i + 2] = t4.z; w[4 * i + 3] = t4.w;
          }
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) w[i] = 0.0f;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) hin[j] = (active && lane < 16) ? agg.h[(size_t)dnode * TD_H + 64 * HALF + 16 * j + lane] : 0.0f;
        // next tile: weights and destination row -> L1
        const long long nslot = dslot + 2 * (long long)gridDim.x;
        if (it + 1 < my_tiles && nslot < n_dst) {
          prefetch_l1(agg.logits + (size_t)(idx + kTile * (long long)gridDim.x) * TD_HEADS + 8 * HALF);
          const int nn = row_nodes[nslot];
          if (lane < 2 && nn >= 0) prefetch_l1(agg.h + (size_t)nn * TD_H + 64 * HALF + 32 * lane);
        }
      } else {
        if (idx < n_rows) {
          const unsigned a = row_dst(idx, jj);
          dst = row_nodes[a];
          if (dst >= 0 && key_sm) {
            const size_t e = (size_t)dst * k + jj;
            valid_e = src[e] >= 0;
            ew = agg.e_w[e];
          }
        }
        // key launches: next tile's query half row (2 lines per destination; the 32 rows of a warp share it when k == 32) -> L1
        const long long nidx = idx + kTile * (long long)gridDim.x;
        if (NOUT == 128 && qnode != nullptr && it + 1 < my_tiles && nidx < n_rows && (lane & 15) == 0) {
          int j;
          const unsigned a = row_dst(nidx, j);
          const int nn = row_nodes[a];
          if (nn >= 0) prefetch_l1(qnode + (size_t)nn * TD_H + 64 * HALF + 2 * lane);
        }
      }
      // output row of the non-fused paths: the row index itself, or the edge slot (consumers that index by node * k + j)
      const long long orow = out_by_slot ? ((long long)dst * k + jj) : idx;
      const bool owrite = idx < n_rows && dst >= 0;
      mbar_wait_relaxed(bar(B_D_FULL), ph);
      if (NOUT == 16) {
        // ---- xv: out[row, 0:16] = D[:, 0:16] + b2   (first column half only)
        if (HALF == 0) {
          uint32_t v[16];
          lds16(drow, v);
          if (owrite) {
            float* op = out + (size_t)orow * 16;
            stg256(op, __uint_as_float(v[0]) + lp.b2[0], __uint_as_float(v[1]) + lp.b2[1], __uint_as_float(v[2]) + lp.b2[2],
                   __uint_as_float(v[3]) + lp.b2[3], __uint_as_float(v[4]) + lp.b2[4], __uint_as_float(v[5]) + lp.b2[5],
                   __uint_as_float(v[6]) + lp.b2[6], __uint_as_float(v[7]) + lp.b2[7]);
            stg256(op + 8, __uint_as_float(v[8]) + lp.b2[8], __uint_as_float(v[9]) + lp.b2[9], __uint_as_float(v[10]) + lp.b2[10],
                   __uint_as_float(v[11]) + lp.b2[11], __uint_as_float(v[12]) + lp.b2[12], __uint_as_float(v[13]) + lp.b2[13],
                   __uint_as_float(v[14]) + lp.b2[14], __uint_as_float(v[15]) + lp.b2[15]);
          }
        }
      } else if (do_agg) {
        // ---- value MLP with the attention aggregation fused in: this warp's 32 rows are the edges of destination `dnode`
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int cb = 64 * HALF;
          const int c0 = 16 * j;
          uint32_t v[16];
          lds16(drow + 4u * (uint32_t)c0, v);
          float t[16];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float wh = w[c0 / 8 + i / 4];
            upk2(mul2(add2(pk2(__uint_as_float(v[2 * i]), __uint_as_float(v[2 * i + 1])),
                           pk2(lp.b2[cb + c0 + 2 * i], lp.b2[cb + c0 + 2 * i + 1])), pk2(wh, wh)), t[2 * i], t[2 * i + 1]);
          }
          const float tot = warp_transpose_reduce<16, false>(t, lane);
          if (active && lane < 16) agg.h[(size_t)dnode * TD_H + cb + c0 + lane] = hin[j] + tot;
        }
      } else if (qnode == nullptr) {
        // ---- value MLPs: out[row, 64 HALF .. + 64] = D + b2
        float* op = out + (size_t)orow * 128 + 64 * HALF;
#pragma unroll 1
        for (int c0 = 0; c0 < 64; c0 += 32) {
          uint32_t v[32];
          lds32(drow + 4u * (uint32_t)c0, v);
          if (owrite) {
#pragma unroll
            for (int c = 0; c < 32; c += 8) {
              const float* bb = lp.b2 + 64 * HALF + c0 + c;
              stg256(op + c0 + c, __uint_as_float(v[c]) + bb[0], __uint_as_float(v[c + 1]) + bb[1], __uint_as_float(v[c + 2]) + bb[2],
                     __uint_as_float(v[c + 3]) + bb[3], __uint_as_float(v[c + 4]) + bb[4], __uint_as_float(v[c + 5]) + bb[5],
                     __uint_as_float(v[c + 6]) + bb[6], __uint_as_float(v[c + 7]) + bb[7]);
            }
          }
        }
      } else {
        // ---- key MLPs: the keys never leave the SM.  out[row, 8 HALF .. + 8] = attention logits sum_d q[dst, 8h+d] k[row, 8h+d] / sqrt(8)
        //      (reference models/uni_transformer.py:73,135); thread = edge row, q row of the destination read as broadcast loads.
        const float* qrow = qnode + (size_t)(dst >= 0 ? dst : 0) * TD_H + 64 * HALF;
        float lg[8];
#pragma unroll
        for (int c0 = 0; c0 < 64; c0 += 16) {
          float4 qv[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) qv[i] = __ldg(reinterpret_cast<const float4*>(qrow + c0 + 4 * i));
          uint32_t v[16];
          lds16(drow + 4u * (uint32_t)c0, v);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const float* bb = lp.b2 + 64 * HALF + c0 + 8 * hh;
            const float4 qa = qv[2 * hh], qb = qv[2 * hh + 1];
            float sacc = (__uint_as_float(v[8 * hh]) + bb[0]) * qa.x;
            sacc = fmaf(__uint_as_float(v[8 * hh + 1]) + bb[1], qa.y, sacc);
            sacc = fmaf(__uint_as_float(v[8 * hh + 2]) + bb[2], qa.z, sacc);
            sacc = fmaf(__uint_as_float(v[8 * hh + 3]) + bb[3], qa.w, sacc);
            sacc = fmaf(__uint_as_float(v[8 * hh + 4]) + bb[4], qb.x, sacc);
            sacc = fmaf(__uint_as_float(v[8 * hh + 5]) + bb[5], qb.y, sacc);
            sacc = fmaf(__uint_as_float(v[8 * hh + 6]) + bb[6], qb.z, sacc);
            sacc = fmaf(__uint_as_float(v[8 * hh + 7]) + bb[7], qb.w, sacc);
            lg[c0 / 8 + hh] = sacc * 0.35355339059327373f;          // 1/sqrt(8)
          }
        }
        if (key_sm) {
          // softmax over the destination's 32 edges (= this warp's rows) for this warp's 8 heads, times the edge gate: the value
          // launch's epilogue only has to weight and sum.  Head hh's max / sum end up in the lanes = hh (mod 8), then are broadcast.
          float tmp[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) tmp[i] = lg[i] = valid_e ? lg[i] * 1.4426950408889634f : -INFINITY;
          const float mx_mine = warp_transpose_reduce<8, true>(tmp, lane);
#pragma unroll
          for (int hh = 0; hh < 8; ++hh) {
            const float mx = __shfl_sync(0xffffffffu, mx_mine, hh);
            lg[hh] = valid_e ? ex2_approx(lg[hh] - mx) : 0.0f;
            tmp[hh] = lg[hh];
          }
          const float l_mine = warp_transpose_reduce<8, false>(tmp, lane);
          const float inv_mine = l_mine > 0.0f ? 1.0f / l_mine : 0.0f;
#pragma unroll
          for (int hh = 0; hh < 8; ++hh) lg[hh] = lg[hh] * ew * __shfl_sync(0xffffffffu, inv_mine, hh);      // alpha * e_w
        }
        if (key_sm ? (idx < n_rows) : owrite)
          stg256(out + (size_t)(key_sm ? idx : orow) * TD_HEADS + 8 * HALF, lg[0], lg[1], lg[2], lg[3], lg[4], lg[5], lg[6], lg[7]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_D_EMPTY));
    }
  }
}

// n_dst destinations (device counts {n_dst, split_dst} in d_counts override the host values); see the kernel comment for the row model
void td_launch_edge_mlp_v4(const float* P, int zero_row, const int* src, const unsigned char* etype, const float* dist, const int* row_nodes, long long n_dst,
                           long long split_dst, const int* d_counts, int k, const TdMlp& m, const float* h_offsets, float coeff,
                           const float* h_ln_g, const float* h_ln_b, const float* h_b2, const float* qnode, float* out, int out_by_slot,
                           const float* agg_logits, const float* agg_e_w, float* agg_h, int key_softmax, int sm_count, cudaStream_t st) {
  if (n_dst == 0) return;
  LnParams lp;
  memcpy(lp.g4, h_ln_g, sizeof(lp.g4));
  memcpy(lp.b4, h_ln_b, sizeof(lp.b4));
  memset(lp.b2, 0, sizeof(lp.b2));
  memcpy(lp.b2, h_b2, sizeof(float) * (size_t)m.nout);
  memcpy(lp.mu, h_offsets, sizeof(lp.mu));
  static size_t opted128[TD_MAX_DEVICES] = {0}, opted16[TD_MAX_DEVICES] = {0};
  td_opt_in_smem(edge_mlp_v4_kernel<128>, kSmem, opted128);
  td_opt_in_smem(edge_mlp_v4_kernel<16>, kSmem, opted16);
  const long long n_tiles = (n_dst * k + kTile - 1) / kTile;         // with d_counts: upper bound
  const int grid = (int)(n_tiles < sm_count ? n_tiles : sm_count);
  AggArgs agg = {agg_logits, agg_e_w, agg_h, (key_softmax && k == 32) ? 1 : 0};
  if (m.nout == 16)
    edge_mlp_v4_kernel<16><<<grid, kThreads, kSmem, st>>>(P, zero_row, src, etype, dist, row_nodes, n_dst, split_dst, d_counts, k, m.offA, m.offB, m.w2_img,
                                                         m.tabcls_img, coeff, nullptr, out, out_by_slot, agg, lp);
  else
    edge_mlp_v4_kernel<128><<<grid, kThreads, kSmem, st>>>(P, zero_row, src, etype, dist, row_nodes, n_dst, split_dst, d_counts, k, m.offA, m.offB, m.w2_img,
                                                          m.tabcls_img, coeff, qnode, out, out_by_slot, agg, lp);
}
