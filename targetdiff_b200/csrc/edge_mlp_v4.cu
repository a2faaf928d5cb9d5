// edge_mlp_v4.cu -- per-edge MLP, fourth generation (default): both Linear layers and every edge type's gaussian block on the Hopper
// tensor cores (wgmma), fp32-faithful through bf16 operand splitting.
//
// Math (reference models/uni_transformer.py:45-56,111-120, models/common.py:60-80 after the exact first-layer split, SURVEY App. B):
//   pre[e]  = P[dst, offA:+128] + P[src, offB:+128] + tab[type][20] + sum_j g_j(dist_e) * tab[type][j]
//   hid     = relu(LN(pre) * ln_g + ln_b)
//   out[e]  = hid . W2^T + b2
//
//   Packer contract (engine.cu, pack_edge_mlp with sign_in_w1): every term of pre comes from a first Linear whose rows are centred over
//   the 128 features and multiplied by the sign of the LayerNorm gain, and the gain's magnitude is folded into W2 / b2.  So pre arrives
//   as s * (pre - mean(pre)) and the LayerNorm reduces to  hid = relu(pre * rsqrt(sum(pre^2) / 128 + eps) + ln_b):  no mean pass and
//   no gain (ln_g = 1 is not read).  The mean left by rounding is ~1e-6 of the row's scale; its effect on the variance is its square.
//
//   * rows are visited through a CLASS-SORTED destination list (protein destinations, padded to a tile multiple, then ligand
//     destinations): a tile holds destinations of one class, hence at most two edge types -- protein destination: P->P (3) or
//     L->P (1); ligand destination: P->L (2) or L->L (0).  The gaussian/type block of BOTH is one small MMA
//         Dpre[64 x 128] = G[64 x 64] . TabClass^T,   G row = the row's 20 gaussians and a constant 1 in the 32-slot half of its type;
//   * a tile's whole chain runs in the registers of one warpgroup: G is computed in the A-fragment layout of m64k16 (register-A
//     wgmma), the Dpre accumulator is LayerNorm-ed where it lies (a row's 128 values sit in the 4 lanes of a quad: the statistics
//     are two quad shuffles), and the split hidden layer is the register A operand of D = hid . W2^T;
//   * the epilogues work on the D fragment; only the key softmax and the fused aggregation exchange per-warp partials through a
//     small shared-memory slot between the two warps that hold one destination's 32 rows.
//
// CTA = one producer warpgroup + kCons consumer warpgroups (3 for the unfolded NOUT = 128 launches, else 2: Map), one CTA per SM,
// persistent over tiles of 64 edge rows (one wgmma M).  The producer (one warp per consumer; `setmaxnreg` leaves it 32 registers and
// gives the consumers 160 with 3 consumers, 40 / 232 with 2) stages each tile in shared memory ahead of its consumer: the rows' metadata
// and the P[src] / P[dst] rows as 512-byte bulk copies.  Consumer c takes the CTA's tiles c, c + kCons, ... and owns P stage c, which it
// hands back right after reading it (before its pre-MMA).  With 2 consumers the tensor-core phases (pre-MMA, main MMA) run in a fixed
// alternating order (named barriers): one consumer's MMAs are issued whole while the other does its LayerNorm, split and epilogue.
// 3 consumers issue unordered (measured faster).  A launch covers one destination class, with that class's table resident.
// Shared memory: W2 pieces 64 KB | the class table 32 KB | ln_b + b2 1 KB | exchange slots 4 KB per consumer |
// kCons P stages of 39 KB (64 P[src] rows with a 544-byte stride, which makes the fragment-order reads free of bank conflicts,
// kDst P[dst] rows, 64 metadata records) | mbarriers.  226 KB with 3 consumers.
//
// Folded key launch (FOLD, k = 32 or 64: a tile holds at most 2 destinations).  The key epilogue only needs
//   logit[e, hd] = 1/sqrt(8) sum_d q[dst, 8 hd + d] (hid_e . W2^T + b2)[8 hd + d] = hid_e . M_dst[hd, :] + c_dst[hd],
//   M_dst[hd, f] = 1/sqrt(8) sum_d q[dst, 8 hd + d] W2[8 hd + d, f],   c_dst[hd] = 1/sqrt(8) sum_d q[dst, 8 hd + d] b2[8 hd + d],
// so the main MMA runs at N = 32 (16 heads x 2 destination slots) instead of 128.  The producer also stages the tile's q[dst] rows (in
// P[dst] slots 2 and 3, unused for k >= 32); each consumer reads them before handing the stage back, builds M (fp32 W2 from shared
// memory, CUDA cores, bf16-split) for its tile while its own pre-MMA runs, and preloads the accumulator with c_dst.  M row
// n = 8 i + 2 q + c is head 4 q + 2 (i / 2) + c of destination slot i % 2, so lane q of a row's quad holds that row's heads
// 4 q .. 4 q + 3 and the softmax / output need no exchange inside the quad.  One launch per destination class keeps one table resident.
// Shared memory: W2 fp32 64 KB | the class table 32 KB | ln_b + b2 1 KB | exchange slots 8 KB | M images 16 KB per consumer |
// c_dst 128 B per consumer | 2 P stages of 39 KB | mbarriers.  215 KB.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "tdiff_common.cuh"
#include "hopper_mma.cuh"

namespace v4 {

constexpr int kTile = 64;                  // rows per tile
constexpr int kTabClassBytes = 2 * 128 * 128;   // one class table: 2 bf16 pieces of [128 x 64]
// P stage: P[src] rows (stride padded by 32 B: the 8 rows one fragment load touches fall in distinct banks), the tile's first kDst
// destinations' P[dst] rows (k >= 8 never needs more; rows of further destinations, k <= 7, are read from global memory), and per row
// the metadata record {node, src, dist, type | (dst slot + 1) << 8 | neighbour slot << 16}
constexpr int kSrcStride = 512 + 32, kDst = 8;
constexpr int sSrc = 0, sDstRows = sSrc + kTile * kSrcStride, sMeta = sDstRows + kDst * 512, kStage = sMeta + kTile * 16;
// folded key launch: per consumer the B image of M, 2 bf16 pieces of [32 rows x 128 K] (K halves of 32 x 128 B), and the 2 x 16 c_dst
constexpr int kMAtom = 32 * 128, kMPiece = 2 * kMAtom, kMImg = 2 * kMPiece;
// Per instantiation: the consumer count, the register split and the shared-memory map (bytes from the 1024-aligned base).  The
// unfolded NOUT = 128 launches run three consumers; the folded key launch (its M images would need 274 KB with a third) and the h2x
// xv launch keep two.  FOLD: W2 in fp32 instead of its bf16 image (both 64 KB), plus the M images and c_dst.
template <int NOUT, bool FOLD>
struct Map {
  static constexpr int kCons = (NOUT == 128 && !FOLD) ? 3 : 2;   // consumer warpgroups
  static constexpr int kThreads = (kCons + 1) * 128;              // warpgroup 0 is the producer
  // setmaxnreg split of the launch's allocation: 3 consumers 128 * 32 + 3 * 128 * 160 = 512 * 128,
  // 2 consumers 128 * 40 + 2 * 128 * 232 = 384 * 168
  static constexpr int kProdRegs = kCons == 3 ? 32 : 40, kConsRegs = kCons == 3 ? 160 : 232;
  static constexpr int W = 0, T = W + 4 * 128 * 128, Par = T + kTabClassBytes, X = Par + 2 * 128 * 4,
                       M = X + kCons * 4 * 2 * 128 * 4, C = M + (FOLD ? kCons * kMImg : 0), Stage = C + (FOLD ? kCons * 32 * 4 : 0),
                       Bar = Stage + kCons * kStage, Smem = Bar + 8 * (1 + 2 * kCons);   // barriers: weights, full[kCons], empty[kCons]
  // MMA phase order (kernel comment): two consumers take turns; three issue unordered (measured faster than a ring on cfg3)
  static constexpr bool kOrdered = kCons == 2;
  // named barriers (0 is __syncthreads): 2 warp pairs per consumer, then per consumer its MMA-order barrier, then (FOLD) its
  // M-image barrier
  static constexpr int kPairBar = 1, kOrderBar = kPairBar + 2 * kCons, kFoldBar = kOrderBar + kCons;
  static_assert(M % 1024 == 0 && Stage % 128 == 0 && kStage % 128 == 0 && Smem <= 227 * 1024, "shared-memory map");
  static_assert(128 * kProdRegs + kCons * 128 * kConsRegs == kThreads * (65536 / kThreads / 8 * 8), "register split");
  static_assert(kFoldBar + kCons <= 16, "named barriers");
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_LOOP:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra WAIT_DONE;\n\tbra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
// TMA bulk copy (1-D): global -> shared, completion counted in bytes on an mbarrier
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst), "l"(gsrc), "r"(bytes),
               "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx_only(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ uint32_t cvt_bf16x2(float hi, float lo) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ void stg64(float* p, float a, float b) { asm volatile("st.global.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(a), "f"(b) : "memory"); }
__device__ __forceinline__ void stg128(float* p, float a, float b, float c, float d) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// LayerNorm bias, the output bias and the gaussian centres travel as a kernel argument (copied to shared memory)
struct LnParams { float b[128]; float b2[128]; float mu[20]; };
// Fused attention in the epilogues (k == 32: rows 0-31 and 32-63 of a tile are the edges of one destination each, held by warps
// {0, 1} and {2, 3} of the warpgroup), reference models/uni_transformer.py:73-83:  key launch writes softmax_e(q.k/sqrt 8) * e_w,
// value launch does h[dst] += sum_e w * v.
struct AggArgs {
  const float* logits;   // [rows,16] written by the key launch; NULL = plain value output
  const float* e_w;      // [N*k]
  float* h;              // [N,128] node features, updated in place (a destination's row is touched by one warp pair only)
  int key_softmax;       // key launch (k == 32): write softmax weights * e_w instead of raw logits
};

// Transposing butterfly sum over the log2(N / M) lane bits from LO_BIT up: N per-lane values in, M out (N - M shuffles instead of
// M log2(N / M) per kept value).  Each step halves the values a lane keeps -- lanes with the step's bit set keep the upper half --
// and adds what the partner lane sent, highest bit first; on return t[u] holds element (lane bits) * M + u summed over those lanes.
template <int N, int M, int LO_BIT>
__device__ __forceinline__ void transpose_reduce(float (&t)[N], int lane) {
  if constexpr (N > M) {
    constexpr int h = (N / M / 2) << LO_BIT;
    const bool up = lane & h;
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
      const float send = up ? t[i] : t[i + N / 2];
      const float keep = up ? t[i + N / 2] : t[i];
      t[i] = keep + __shfl_xor_sync(0xffffffffu, send, h);
    }
    transpose_reduce<N / 2, M, LO_BIT>(reinterpret_cast<float(&)[N / 2]>(t), lane);
  }
}
// two fp32 values -> packed bf16 high pieces and packed bf16 residuals (the residual of the first piece is exact in fp32)
__device__ __forceinline__ void split2(float y0, float y1, uint32_t& hi, uint32_t& lo) {
  hi = cvt_bf16x2(y1, y0);
  const float r0 = __fsub_rn(y0, __uint_as_float(hi << 16)), r1 = __fsub_rn(y1, __uint_as_float(hi & 0xffff0000u));
  lo = cvt_bf16x2(r1, r0);
}

}  // namespace v4

using namespace v4;

// NOUT = 128: key / value MLPs (hk, hv, xk);  NOUT = 16: the per-head scalar value MLP of h2x (xv).
// Rows: idx = a * k + j over the destination list `row_nodes` (a < n_dst; entries < 0 are padding), edge slot e = row_nodes[a] * k + j.
// Destinations below `split` are protein destinations (class table 0), the others ligand destinations (table 1); a launch covers the
// tiles of destination class `cls` only, with that class's table resident.
//
// Fragment ownership (thread t of warpgroup c, w = (t / 32) % 4, l = t % 32, q = l % 4): rows 16 w + l / 4 + 8 h (h = 0, 1), columns
// 8 i + 2 q + {0, 1} (i < NOUT / 8) -- accumulator element d[4 i + 2 h + c] (hopper_mma.cuh).
// FOLD (key MLPs, k = 32 or 64): the folded key path of the header; `w2_image` is then W2^T in fp32 ([128 f][128 out]).
template <int NOUT, bool FOLD>
__global__ void __launch_bounds__(Map<NOUT, FOLD>::kThreads, 1)
edge_mlp_v4_kernel(const float* __restrict__ P, int zero_row, const int* __restrict__ src, const unsigned char* __restrict__ etype,
                   const float* __restrict__ dist_arr, const int* __restrict__ row_nodes, long long n_dst, long long split_dst,
                   const int* __restrict__ d_counts, int k, int offA, int offB, const unsigned char* __restrict__ w2_image,
                   const unsigned char* __restrict__ tab_image, float coeff, const float* __restrict__ qnode, float* __restrict__ out, int out_by_slot, AggArgs agg,
                   int cls, const __grid_constant__ LnParams lp) {
  static_assert(!FOLD || NOUT == 128, "the fold applies to the key MLPs");
  using L = Map<NOUT, FOLD>;
  constexpr int kCons = L::kCons, kThreads = L::kThreads;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const uint32_t sbase = smem_u32(smem_raw);
  const uint32_t sW = sbase + L::W, sT = sbase + L::T, sBar = sbase + L::Bar;
  float* const s_b = reinterpret_cast<float*>(smem_raw + L::Par);       // ln_b | b2
  float* const s_b2 = s_b + 128;
  // the warp index is broadcast from lane 0 so that the compiler knows it is warp-uniform
  const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int w = warp & 3, q = lane & 3;
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
  const long long row_lo = cls ? split_rows : 0, row_hi = cls ? n_rows : split_rows;   // the launch's rows: one destination class
  const long long n_tiles = row_hi > row_lo ? (row_hi - row_lo + kTile - 1) / kTile : 0;
  const long long my_tiles = (n_tiles > blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  // P stage c: full[c] (producer -> consumer c, 32 producer lanes + the bytes of the copies), empty[c] (consumer c's 128 threads)
  auto full_bar = [&](int c) { return sBar + 8u * (1 + c); };
  auto empty_bar = [&](int c) { return sBar + 8u * (1 + kCons + c); };

  // ---- one-time setup: weight image and the launch's class table -> smem (TMA bulk copies), bias vectors -> smem
  constexpr int kWAtom = NOUT * 128;            // one K-half of a weight piece: NOUT rows x 128 B
  constexpr int kWPiece = 2 * kWAtom;
  constexpr uint32_t kWBytes = FOLD ? 4u * 128 * 128 : 2u * kWPiece;   // FOLD: W2^T fp32 (the same 64 KB as the two bf16 pieces)
  if (tid == 0) {
    mbar_init(sBar, 1);
    for (int c = 0; c < kCons; ++c) { mbar_init(full_bar(c), 32); mbar_init(empty_bar(c), 128); }
    fence_barrier_init();
    mbar_expect_tx(sBar, kWBytes + kTabClassBytes);
    bulk_g2s(sW, w2_image, kWBytes, sBar);
    bulk_g2s(sT, tab_image + (size_t)cls * kTabClassBytes, kTabClassBytes, sBar);
  }
  for (int i = tid; i < 128; i += kThreads) { s_b[i] = lp.b[i]; s_b2[i] = lp.b2[i]; }
  __syncthreads();

  if (warp < 4) {
    // ================================================================= producer
    setmaxnreg_dec<L::kProdRegs>();
    // producer warp c fills stage c for consumer c.  A tile's metadata is gathered before the wait for the stage, so only the bulk
    // copies remain between the consumer's hand-back and its next tile.
    if (warp >= kCons) return;
    const int c = warp;
    const uint32_t st = sbase + L::Stage + (uint32_t)c * kStage;
    for (long long it = c, use = 0; it < my_tiles; it += kCons, ++use) {
      const long long tile = blockIdx.x + it * (long long)gridDim.x, row0 = row_lo + tile * kTile;
      int j0;
      const unsigned a0 = row_dst(row0, j0);
      const long long last = (row0 + kTile - 1 < row_hi ? row0 + kTile - 1 : row_hi - 1);
      const int n_d = min(kDst, (int)(row_dst(last, j0) - a0) + 1);   // destinations with a staged P[dst] row (FOLD: at most 2, + q rows)
      int s[2];
      int4 meta[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long idx = row0 + lane + 32 * h;
        int jj = 0, ty = 3, slot = 0, node = -1;
        float dist = 0.f;
        s[h] = -1;
        if (idx < n_rows) {
          const unsigned a = row_dst(idx, jj);
          slot = a - a0 < (unsigned)kDst ? (int)(a - a0) + 1 : 0;
          node = row_nodes[a];
          if (node >= 0) {
            const size_t e = (size_t)node * k + jj;
            s[h] = src[e]; ty = etype[e]; dist = dist_arr[e];
          }
        }
        meta[h] = make_int4(node, s[h], __float_as_int(dist), ty | (slot << 8) | (jj << 16));
      }
      int dnode = -1;
      if (lane < n_d) dnode = row_nodes[a0 + lane];
      mbar_wait(empty_bar(c), (uint32_t)(use & 1) ^ 1u);              // the first use of a stage passes at once
#pragma unroll
      for (int h = 0; h < 2; ++h) *reinterpret_cast<int4*>(smem_raw + L::Stage + c * kStage + sMeta + 16 * (lane + 32 * h)) = meta[h];
      if (lane == 0) mbar_expect_tx_only(full_bar(c), (uint32_t)(kTile + (FOLD ? 2 : 1) * n_d) * 512u);
      __syncwarp();
      // absent slots read the all-zero row `zero_row` kept by the engine
#pragma unroll
      for (int h = 0; h < 2; ++h)
        bulk_g2s(st + sSrc + (uint32_t)(lane + 32 * h) * kSrcStride, P + (size_t)(s[h] >= 0 ? s[h] : zero_row) * TD_NPROJ + offB, 512u, full_bar(c));
      if (lane < n_d) bulk_g2s(st + sDstRows + (uint32_t)lane * 512u, P + (size_t)(dnode >= 0 ? dnode : zero_row) * TD_NPROJ + offA, 512u, full_bar(c));
      // FOLD: q[dst] rows in P[dst] slots 2 + lane (a padding destination, which has no valid edge: row 0)
      if (FOLD && lane < n_d) bulk_g2s(st + sDstRows + (uint32_t)(2 + lane) * 512u, qnode + (size_t)(dnode >= 0 ? dnode : 0) * TD_H, 512u, full_bar(c));
      mbar_arrive(full_bar(c));
    }
    return;
  }

  // ================================================================= consumers
  setmaxnreg_inc<L::kConsRegs>();
  const int cwg = (warp >> 2) - 1;
  float mu[5];
#pragma unroll
  for (int m = 0; m < 5; ++m) mu[m] = lp.mu[5 * q + m];
  const float coeff2 = coeff * 1.4426950408889634f;
  mbar_wait(sBar, 0);

  const int r_base = 16 * w + (lane >> 2);
  const int pair_bar = L::kPairBar + 2 * cwg + (w >> 1);        // named barrier of the warp pair {w & 2, (w & 2) + 1}
  float* const xslot = reinterpret_cast<float*>(smem_raw + L::X) + (size_t)(cwg * 4 + w) * 256;   // 2 sets x 128; partner at (w ^ 1)
  float* const xpart = xslot + ((w & 1) ? -256 : 256);
  const bool do_agg = !FOLD && NOUT == 128 && qnode == nullptr && agg.logits != nullptr;
  const bool key_sm = NOUT == 128 && qnode != nullptr && agg.key_softmax;
  const unsigned char* const stage = smem_raw + L::Stage + cwg * kStage;
  // FOLD: this thread builds M rows of head fhd (both slots) over K runs frun and frun + 8 (8 f each).  In a quarter warp the W2
  // reads (first half fs of the head's 8 values) and the 16-byte image stores each fall in 8 distinct bank groups.
  const int ct = tid & 127, fu = ct & 7, fg = ct >> 3;
  const int fhd = 8 * (fg & 1) + 4 * (fu >> 2) + (fu & 3), fs = fu >> 2, frun = (fg >> 1) ^ (((fu >> 1) & 1) << 2);
  const int fn0 = 16 * ((fhd >> 1) & 1) + 2 * (fhd >> 2) + (fhd & 1);         // M row of (head fhd, slot 0); slot 1 is fn0 + 8
  unsigned char* const mimg = smem_raw + L::M + cwg * kMImg;
  float* const s_c = reinterpret_cast<float*>(smem_raw + L::C) + cwg * 32;      // c_dst[slot][head]
  const int srow = k == 32 ? (w >> 1) : 0;                                        // FOLD: destination slot of this warp's rows
  // MMA phase order (kOrdered), a ring: consumer 0 first, then 1, ..., kCons - 1, 0, ...  Consumer c waits on its own barrier and
  // hands over on that of c + 1 (mod kCons).  Every consumer runs the same number of iterations (one without a tile only passes the
  // order on); the last consumer's first hand-over and consumer 0's wait after the loop keep the counts equal, so no barrier is left
  // half-arrived.
  const int order_mine = L::kOrderBar + cwg, order_next = L::kOrderBar + (cwg + 1) % kCons;
  auto order_wait = [&] { if constexpr (L::kOrdered) named_bar_sync(order_mine, 256); };
  auto order_pass = [&] { if constexpr (L::kOrdered) named_bar_arrive(order_next, 256); };
  const long long n_iter = (my_tiles + kCons - 1) / kCons;
  if (n_iter == 0) return;
  if (cwg == kCons - 1) order_pass();
  int set = 0;

  for (long long n = 0; n < n_iter; ++n, set ^= 1) {
    const long long it = n * kCons + cwg;
    if (it >= my_tiles) {
      if constexpr (L::kOrdered)
        for (int phase = 0; phase < 2; ++phase) { order_wait(); order_pass(); }
      continue;
    }
    const long long row0 = row_lo + (blockIdx.x + it * (long long)gridDim.x) * kTile;
    // ---- metadata of this thread's two rows (s < 0: absent edge / padding destination / beyond the end)
    long long idx[2];
    int node[2], s[2], ty[2], jj[2], dsl[2];
    float dist[2];
    mbar_wait(full_bar(cwg), (uint32_t)(n & 1));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      idx[h] = row0 + r_base + 8 * h;
      const int4 m4 = *reinterpret_cast<const int4*>(stage + sMeta + 16 * (r_base + 8 * h));
      node[h] = m4.x; s[h] = m4.y; dist[h] = __int_as_float(m4.z);
      ty[h] = m4.w & 0xff; dsl[h] = ((m4.w >> 8) & 0xff) - 1; jj[h] = m4.w >> 16;
    }
    // ---- FOLD: the edge gates (used after the main MMA) and this thread's q rows, times 1/sqrt(8), in the order its W2 reads take
    //      (half fs first); slot 1 is zero when a tile is one destination (k = 64)
    float ewp[2] = {0.f, 0.f};
    float4 qf[2][2];
    if constexpr (FOLD) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (key_sm && idx[h] < n_rows && node[h] >= 0) ewp[h] = agg.e_w[(size_t)node[h] * k + jj[h]];
#pragma unroll
      for (int sl = 0; sl < 2; ++sl)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (sl == 0 || k == 32) {
            v = *reinterpret_cast<const float4*>(stage + sDstRows + (2 + sl) * 512 + 32 * fhd + 16 * (hf ^ fs));
            v.x *= 0.35355339059327373f; v.y *= 0.35355339059327373f; v.z *= 0.35355339059327373f; v.w *= 0.35355339059327373f;
          }
          qf[sl][hf] = v;
        }
    }
    // ---- G in the A fragment: K-slot half 0 = edge from a protein atom (types 3 / 2), half 1 = from a ligand atom (types 1 / 0).
    //      Inside the row's half, this lane's slots (kk, register) carry m = 4 (kk % 2) + 2 (register / 2) + {0, 1}: gaussian 5 q + m
    //      for m < 5, the constant 1 (type column + bias) for q = 3, m = 5 (the table image is packed to match, engine.cu).
    uint32_t ghi[4][4], glo[4][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const bool ok = s[h] >= 0;
      float v[8];
#pragma unroll
      for (int m = 0; m < 5; ++m) {
        const float t = dist[h] - mu[m];
        v[m] = ok ? ex2_approx(coeff2 * (t * t)) : 0.0f;          // exp(coeff t^2); the bf16 split below keeps 16 bits of it
      }
      v[5] = (ok && q == 3) ? 1.0f : 0.0f;
      v[6] = v[7] = 0.0f;
      const int half = ty[h] < 2 ? 1 : 0;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int hk = 0; hk < 2; ++hk) {
          uint32_t hi, lo;
          split2(v[4 * (kk & 1) + 2 * hk], v[4 * (kk & 1) + 2 * hk + 1], hi, lo);
          const bool own = (kk >> 1) == half;
          ghi[kk][h + 2 * hk] = own ? hi : 0u;
          glo[kk][h + 2 * hk] = own ? lo : 0u;
        }
    }
    // ---- x = P[src] + P[dst] from the stage, which then goes back to the producer; the pre-MMA adds Dpre = G . TabClass^T to it
    //      (K = 64: four K=16 instructions per product term), so the tensor core does that add and the stage is free before the MMA
    float x[64];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const bool valid = s[h] >= 0;
      const float* ps = reinterpret_cast<const float*>(stage + sSrc + (r_base + 8 * h) * kSrcStride) + 2 * q;
      // P[dst]: the staged row, or (a destination beyond the first kDst of the tile) global memory
      const float* pd = (dsl[h] >= 0 ? reinterpret_cast<const float*>(stage + sDstRows + dsl[h] * 512)
                                     : P + (size_t)(valid ? node[h] : zero_row) * TD_NPROJ + offA) + 2 * q;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float2 b = *reinterpret_cast<const float2*>(ps + 8 * i);
        float2 a = make_float2(0.f, 0.f);
        if (valid) a = *reinterpret_cast<const float2*>(pd + 8 * i);
        x[4 * i + 2 * h] = __fadd_rn(b.x, a.x);
        x[4 * i + 2 * h + 1] = __fadd_rn(b.y, a.y);
      }
    }
    mbar_arrive(empty_bar(cwg));                                  // P stage read: the producer may refill it
    wgmma_fence();
    order_wait();
#pragma unroll
    for (int term = 0; term < 3; ++term) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_n128_rs(x, term == 2 ? glo[kk] : ghi[kk], gmma_desc_sw128(sT + (term == 1 ? kTabClassBytes / 2 : 0) + kk * 32),
                      1u);                        // a1b1, a1b2, a2b1
    }
    wgmma_commit();
    order_pass();
    if constexpr (FOLD) {
      // ---- while the pre-MMA runs: M rows fn0 (slot 0) and fn0 + 8 (slot 1) over this thread's two K runs, split into two bf16
      //      pieces and stored in the K-major SWIZZLE_128B image (the previous tile's main MMA has completed in every warp: they all
      //      passed the order barrier above).  Per f the two halves are summed apart, so the value does not depend on fs.
      const float* const w2s = reinterpret_cast<const float*>(smem_raw + L::W) + 8 * fhd;
#pragma unroll
      for (int jr = 0; jr < 2; ++jr) {
        const int f0 = 64 * jr + 8 * frun;
        float mv[2][8];
#pragma unroll
        for (int jf = 0; jf < 8; ++jf) {
          const float4 wa = *reinterpret_cast<const float4*>(w2s + (f0 + jf) * 128 + 4 * fs);
          const float4 wb = *reinterpret_cast<const float4*>(w2s + (f0 + jf) * 128 + 4 * (fs ^ 1));
#pragma unroll
          for (int sl = 0; sl < 2; ++sl) {
            const float4 qa = qf[sl][0], qb = qf[sl][1];
            const float pa = __fmaf_rn(wa.w, qa.w, __fmaf_rn(wa.z, qa.z, __fmaf_rn(wa.y, qa.y, wa.x * qa.x)));
            const float pb = __fmaf_rn(wb.w, qb.w, __fmaf_rn(wb.z, qb.z, __fmaf_rn(wb.y, qb.y, wb.x * qb.x)));
            mv[sl][jf] = pa + pb;
          }
        }
#pragma unroll
        for (int sl = 0; sl < 2; ++sl) {
          uint4 hi, lo;
          split2(mv[sl][0], mv[sl][1], hi.x, lo.x);
          split2(mv[sl][2], mv[sl][3], hi.y, lo.y);
          split2(mv[sl][4], mv[sl][5], hi.z, lo.z);
          split2(mv[sl][6], mv[sl][7], hi.w, lo.w);
          const int nr = fn0 + 8 * sl;
          const int off = jr * kMAtom + (nr >> 3) * 1024 + (nr & 7) * 128 + ((frun ^ (nr & 7)) << 4);
          *reinterpret_cast<uint4*>(mimg + off) = hi;
          *reinterpret_cast<uint4*>(mimg + kMPiece + off) = lo;
        }
      }
      // c_dst (one thread per head)
      if (fg < 2)
#pragma unroll
        for (int sl = 0; sl < 2; ++sl) {
          const float4 ba = *reinterpret_cast<const float4*>(s_b2 + 8 * fhd + 4 * fs), bb = *reinterpret_cast<const float4*>(s_b2 + 8 * fhd + 4 * (fs ^ 1));
          const float4 qa = qf[sl][0], qb = qf[sl][1];
          const float pa = __fmaf_rn(ba.w, qa.w, __fmaf_rn(ba.z, qa.z, __fmaf_rn(ba.y, qa.y, ba.x * qa.x)));
          const float pb = __fmaf_rn(bb.w, qb.w, __fmaf_rn(bb.z, qb.z, __fmaf_rn(bb.y, qb.y, bb.x * qb.x)));
          s_c[16 * sl + fhd] = pa + pb;
        }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the image is read by wgmma (async proxy)
    }
    wgmma_wait_all();
    // ---- LayerNorm over the 128 features of each row (centred by the packer: the variance is the mean square): 32 per lane, the 4
    //      lanes of the quad combine by shuffles
    float rstd[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float qa = 0.f, qb = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        qa = __fmaf_rn(x[4 * i + 2 * h], x[4 * i + 2 * h], qa);
        qb = __fmaf_rn(x[4 * i + 2 * h + 1], x[4 * i + 2 * h + 1], qb);
      }
      float var = qa + qb;
      var += __shfl_xor_sync(0xffffffffu, var, 1);
      var += __shfl_xor_sync(0xffffffffu, var, 2);
      rstd[h] = rsqrtf(var * (1.0f / 128.0f) + 1e-5f);
    }
    // ---- normalise + bias + ReLU (unit gain), bf16 split: the accumulator columns 16 kk .. 16 kk + 15 are the A fragment of K step kk.
    //      Absent rows carry x = P[zero_row] + Dpre(0): their (finite) outputs are never consumed.
    uint32_t ahi[8][4], alo[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int h = r & 1, col = 16 * kk + 8 * (r >> 1) + 2 * q, e = 8 * kk + 2 * r;
        const float2 b = *reinterpret_cast<const float2*>(s_b + col);
        const float y0 = __fmaf_rn(x[e], rstd[h], b.x), y1 = __fmaf_rn(x[e + 1], rstd[h], b.y);
        split2(fmaxf(y0, 0.f), fmaxf(y1, 0.f), ahi[kk][r], alo[kk][r]);
      }
    // ---- D = hid . W2^T   (FOLD: D = c_dst + hid . M^T, N = 32; o[4 i + 2 h + c] is head 4 q + 2 (i / 2) + c of slot i % 2)
    float o[NOUT / 2];
    if constexpr (FOLD) {
      named_bar_sync(L::kFoldBar + cwg, 128);                        // M image and c_dst written by all 4 warps
#pragma unroll
      for (int sl = 0; sl < 2; ++sl) {
        const float4 cv = *reinterpret_cast<const float4*>(s_c + 16 * sl + 4 * q);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          o[4 * sl + 2 * h] = cv.x; o[4 * sl + 2 * h + 1] = cv.y;
          o[4 * (2 + sl) + 2 * h] = cv.z; o[4 * (2 + sl) + 2 * h + 1] = cv.w;
        }
      }
    }
    wgmma_fence();
    order_wait();
#pragma unroll
    for (int term = 0; term < 3; ++term) {
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        if constexpr (FOLD) {
          const uint64_t desc = gmma_desc_sw128(sbase + L::M + cwg * kMImg + (term == 1 ? kMPiece : 0) + (kk >> 2) * kMAtom + (kk & 3) * 32);
          wgmma_n32_rs(reinterpret_cast<float(&)[16]>(o), term == 2 ? alo[kk] : ahi[kk], desc, 1u);
        } else {
          const uint64_t desc = gmma_desc_sw128(sW + (term == 1 ? kWPiece : 0) + (kk >> 2) * kWAtom + (kk & 3) * 32);
          if constexpr (NOUT == 128) wgmma_n128_rs(o, term == 2 ? alo[kk] : ahi[kk], desc, (term | kk) ? 1u : 0u);
          else wgmma_n16_rs(o, term == 2 ? alo[kk] : ahi[kk], desc, (term | kk) ? 1u : 0u);
        }
      }
    }
    wgmma_commit();
    order_pass();
    wgmma_wait_all();

    // ================================================================= epilogue on the D fragment
    // output row of the non-fused paths: the row index itself, or the edge slot (consumers that index by node * k + j)
    long long orow[2];
    bool owrite[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      orow[h] = out_by_slot ? ((long long)node[h] * k + jj[h]) : idx[h];
      owrite[h] = idx[h] < n_rows && node[h] >= 0;
    }
    if constexpr (NOUT == 16) {
      // ---- xv: out[row, 0:16] = D + b2
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (owrite[h])
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float2 bb = *reinterpret_cast<const float2*>(s_b2 + 8 * i + 2 * q);
            stg64(out + (size_t)orow[h] * 16 + 8 * i + 2 * q, o[4 * i + 2 * h] + bb.x, o[4 * i + 2 * h + 1] + bb.y);
          }
    } else if (do_agg) {
      // ---- value MLP with the attention aggregation fused in: the warp pair's 32 rows are the edges of destination `dnode`, the
      //      staged node of each of them (-1: padding destination or beyond the end)
      const int dnode = node[0];                                      // warp-uniform
      const bool active = dnode >= 0;
      const int ccol = 64 * (w & 1) + 2 * lane;                       // the two h columns this lane writes
      float2 hin = make_float2(0.f, 0.f);
      if (active) hin = *reinterpret_cast<const float2*>(agg.h + (size_t)dnode * TD_H + ccol);
      float wt[2][16];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float4 t4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (active) t4 = __ldg(reinterpret_cast<const float4*>(agg.logits + (size_t)idx[h] * TD_HEADS + 4 * i));
          wt[h][4 * i] = t4.x; wt[h][4 * i + 1] = t4.y; wt[h][4 * i + 2] = t4.z; wt[h][4 * i + 3] = t4.w;
        }
      // t[2 i + c] = sum over this lane's two rows of (D + b2) * w[head i], column 8 i + 2 q + c
      float t[32];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float2 bb = *reinterpret_cast<const float2*>(s_b2 + 8 * i + 2 * q);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float b = c ? bb.y : bb.x;
          t[2 * i + c] = __fadd_rn(__fmul_rn(__fadd_rn(o[4 * i + c], b), wt[0][i]), __fmul_rn(__fadd_rn(o[4 * i + 2 + c], b), wt[1][i]));
        }
      }
      // over the 8 quads of the warp: lane l keeps elements 4 (l / 4) + u, i.e. columns 16 (l / 4) + 8 (u / 2) + 2 q + u % 2
      transpose_reduce<32, 4, 2>(t, lane);
      float* slot = xslot + 128 * set;
      const int c0 = 16 * (lane >> 2) + 2 * q;
      *reinterpret_cast<float2*>(slot + c0) = make_float2(t[0], t[1]);
      *reinterpret_cast<float2*>(slot + c0 + 8) = make_float2(t[2], t[3]);
      named_bar_sync(pair_bar, 64);
      if (active) {
        const float* se = ((w & 1) ? xpart : xslot) + 128 * set;       // even warp's partial first: both warps sum in one order
        const float* so = ((w & 1) ? xslot : xpart) + 128 * set;
        const float2 a = *reinterpret_cast<const float2*>(se + ccol), b = *reinterpret_cast<const float2*>(so + ccol);
        *reinterpret_cast<float2*>(agg.h + (size_t)dnode * TD_H + ccol) = make_float2(hin.x + (a.x + b.x), hin.y + (a.y + b.y));
      }
    } else if (!FOLD && qnode == nullptr) {
      // ---- value MLPs: out[row, :] = D + b2
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (owrite[h])
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float2 bb = *reinterpret_cast<const float2*>(s_b2 + 8 * i + 2 * q);
            stg64(out + (size_t)orow[h] * 128 + 8 * i + 2 * q, o[4 * i + 2 * h] + bb.x, o[4 * i + 2 * h + 1] + bb.y);
          }
    } else {
      // ---- key MLPs: the keys never leave the SM.  logits[row, hd] = sum_d q[dst, 8 hd + d] k[row, 8 hd + d] / sqrt(8)
      //      (reference models/uni_transformer.py:73,135): head hd is fragment column block i = hd; 2 products per lane, then the quad.
      //      lg[4 h + u] (after the quad reduction) = head 4 q + u of row h.
      float lg[32];
      if constexpr (FOLD) {
        // the logits are the D fragment itself: this row's slot srow, heads 4 q + 2 jb + c in o[4 (2 jb + srow) + 2 h + c]
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int e0 = 4 * (2 * (u >> 1)) + 2 * h + (u & 1);
            lg[4 * h + u] = srow ? o[e0 + 4] : o[e0];
          }
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float* qrow = qnode + (size_t)(node[h] >= 0 ? node[h] : 0) * TD_H + 2 * q;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float2 qv = __ldg(reinterpret_cast<const float2*>(qrow + 8 * i));
            const float2 bb = *reinterpret_cast<const float2*>(s_b2 + 8 * i + 2 * q);
            // element order for the reduction over the quad: 8 (i / 4) + 4 h + i % 4 -> lane q keeps heads 4 q ..
            lg[8 * (i >> 2) + 4 * h + (i & 3)] = __fmaf_rn(o[4 * i + 2 * h + 1] + bb.y, qv.y, (o[4 * i + 2 * h] + bb.x) * qv.x);
          }
        }
        transpose_reduce<32, 8, 0>(lg, lane);
#pragma unroll
        for (int u = 0; u < 8; ++u) lg[u] *= 0.35355339059327373f;          // 1/sqrt(8)
      }
      if (key_sm) {
        // softmax over the destination's 32 edges (the warp pair's rows) for this lane's 4 heads, times the edge gate: the value
        // launch's epilogue only has to weight and sum.
        bool valid_e[2];
        float ew[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          valid_e[h] = false; ew[h] = 0.f;
          if (owrite[h]) {
            valid_e[h] = s[h] >= 0;
            ew[h] = FOLD ? ewp[h] : agg.e_w[(size_t)node[h] * k + jj[h]];
          }
        }
        float mx[4], sm[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          lg[u] = valid_e[0] ? lg[u] * 1.4426950408889634f : -INFINITY;
          lg[4 + u] = valid_e[1] ? lg[4 + u] * 1.4426950408889634f : -INFINITY;
          mx[u] = fmaxf(lg[u], lg[4 + u]);
#pragma unroll
          for (int m = 4; m < 32; m <<= 1) mx[u] = fmaxf(mx[u], __shfl_xor_sync(0xffffffffu, mx[u], m));
        }
        if (lane < 4) *reinterpret_cast<float4*>(xslot + 4 * q) = make_float4(mx[0], mx[1], mx[2], mx[3]);
        named_bar_sync(pair_bar, 64);
        const float4 pm = *reinterpret_cast<const float4*>(xpart + 4 * q);
        mx[0] = fmaxf(mx[0], pm.x); mx[1] = fmaxf(mx[1], pm.y); mx[2] = fmaxf(mx[2], pm.z); mx[3] = fmaxf(mx[3], pm.w);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          lg[u] = valid_e[0] ? ex2_approx(lg[u] - mx[u]) : 0.0f;
          lg[4 + u] = valid_e[1] ? ex2_approx(lg[4 + u] - mx[u]) : 0.0f;
          sm[u] = lg[u] + lg[4 + u];
#pragma unroll
          for (int m = 4; m < 32; m <<= 1) sm[u] += __shfl_xor_sync(0xffffffffu, sm[u], m);
        }
        if (lane < 4) *reinterpret_cast<float4*>(xslot + 128 + 4 * q) = make_float4(sm[0], sm[1], sm[2], sm[3]);
        named_bar_sync(pair_bar, 64);
        const float4 ps = *reinterpret_cast<const float4*>(xpart + 128 + 4 * q);
        const float pl[4] = {ps.x, ps.y, ps.z, ps.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float l = sm[u] + pl[u];
          const float inv = l > 0.0f ? 1.0f / l : 0.0f;
          lg[u] = lg[u] * ew[0] * inv;                                 // alpha * e_w
          lg[4 + u] = lg[4 + u] * ew[1] * inv;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (idx[h] < n_rows) stg128(out + (size_t)idx[h] * TD_HEADS + 4 * q, lg[4 * h], lg[4 * h + 1], lg[4 * h + 2], lg[4 * h + 3]);
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (owrite[h]) stg128(out + (size_t)orow[h] * TD_HEADS + 4 * q, lg[4 * h], lg[4 * h + 1], lg[4 * h + 2], lg[4 * h + 3]);
      }
    }
  }
  if (cwg == 0) order_wait();                                    // matches the last consumer's last hand-over
}

// n_dst destinations (device counts {n_dst, split_dst} in d_counts override the host values); see the kernel comment for the row model
void td_launch_edge_mlp_v4(const float* P, int zero_row, const int* src, const unsigned char* etype, const float* dist, const int* row_nodes, long long n_dst,
                           long long split_dst, const int* d_counts, int k, const TdMlp& m, const float* h_offsets, float coeff,
                           const float* h_ln_b, const float* h_b2, const float* qnode, float* out, int out_by_slot,
                           const float* agg_logits, const float* agg_e_w, float* agg_h, int key_softmax, int sm_count, cudaStream_t st) {
  if (n_dst == 0) return;
  LnParams lp;
  memcpy(lp.b, h_ln_b, sizeof(lp.b));
  memset(lp.b2, 0, sizeof(lp.b2));
  memcpy(lp.b2, h_b2, sizeof(float) * (size_t)m.nout);
  memcpy(lp.mu, h_offsets, sizeof(lp.mu));
  static size_t opted128[TD_MAX_DEVICES] = {0}, opted16[TD_MAX_DEVICES] = {0}, optedF[TD_MAX_DEVICES] = {0};
  td_opt_in_smem(edge_mlp_v4_kernel<128, false>, Map<128, false>::Smem, opted128);
  td_opt_in_smem(edge_mlp_v4_kernel<16, false>, Map<16, false>::Smem, opted16);
  td_opt_in_smem(edge_mlp_v4_kernel<128, true>, Map<128, true>::Smem, optedF);
  AggArgs agg = {agg_logits, agg_e_w, agg_h, (key_softmax && k == 32) ? 1 : 0};
  // the folded key launch needs a tile to hold at most 2 destinations (k = 32 or 64); for k <= 31 or k = 48 keys are computed whole
  const bool fold = m.nout == 128 && qnode && (k == 32 || k == 64);
  // One launch per destination class (protein destinations, then ligand destinations), so that one class table is resident.  With
  // device counts the host split bounds the device one from above and the ligand part is the same on both: a class the host counts
  // as empty is empty on the device too, and the host counts give each launch an upper bound on its tiles.
  const long long n_cls[2] = {split_dst, n_dst - split_dst};
  for (int cls = 0; cls < 2; ++cls) {
    if (n_cls[cls] == 0) continue;
    const long long n_tiles = (n_cls[cls] * k + kTile - 1) / kTile;
    const int grid = (int)(n_tiles < sm_count ? n_tiles : sm_count);
    if (m.nout == 16)
      edge_mlp_v4_kernel<16, false><<<grid, Map<16, false>::kThreads, Map<16, false>::Smem, st>>>(
          P, zero_row, src, etype, dist, row_nodes, n_dst, split_dst, d_counts, k, m.offA, m.offB, m.w2_img, m.tabcls_img, coeff, nullptr,
          out, out_by_slot, agg, cls, lp);
    else if (fold)
      edge_mlp_v4_kernel<128, true><<<grid, Map<128, true>::kThreads, Map<128, true>::Smem, st>>>(
          P, zero_row, src, etype, dist, row_nodes, n_dst, split_dst, d_counts, k, m.offA, m.offB,
          reinterpret_cast<const unsigned char*>(m.w2t), m.tabcls_img, coeff, qnode, out, out_by_slot, agg, cls, lp);
    else
      edge_mlp_v4_kernel<128, false><<<grid, Map<128, false>::kThreads, Map<128, false>::Smem, st>>>(
          P, zero_row, src, etype, dist, row_nodes, n_dst, split_dst, d_counts, k, m.offA, m.offB, m.w2_img, m.tabcls_img, coeff, qnode,
          out, out_by_slot, agg, cls, lp);
  }
}
