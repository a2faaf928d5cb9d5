// edge_mlp_tc.cu -- per-edge MLPs and node-side GEMMs with the second Linear on the Hopper tensor cores (wgmma), fp32-faithful.
//
// Same math as edge_mlp.cu (reference models/uni_transformer.py:45-56,111-120 + models/common.py:60-80 after the exact
// first-layer split of SURVEY.md Appendix B); different execution:
//
//   * the [128 edges x 128] hidden tile and the [128 x 128] weight are split into NP bf16 pieces each
//     (x = x1 + x2 (+ x3), xi = bf16(residual)); the product is recovered with 3 (NP=2) or 6 (NP=3) wgmma
//     bf16 passes accumulating in fp32 registers:  a1b1 + a1b2 + a2b1 (+ a1b3 + a2b2 + a3b1).
//     NP=3 keeps 24 mantissa bits of both operands (error ~2^-22, i.e. fp32 GEMM class); NP=2 keeps 16.
//     Plain TF32 / BF16 single-pass MMA would break the 1e-4 position tolerance (SURVEY.md section 7).
//   * warp-specialised persistent CTA (one per SM):
//       warps 0-7   two consumer warpgroups: warpgroup g issues the wgmma of tile rows 64g..64g+63 and stores its accumulator
//                   fragment (+bias) straight to global memory
//       warps 8-15  producers: 8 edge rows per warp in registers -- coalesced 512 B gathers of the projected node
//                   rows, gaussians by 4 lanes per row, type/gaussian table through L1 (one table row feeds 8 edge rows),
//                   LayerNorm by shuffles, ReLU, bf16 split, 8-byte stores into the K-major SWIZZLE_128B layout
//     mbarriers: a_full/a_empty (producers <-> consumers), activation tiles multi-buffered (NBUF).
//   * the weight pieces are pre-swizzled on the host into the exact shared-memory image (engine.cu: pack_umma_image).
//
// Shared memory: NP*32 KB weights + NBUF*NP*32 KB activation tiles (+2 KB) -> 194 KB for (NP=3,NBUF=1) and (NP=2,NBUF=2).
#include "tdiff_common.cuh"
#include "hopper_mma.cuh"

namespace {

constexpr int kConsWarps = 8;      // warps 0-7: two consumer warpgroups (64 rows each)
constexpr int kProdWarp0 = 8;      // warps 8.. : producers, 8 warps per producer set
constexpr int kProdWarps = 8;      // warps per producer set == arrivals per activation tile
constexpr int kPieceBytes = 128 * 128 * 2;                 // one bf16 piece of a 128x128 tile
constexpr int kAtomBytes = 128 * 128;                      // 128 rows x 64 bf16 (128 B) : one K-half

// ---------------------------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// two fp32 -> packed bf16x2 (round-to-nearest-even): `lo` in bits [0,16), `hi` in bits [16,32)
__device__ __forceinline__ uint32_t cvt_bf16x2(float hi, float lo) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

// explicit shared-space accesses (the carve-up goes through uintptr_t, so plain dereferences would compile to generic LD/ST)
__device__ __forceinline__ void sts64(uint32_t addr, uint2 v) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
// streaming 16-byte gather that does not allocate in L1 (keeps the L1-resident table / destination rows from being evicted)
__device__ __forceinline__ float4 ldg_stream(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

// (d0, d1) += w * (a0, a1), two fused multiply-adds
__device__ __forceinline__ void ffma2(float& d0, float& d1, float w, float a0, float a1) {
  d0 = __fmaf_rn(w, a0, d0);
  d1 = __fmaf_rn(w, a1, d1);
}

template <int NP>
__device__ __forceinline__ void split_store_row(uint32_t a_tile, int row, int lane, const float (&y)[4]) {
  // features 4*lane .. 4*lane+3 of `row` -> NP pieces; byte offset inside a piece (K-major SWIZZLE_128B, two K-halves)
  const int khalf = lane >> 4, chunk = (lane & 15) >> 1;
  const uint32_t off = khalf * kAtomBytes + row * 128 + ((chunk ^ (row & 7)) << 4) + ((lane & 1) << 3);
  float r[4] = {y[0], y[1], y[2], y[3]};
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const uint2 v = make_uint2(cvt_bf16x2(r[1], r[0]), cvt_bf16x2(r[3], r[2]));
    r[0] -= __uint_as_float(v.x << 16); r[1] -= __uint_as_float(v.x & 0xffff0000u);       // residuals are exact in fp32
    r[2] -= __uint_as_float(v.y << 16); r[3] -= __uint_as_float(v.y & 0xffff0000u);
    sts64(a_tile + p * kPieceBytes + off, v);
  }
}

}  // namespace

// MODE 0: edge MLP (gathers + gaussian block + LN + ReLU -> second Linear), out [n_rows,128]
// MODE 1: dense rows: out[:, y*128:(y+1)*128] = in[:, :128] . W_y^T + b_y for column block y = blockIdx.y (node projection)
// MODE 2: LN rows:    out = relu(LN(in[:, in_off:in_off+128])) . W^T + b                                   (query MLP tail)
struct TcRows {
  const float* in;       // [*, ldi]
  int ldi, in_off, ldo;
  const int* row_list;   // optional: logical row i reads in[row_list[i]] and writes out[row_list[i]] (a node subset)
  const int* d_n_rows;   // optional: number of logical rows lives in device memory (list compacted on the device)
};

template <int NP, int NBUF, int NSETS, int MODE>
__global__ void __launch_bounds__((kProdWarp0 + kProdWarps * NSETS) * 32, 1)
edge_mlp_tc_kernel(const float* __restrict__ P, const float4* __restrict__ xm, const int* __restrict__ src,
                   const unsigned char* __restrict__ etype, const float* __restrict__ dist_arr, const int* __restrict__ row_nodes,
                   long long n_rows, int k, TdMlp m, const unsigned char* __restrict__ w2_image, const float* __restrict__ offsets, float coeff,
                   float* __restrict__ out, TcRows rw) {
  extern __shared__ unsigned char smem_raw[];
  // carve (1024-byte aligned: SWIZZLE_128B atoms)
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* sB = base;                                   // NP pieces
  unsigned char* sA = sB + NP * kPieceBytes;                  // NBUF x NP pieces
  float* s_b2 = reinterpret_cast<float*>(sA + NBUF * NP * kPieceBytes);   // [128]
  float* s_g = s_b2 + TD_H;
  float* s_b = s_g + TD_H;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_b + TD_H);  // a_full[NBUF], a_empty[NBUF]
  const uint32_t bar_a_full = smem_u32(bars), bar_a_empty = smem_u32(bars + NBUF);

  // the warp index is broadcast from lane 0 so that the compiler KNOWS it is warp-uniform: role branches become uniform branches and
  // every constant-bank read indexed by it (LayerNorm parameters, biases) goes through the uniform datapath (LDCU + UR operands)
  // instead of per-thread LDC into vector registers
  const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  // ---- one-time setup: weights image -> smem, params, barriers
  constexpr int kThreads = (kProdWarp0 + kProdWarps * NSETS) * 32;
  static_assert(NBUF >= NSETS, "every producer set needs its own activation buffer");
  for (int i = tid; i < NP * kPieceBytes / 16; i += kThreads)
    reinterpret_cast<uint4*>(sB)[i] = reinterpret_cast<const uint4*>(w2_image + (MODE == 1 ? (size_t)blockIdx.y * 3 * kPieceBytes : 0))[i];
  for (int i = tid; i < TD_H; i += kThreads) {
    s_b2[i] = m.b2[(MODE == 1 ? blockIdx.y * TD_H : 0) + i];
    if (MODE != 1) { s_g[i] = m.ln_g[i]; s_b[i] = m.ln_b[i]; }
  }
  if (tid == 0) {
    for (int i = 0; i < NBUF; ++i) {
      mbar_init(bar_a_full + 8 * i, kProdWarps);
      mbar_init(bar_a_empty + 8 * i, kConsWarps);
    }
    fence_barrier_init();
  }
  fence_proxy_async();            // weight image (generic-proxy stores) -> visible to the tensor-core (async) proxy
  __syncthreads();

  if (MODE != 0 && rw.d_n_rows) n_rows = *rw.d_n_rows;
  const long long n_tiles = (n_rows + 127) / 128;
  const long long my_tiles = (n_tiles > blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  if (warp >= kProdWarp0) {
    // =============================================================== producers
    // Producer set `ps` (8 warps) builds the activation tiles of the CTA's local tiles it = ps, ps+NSETS, ...; inside a set,
    // warp pw owns rows pw*16 .. pw*16+15 as two "groups" of 8 rows held in registers.
    const int ps = (warp - kProdWarp0) / kProdWarps, pw = (warp - kProdWarp0) % kProdWarps;
    if constexpr (MODE != 0) {
      // ---- dense / LN row producers: 8 rows per warp-iteration straight from `in` (coalesced 512 B rows)
      const long long n_my = (my_tiles > ps) ? (my_tiles - ps + NSETS - 1) / NSETS : 0;
      const float4 g4 = MODE == 2 ? lds128(smem_u32(s_g + 4 * lane)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 b4 = MODE == 2 ? lds128(smem_u32(s_b + 4 * lane)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
      for (long long q = 0; q < n_my * 2; ++q) {
        const long long it = ps + (q >> 1) * NSETS;
        const int buf = (int)(it % NBUF);
        const int r0 = pw * 16 + (int)(q & 1) * 8;
        const long long row0 = (blockIdx.x + it * (long long)gridDim.x) * 128 + r0;
        float acc[8][4];
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (row0 + r < n_rows) {
            const long long src_row = rw.row_list ? rw.row_list[row0 + r] : row0 + r;
            v = ldg_stream(rw.in + (size_t)src_row * rw.ldi + rw.in_off + 4 * lane);
          }
          acc[r][0] = v.x; acc[r][1] = v.y; acc[r][2] = v.z; acc[r][3] = v.w;
        }
        if (MODE == 2) {
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            const float mean = warp_sum((acc[r][0] + acc[r][1]) + (acc[r][2] + acc[r][3])) * (1.0f / 128.0f);
            const float e0 = acc[r][0] - mean, e1 = acc[r][1] - mean, e2 = acc[r][2] - mean, e3 = acc[r][3] - mean;
            const float var = warp_sum((e0 * e0 + e1 * e1) + (e2 * e2 + e3 * e3)) * (1.0f / 128.0f);
            const float rstd = 1.0f / sqrtf(var + 1e-5f);
            const bool ok = row0 + r < n_rows;
            acc[r][0] = ok ? fmaxf(e0 * rstd * g4.x + b4.x, 0.f) : 0.f;
            acc[r][1] = ok ? fmaxf(e1 * rstd * g4.y + b4.y, 0.f) : 0.f;
            acc[r][2] = ok ? fmaxf(e2 * rstd * g4.z + b4.z, 0.f) : 0.f;
            acc[r][3] = ok ? fmaxf(e3 * rstd * g4.w + b4.w, 0.f) : 0.f;
          }
        }
        if ((q & 1) == 0) mbar_wait(bar_a_empty + 8 * buf, (uint32_t)(((it / NBUF) & 1) ^ 1));
        const uint32_t a_tile = smem_u32(sA) + buf * NP * kPieceBytes;
#pragma unroll
        for (int r = 0; r < 8; ++r) split_store_row<NP>(a_tile, r0 + r, lane, acc[r]);
        if (q & 1) {
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_a_full + 8 * buf);
        }
      }
    } else {
    const int rsub = lane >> 2, jq = lane & 3;   // metadata: 4 lanes per row; lane holds gaussians 5*jq .. 5*jq+4 of row rsub
    float mu[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) mu[i] = offsets[5 * jq + i];
    const long long n_my = (my_tiles > ps) ? (my_tiles - ps + NSETS - 1) / NSETS : 0;   // tiles of this set
    const long long n_groups = n_my * 2;

    auto load_md = [&](long long q, int& s_, int& ty_, int& dst_, float& dist_) {
      s_ = -1; ty_ = 0; dst_ = 0; dist_ = 0.f;
      if (q < n_groups) {
        const long long tile = blockIdx.x + (ps + (q >> 1) * NSETS) * (long long)gridDim.x;
        const long long idx64 = tile * 128 + pw * 16 + (int)(q & 1) * 8 + rsub;
        if (idx64 < n_rows) {
          const unsigned idx = (unsigned)idx64;
          const unsigned a = idx / (unsigned)k;
          const int j = (int)(idx - a * (unsigned)k);
          dst_ = row_nodes ? row_nodes[a] : (int)a;
          const size_t e = (size_t)dst_ * k + j;
          s_ = src[e];
          ty_ = etype[e];
          dist_ = dist_arr[e];
        }
      }
    };
    int s0, t0, d0, s1, t1, d1;
    float dist0, dist1;
    load_md(0, s0, t0, d0, dist0);
#pragma unroll 1
    for (long long q = 0; q < n_groups; ++q) {
      load_md(q + 1, s1, t1, d1, dist1);        // coalesced metadata of the next group, consumed one iteration later
      const long long it = ps + (q >> 1) * NSETS;
      const int buf = (int)(it % NBUF);
      const int r0 = pw * 16 + (int)(q & 1) * 8;
      const bool valid = s0 >= 0;
      // ---- gathers: acc[r] = P[src_r, offB + 4l..] (8 x 512 B coalesced rows), + P[dst, offA + 4l..]
      float acc[8][4];
      unsigned vmask = 0;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int sr = __shfl_sync(0xffffffffu, s0, r * 4);
        float4 pb = make_float4(0.f, 0.f, 0.f, 0.f);
        if (sr >= 0) {
          vmask |= 1u << r;
          pb = __ldg(reinterpret_cast<const float4*>(P + (size_t)sr * TD_NPROJ + m.offB + 4 * lane));   // neighbour lists overlap: L1 reuse
        }
        acc[r][0] = pb.x; acc[r][1] = pb.y; acc[r][2] = pb.z; acc[r][3] = pb.w;
      }
      const int dfirst = __shfl_sync(0xffffffffu, d0, 0);
      if (__all_sync(0xffffffffu, !valid || d0 == dfirst)) {          // usual case (k % 8 == 0): one destination per group
        const float4 pa = __ldg(reinterpret_cast<const float4*>(P + (size_t)dfirst * TD_NPROJ + m.offA + 4 * lane));
#pragma unroll
        for (int r = 0; r < 8; ++r)
          if ((vmask >> r) & 1u) { acc[r][0] += pa.x; acc[r][1] += pa.y; acc[r][2] += pa.z; acc[r][3] += pa.w; }
      } else {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const int dr = __shfl_sync(0xffffffffu, d0, r * 4);
          if ((vmask >> r) & 1u) {
            const float4 pa = __ldg(reinterpret_cast<const float4*>(P + (size_t)dr * TD_NPROJ + m.offA + 4 * lane));
            acc[r][0] += pa.x; acc[r][1] += pa.y; acc[r][2] += pa.z; acc[r][3] += pa.w;
          }
        }
      }
      float g[5];
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const float t = dist0 - mu[i];
        g[i] = valid ? expf(coeff * (t * t)) : 0.0f;
      }
      // ---- type / gaussian block of the first Linear: one table row (through L1) feeds the 8 edge rows of the group
#pragma unroll 1
      for (int t = 0; t < 4; ++t) {
        const bool mine = valid && (t0 == t);
        if (!__any_sync(0xffffffffu, mine)) continue;
        const float* tb = m.tab + (size_t)t * TD_TAB * TD_H + 4 * lane;
        {
          const float4 c = __ldg(reinterpret_cast<const float4*>(tb + TD_NG * TD_H));       // type column + bias
          const float wm = mine ? 1.0f : 0.0f;
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            const float w = __shfl_sync(0xffffffffu, wm, r * 4);
            ffma2(acc[r][0], acc[r][1], w, c.x, c.y);
            ffma2(acc[r][2], acc[r][3], w, c.z, c.w);
          }
        }
#pragma unroll
        for (int jj = 0; jj < TD_NG; ++jj) {
          const float4 c = __ldg(reinterpret_cast<const float4*>(tb + jj * TD_H));
          const float gm = mine ? g[jj % 5] : 0.0f;
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            const float w = __shfl_sync(0xffffffffu, gm, r * 4 + jj / 5);
            ffma2(acc[r][0], acc[r][1], w, c.x, c.y);
            ffma2(acc[r][2], acc[r][3], w, c.z, c.w);
          }
        }
      }
      // ---- LayerNorm + ReLU (rows are independent: 8 interleaved shuffle chains)
      const float4 g4 = lds128(smem_u32(s_g + 4 * lane));
      const float4 b4 = lds128(smem_u32(s_b + 4 * lane));
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float mean = warp_sum((acc[r][0] + acc[r][1]) + (acc[r][2] + acc[r][3])) * (1.0f / 128.0f);
        const float e0 = acc[r][0] - mean, e1 = acc[r][1] - mean, e2 = acc[r][2] - mean, e3 = acc[r][3] - mean;
        const float var = warp_sum((e0 * e0 + e1 * e1) + (e2 * e2 + e3 * e3)) * (1.0f / 128.0f);
        const float rstd = 1.0f / sqrtf(var + 1e-5f);
        const bool ok = (vmask >> r) & 1u;
        acc[r][0] = ok ? fmaxf(e0 * rstd * g4.x + b4.x, 0.f) : 0.f;
        acc[r][1] = ok ? fmaxf(e1 * rstd * g4.y + b4.y, 0.f) : 0.f;
        acc[r][2] = ok ? fmaxf(e2 * rstd * g4.z + b4.z, 0.f) : 0.f;
        acc[r][3] = ok ? fmaxf(e3 * rstd * g4.w + b4.w, 0.f) : 0.f;
      }
      // ---- bf16 split + swizzled store into the activation tile (wait for the tensor core to be done with the buffer)
      if ((q & 1) == 0) mbar_wait(bar_a_empty + 8 * buf, (uint32_t)(((it / NBUF) & 1) ^ 1));
      const uint32_t a_tile = smem_u32(sA) + buf * NP * kPieceBytes;
#pragma unroll
      for (int r = 0; r < 8; ++r) split_store_row<NP>(a_tile, r0 + r, lane, acc[r]);
      if (q & 1) {
        fence_proxy_async();          // activation tile -> visible to the tensor-core (async) proxy
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_a_full + 8 * buf);
      }
      s0 = s1; t0 = t1; d0 = d1; dist0 = dist1;
    }
    }
  } else {
    // =============================================================== consumers: warpgroup g = rows 64g..64g+63 of every tile
    const int g = warp >> 2, wq = warp & 3;
    for (long long it = 0; it < my_tiles; ++it) {
      const long long tile = blockIdx.x + it * gridDim.x;
      const int buf = (int)(it % NBUF);
      mbar_wait(bar_a_full + 8 * buf, (uint32_t)((it / NBUF) & 1));      // activation tile written
      const uint32_t a_addr = smem_u32(sA + buf * NP * kPieceBytes) + (uint32_t)g * 64u * 128u, b_addr = smem_u32(sB);
      float d[64];
      wgmma_fence();
      uint32_t accum = 0;
      // terms (pa, pb) with pa + pb <= NP-1:  a1b1 | a1b2, a2b1 | a1b3, a2b2, a3b1 ; smallest contributions last
#pragma unroll
      for (int sum = 0; sum < NP; ++sum) {
#pragma unroll
        for (int pa = 0; pa <= sum; ++pa) {
          const int pb = sum - pa;
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) {             // K = 128 in 8 instructions of K=16 (32 B inside a 128 B swizzle row)
            const uint32_t koff = (kk >> 2) * kAtomBytes + (kk & 3) * 32;
            wgmma_n128(d, gmma_desc_sw128(a_addr + pa * kPieceBytes + koff), gmma_desc_sw128(b_addr + pb * kPieceBytes + koff), accum);
            accum = 1;
          }
        }
      }
      wgmma_commit();
      wgmma_wait_all();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_a_empty + 8 * buf);        // activation tile may be overwritten
      // ---- fragment -> global: rows r0 and r0 + 8, columns 8i + 2 (lane % 4) + {0, 1}
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long idx = tile * 128 + 64 * g + 16 * wq + (lane >> 2) + 8 * h;
        if (idx >= n_rows) continue;
        const long long orow_i = (MODE != 0 && rw.row_list) ? rw.row_list[idx] : idx;
        float* orow = out + (size_t)orow_i * (MODE == 0 ? 128 : rw.ldo) + (MODE == 1 ? blockIdx.y * 128 : 0);
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int c = 8 * i + 2 * (lane & 3);
          *reinterpret_cast<float2*>(orow + c) = make_float2(d[4 * i + 2 * h] + s_b2[c], d[4 * i + 2 * h + 1] + s_b2[c + 1]);
        }
      }
    }
  }
}

template <int NP, int NBUF, int NSETS, int MODE>
static void launch_tc(const float* P, const float4* xm, const int* src, const unsigned char* etype, const float* dist, const int* row_nodes,
                      long long n_rows, int k, TdMlp m, const unsigned char* w2_image, const float* offsets, float coeff, float* out, TcRows rw,
                      int nblocks, int sm_count, cudaStream_t st) {
  const size_t smem = 1024 + (size_t)NP * kPieceBytes + (size_t)NBUF * NP * kPieceBytes + 3 * TD_H * sizeof(float) + 2 * NBUF * 8;
  static size_t opted[TD_MAX_DEVICES] = {0};
  td_opt_in_smem(edge_mlp_tc_kernel<NP, NBUF, NSETS, MODE>, smem, opted);
  const long long n_tiles = (n_rows + 127) / 128;
  int per = sm_count / nblocks;
  if (per < 1) per = 1;
  dim3 grid((unsigned)(n_tiles < per ? n_tiles : per), (unsigned)nblocks);
  edge_mlp_tc_kernel<NP, NBUF, NSETS, MODE><<<grid, (kProdWarp0 + kProdWarps * NSETS) * 32, smem, st>>>(P, xm, src, etype, dist, row_nodes, n_rows, k,
                                                                                                     m, w2_image, offsets, coeff, out, rw);
}

// pieces = 3: 6-term product (fp32-class accuracy); pieces = 2: 3-term product (16 mantissa bits).  nout must be 128.
void td_launch_edge_mlp_tc(const float* P, const float4* xm, const int* src, const unsigned char* etype, const float* dist,
                           const int* row_nodes, long long n_rows, int k, TdMlp m, const unsigned char* w2_image, int pieces, const float* offsets, float coeff,
                           float* out, int sm_count, cudaStream_t st) {
  if (n_rows == 0) return;
  TcRows rw = {nullptr, 0, 0, 128, nullptr, nullptr};
  if (pieces == 2) launch_tc<2, 2, 1, 0>(P, xm, src, etype, dist, row_nodes, n_rows, k, m, w2_image, offsets, coeff, out, rw, 1, sm_count, st);
  else launch_tc<3, 1, 1, 0>(P, xm, src, etype, dist, row_nodes, n_rows, k, m, w2_image, offsets, coeff, out, rw, 1, sm_count, st);
}

// Node-side GEMMs on the same tensor-core pipeline.
//   mode 1: out[n_rows, nblocks*128] = in[n_rows,128] . W^T + bias, W given as `nblocks` images of [128 x 128] (node projection, nblocks = 5)
//   mode 2: out[n_rows,128] = relu(LN(in[:, in_off:in_off+128]; m.ln_g, m.ln_b)) . W^T + m.b2                         (query MLP tail)
void td_launch_rows_tc(int mode, const float* in, int ldi, int in_off, long long n_rows, TdMlp m, const unsigned char* w_image, int pieces, float* out,
                       int ldo, int nblocks, const int* row_list, const int* d_n_rows, int sm_count, cudaStream_t st) {
  if (n_rows == 0) return;          // with d_n_rows, n_rows is only the upper bound used to size the grid
  TcRows rw = {in, ldi, in_off, ldo, row_list, d_n_rows};
  if (mode == 1) {
    if (pieces == 2) launch_tc<2, 2, 1, 1>(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, n_rows, 1, m, w_image, nullptr, 0.f, out, rw, nblocks, sm_count, st);
    else launch_tc<3, 1, 1, 1>(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, n_rows, 1, m, w_image, nullptr, 0.f, out, rw, nblocks, sm_count, st);
  } else {
    if (pieces == 2) launch_tc<2, 2, 1, 2>(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, n_rows, 1, m, w_image, nullptr, 0.f, out, rw, 1, sm_count, st);
    else launch_tc<3, 1, 1, 2>(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, n_rows, 1, m, w_image, nullptr, 0.f, out, rw, 1, sm_count, st);
  }
}
