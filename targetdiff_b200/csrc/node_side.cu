// node_side.cu -- node-side GEMMs of an attention sub-layer for the default edge-MLP mode (edge_mlp_v4, 2-piece bf16 splits), two launches:
//
//   node_proj_kernel   P[:, 0:512] = h . Wn[0:512]^T + bn[0:512]          (the [A_k | A_v | B_k | B_v] blocks the edge MLPs gather)
//   node_query_kernel  q = relu(LN(h . Wq^T + bq; ln_g, ln_b)) . W2q^T + b2q  (query MLP; q_pre = h . Wq^T + bq stays in registers)
//
// Arithmetic (same class as edge_mlp_tc.cu's modes 1 and 2): both operands as 2 bf16 pieces, x = x1 + x2, x1 = bf16(x),
// x2 = bf16(x - x1), and the 3 products a1 b1 + a1 b2 + a2 b1 accumulated in fp32 on wgmma; LayerNorm in fp32.  The q_pre block of P
// (columns 512-639) is not written: in this mode only the older edge-MLP paths would read it.
//
// Execution: one CTA per SM (grid.y = column group in node_proj_kernel), persistent over tiles of 64 rows; kWG independent warpgroups,
// warpgroup slot s = blockIdx.x * kWG + wg takes tiles s, s + gridDim.x * kWG, ...  Each warpgroup owns a 32 KB h buffer: it reads a
// tile's 64 rows from there into the register layout of the m64k16 A fragment (hopper_mma.cuh), splits them once, starts the cp.async
// copies of its next tile into the freed buffer, and runs every MMA of the tile from the registers (RS form) while those copies are in
// flight; the B operands (weight pieces) stay resident in shared memory.  The output goes straight from the accumulators to global
// memory; while one warpgroup drains its stores, the others keep the tensor cores busy.
//   node_proj_kernel: the 4 edge blocks are 2 column groups of 256 columns (2 blocks x 2 pieces = 128 KB of weights each); CTA x of both
//     groups takes the same tiles at about the same time, so h is read from HBM once and from L2 the second time.
//   node_query_kernel: Wq and W2q pieces (128 KB); the first MMA's accumulator gets the bias and the LayerNorm where it lies (a row's 128
//     values sit in the 4 lanes of a quad: two quad shuffles per statistic), then becomes the second MMA's A operand.
#include "tdiff_common.cuh"
#include "hopper_mma.cuh"

namespace ns {

constexpr int kWG = 3;                       // warpgroups per CTA (168 registers each at one CTA per SM)
constexpr int kThreads = kWG * 128;
constexpr int kTile = 64;                    // rows per warpgroup tile (one wgmma M)
constexpr int kAtom = 128 * 128;             // one K-half of a [128 x 128] bf16 piece: 128 rows x 128 B
constexpr int kPiece = 2 * kAtom;            // one bf16 piece of a [128 x 128] weight block
constexpr int kBlock = 2 * kPiece;           // a block's two pieces (the first two of its 3-piece image)
constexpr int kImgStride = 3 * kPiece;       // blocks of the packed 3-piece images (engine.cu, pack_umma_image)
constexpr int kHBuf = kTile * TD_H * 4;     // one warpgroup's h tile (32 KB)
// shared memory: 2 weight blocks 128 KB | kWG h tiles 96 KB | 4 x 128 fp32 parameters 2 KB  (+ 1 KB alignment slack) = 227 KB
constexpr size_t kSmem = 1024 + 2 * kBlock + kWG * kHBuf + 4 * TD_H * sizeof(float);
static_assert(kSmem <= 227 * 1024, "shared-memory map");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t cvt_bf16x2(float hi, float lo) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
__device__ __forceinline__ void stg64(float* p, float a, float b) { asm volatile("st.global.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(a), "f"(b) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// the two 64 KB weight blocks (pieces 1 and 2 of each) -> shared memory, and up to 4 x 128 fp32 parameters
__device__ __forceinline__ void stage_weights(unsigned char* sW, const unsigned char* w0, const unsigned char* w1, float* sPar,
                                              const float* p0, const float* p1, const float* p2, const float* p3) {
  for (int i = threadIdx.x; i < kBlock / 16; i += kThreads) {
    reinterpret_cast<uint4*>(sW)[i] = reinterpret_cast<const uint4*>(w0)[i];
    reinterpret_cast<uint4*>(sW + kBlock)[i] = reinterpret_cast<const uint4*>(w1)[i];
  }
  for (int i = threadIdx.x; i < TD_H; i += kThreads) {
    if (p0) sPar[i] = p0[i];
    if (p1) sPar[TD_H + i] = p1[i];
    if (p2) sPar[2 * TD_H + i] = p2[i];
    if (p3) sPar[3 * TD_H + i] = p3[i];
  }
  fence_proxy_async();            // generic-proxy stores -> visible to the tensor cores
  __syncthreads();
}

using Rows = TdRows;

// A warpgroup's h tile in shared memory: 64 rows of 512 B, 16-byte chunk c of row r at chunk position c ^ 2 (r % 4), which makes both
// the row-wise copies and the fragment-order reads below free of bank conflicts.
__device__ __forceinline__ uint32_t chunk_pos(int r, int c) { return (uint32_t)(r * 512 + ((c ^ ((r & 3) << 1)) << 4)); }
__device__ __forceinline__ void bar_sync_wg(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

// cp.async of tile `tile`'s 64 h rows into the buffer at `buf` (rows past the end and padding entries are zero-filled); warp w copies rows w, w + 4, ...
// The list entries of the warp's 16 rows are loaded once, one per lane, so that the copies are not issued behind 16 dependent loads.
__device__ __forceinline__ void load_tile_async(uint32_t buf, const float* __restrict__ in, const Rows& rw, long long n, long long tile, int t) {
  const int l = t & 31;
  long long mine = -1;
  if (l < kTile / 4) {
    const long long i = tile * kTile + (t >> 5) + 4 * l;
    mine = i < n ? (rw.list ? (long long)rw.list[i] : i) : -1;
  }
#pragma unroll 1
  for (int r = t >> 5, j = 0; r < kTile; r += 4, ++j) {
    const long long node = __shfl_sync(0xffffffffu, mine, j);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(buf + chunk_pos(r, l)), "l"(in + (size_t)(node >= 0 ? node : 0) * TD_H + 4 * l),
                 "r"(node >= 0 ? 16 : 0) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// the tile's rows (after its copies landed) in the accumulator layout of m64n128 (hopper_mma.cuh): x[4i + 2hh + c] = row hh [8i + 2(l % 4) + c],
// row hh of thread (w, l) being 16 w + l / 4 + 8 hh
__device__ __forceinline__ void read_tile(uint32_t buf, int w, int l, float (&x)[64]) {
  // column 8 i + 2 (l % 4) is chunk 2 i + (l % 4) / 2; with i = 4 I + j its position is 2 (4 I + (j ^ s)) + (l % 4) / 2, s = row % 4 (the
  // same for both rows of the thread): 4 base addresses, the rest immediate offsets
  const int s = (l >> 2) & 3;
  const uint32_t base = buf + (uint32_t)(16 * w + (l >> 2)) * 512 + ((l & 3) >> 1) * 16 + (l & 1) * 8;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t p = base + ((j ^ s) << 5);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int I = 0; I < 4; ++I) {
        const int i = 4 * I + j;
        float2 v;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(p + hh * 8 * 512 + I * 128));
        x[4 * i + 2 * hh] = v.x;
        x[4 * i + 2 * hh + 1] = v.y;
      }
  }
}

// accumulator-layout values -> the two bf16 pieces as RS-form A fragments: a[p][kk] covers K 16 kk .. 16 kk + 15 (columns 2 kk, 2 kk + 1
// of the accumulator layout), lower K in the low half of each register
__device__ __forceinline__ void split_frag(const float (&x)[64], uint32_t (&a)[2][8][4]) {
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int e = 4 * (2 * kk + (j >> 1)) + 2 * (j & 1);     // a0: row 0, K lo | a1: row 8, K lo | a2: row 0, K + 8 | a3: row 8, K + 8
      const float x0 = x[e], x1 = x[e + 1];
      const uint32_t v = cvt_bf16x2(x1, x0);
      a[0][kk][j] = v;
      a[1][kk][j] = cvt_bf16x2(x1 - __uint_as_float(v & 0xffff0000u), x0 - __uint_as_float(v << 16));   // residuals are exact in fp32
    }
}

// d = A . W^T for one [128 x 128] weight block (2 pieces at w_addr): a1 b1 | a1 b2, a2 b1 (edge_mlp_tc.cu's order, smallest last)
__device__ __forceinline__ void mma_block(float (&d)[64], const uint32_t (&a)[2][8][4], uint32_t w_addr) {
  wgmma_fence();
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    const int pa = t == 2 ? 1 : 0, pb = t == 1 ? 1 : 0;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      wgmma_n128_rs(d, a[pa][kk], gmma_desc_sw128(w_addr + pb * kPiece + (kk >> 2) * kAtom + (kk & 3) * 32), (t | kk) ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait_all();
}

// out[prow, col0 + c] = d + bias[c]
__device__ __forceinline__ void store_rows(float* __restrict__ out, int ldo, int col0, const int (&prow)[2], int l, const float (&d)[64],
                                           const float* sBias) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    if (prow[hh] < 0) continue;
    float* o = out + (size_t)prow[hh] * ldo + col0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int c = 8 * i + 2 * (l & 3);
      stg64(o + c, d[4 * i + 2 * hh] + sBias[c], d[4 * i + 2 * hh + 1] + sBias[c + 1]);
    }
  }
}

// the current tile's rows into registers (x, as read_tile), then the copies of tile `next` (>= 0) into the freed buffer: they run while
// the warpgroup does the current tile's MMAs and stores
__device__ __forceinline__ void next_tile(uint32_t buf, const float* __restrict__ in, const Rows& rw, long long n, long long next, int wg, int t,
                                          float (&x)[64]) {
  asm volatile("cp.async.wait_all;" ::: "memory");
  bar_sync_wg(wg);                // every thread's copies of this tile have landed
  read_tile(buf, t >> 5, t & 31, x);
  bar_sync_wg(wg);                // every thread has read the buffer
  if (next >= 0) load_tile_async(buf, in, rw, n, next, t);
}

__device__ __forceinline__ void tile_rows(const Rows& rw, long long n, long long tile, int w, int l, int (&prow)[2]) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const long long i = tile * kTile + 16 * w + (l >> 2) + 8 * hh;
    prow[hh] = i < n ? (rw.list ? rw.list[i] : (int)i) : -1;
  }
}

}  // namespace ns

// grid (CTAs per column group, 2): column group g = blockIdx.y writes P columns 256 g .. 256 g + 255 (weight blocks 2 g, 2 g + 1) of the
// rows of rw[g]: group 0 the A blocks [A_k | A_v] (read at edge destinations), group 1 the B blocks [B_k | B_v] (read at edge sources)
__global__ void __launch_bounds__(ns::kThreads, 1)
node_proj_kernel(const float* __restrict__ h, const unsigned char* __restrict__ wn_img, const float* __restrict__ bn, float* __restrict__ P,
                 const ns::Rows rw_a, const ns::Rows rw_b) {
  using namespace ns;
  const Rows rw = blockIdx.y ? rw_b : rw_a;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sW = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* sBias = reinterpret_cast<float*>(sW + 2 * kBlock + kWG * kHBuf);
  const int g = blockIdx.y;
  const long long n = rw.d_n ? (long long)*rw.d_n : rw.n;
  const long long n_tiles = (n + kTile - 1) / kTile, stride = (long long)gridDim.x * kWG;
  const int t = threadIdx.x & 127, l = t & 31, w = t >> 5;
  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
  const uint32_t buf = smem_u32(sW + 2 * kBlock) + wg * kHBuf, w_addr = smem_u32(sW);
  long long tile = blockIdx.x * kWG + wg;
  if (tile < n_tiles) load_tile_async(buf, h, rw, n, tile, t);        // the first tile's copies overlap the weight staging
  stage_weights(sW, wn_img + (size_t)(2 * g) * kImgStride, wn_img + (size_t)(2 * g + 1) * kImgStride, sBias, bn + 256 * g, bn + 256 * g + 128,
                nullptr, nullptr);
#pragma unroll 1
  for (; tile < n_tiles; tile += stride) {
    int prow[2];
    tile_rows(rw, n, tile, w, l, prow);
    uint32_t a[2][8][4];
    {
      float x[64];
      next_tile(buf, h, rw, n, tile + stride < n_tiles ? tile + stride : -1, wg, t, x);
      split_frag(x, a);
    }
#pragma unroll 1
    for (int j = 0; j < 2; ++j) {
      float d[64];
      mma_block(d, a, w_addr + j * kBlock);
      store_rows(P, TD_NPROJ, 256 * g + 128 * j, prow, l, d, sBias + 128 * j);
    }
  }
}

// q = relu(LN(h . Wq^T + bq)) . W2q^T + b2q, Wq = node-projection block 4 (its bias bq = bn[512:640])
__global__ void __launch_bounds__(ns::kThreads, 1)
node_query_kernel(const float* __restrict__ h, const unsigned char* __restrict__ wq_img, const float* __restrict__ bq, TdMlp m,
                  float* __restrict__ q, ns::Rows rw) {
  using namespace ns;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sW = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* sBq = reinterpret_cast<float*>(sW + 2 * kBlock + kWG * kHBuf);
  float* sG = sBq + TD_H;
  float* sB = sG + TD_H;
  float* sB2 = sB + TD_H;
  const long long n = rw.d_n ? (long long)*rw.d_n : rw.n;
  const long long n_tiles = (n + kTile - 1) / kTile, stride = (long long)gridDim.x * kWG;
  const int t = threadIdx.x & 127, l = t & 31, w = t >> 5;
  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
  const uint32_t buf = smem_u32(sW + 2 * kBlock) + wg * kHBuf, w_addr = smem_u32(sW);
  long long tile = blockIdx.x * kWG + wg;
  if (tile < n_tiles) load_tile_async(buf, h, rw, n, tile, t);
  stage_weights(sW, wq_img, m.w2_img, sBq, bq, m.ln_g, m.ln_b, m.b2);
#pragma unroll 1
  for (; tile < n_tiles; tile += stride) {
    uint32_t a[2][8][4];
    float d[64];
    next_tile(buf, h, rw, n, tile + stride < n_tiles ? tile + stride : -1, wg, t, d);
    split_frag(d, a);
    mma_block(d, a, w_addr);
    // q_pre = d + bq; LayerNorm (mean, then centred second moment) + affine + ReLU, row hh's 128 values in the 4 lanes of a quad
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int c = 8 * i + 2 * (l & 3);
        d[4 * i + 2 * hh] += sBq[c];
        d[4 * i + 2 * hh + 1] += sBq[c + 1];
        s += d[4 * i + 2 * hh] + d[4 * i + 2 * hh + 1];
      }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      const float mean = s * (1.0f / 128.0f);
      float v = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float e0 = d[4 * i + 2 * hh] - mean, e1 = d[4 * i + 2 * hh + 1] - mean;
        d[4 * i + 2 * hh] = e0;
        d[4 * i + 2 * hh + 1] = e1;
        v += e0 * e0 + e1 * e1;
      }
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      const float rstd = 1.0f / sqrtf(v * (1.0f / 128.0f) + 1e-5f);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int c = 8 * i + 2 * (l & 3);
        d[4 * i + 2 * hh] = fmaxf(d[4 * i + 2 * hh] * rstd * sG[c] + sB[c], 0.f);
        d[4 * i + 2 * hh + 1] = fmaxf(d[4 * i + 2 * hh + 1] * rstd * sG[c + 1] + sB[c + 1], 0.f);
      }
    }
    split_frag(d, a);
    mma_block(d, a, w_addr + kBlock);
    int prow[2];
    tile_rows(rw, n, tile, w, l, prow);
    store_rows(q, TD_H, 0, prow, l, d, sB2);
  }
}

// Node-side GEMMs of one sub-layer (2 launches): the A blocks of P and q on the rows of `rows_a`, the B blocks of P on the rows of
// `rows_b`; other rows of P / q are left as they were.  The host bounds `n` size the grids.
void td_launch_node_side_v4(const float* h, const unsigned char* wn_img, const float* bn, const TdMlp& q_mlp, float* P, float* q, const TdRows& rows_a,
                            const TdRows& rows_b, int sm_count, cudaStream_t st) {
  using namespace ns;
  if (rows_a.n == 0 && rows_b.n == 0) return;
  static size_t opted_p[TD_MAX_DEVICES] = {0}, opted_q[TD_MAX_DEVICES] = {0};
  td_opt_in_smem(node_proj_kernel, kSmem, opted_p);
  td_opt_in_smem(node_query_kernel, kSmem, opted_q);
  auto ctas = [](long long n_rows) { return ((n_rows + kTile - 1) / kTile + kWG - 1) / kWG; };     // warpgroup tiles -> CTAs
  const long long cp = ctas(rows_a.n > rows_b.n ? rows_a.n : rows_b.n), cq = ctas(rows_a.n);
  const int per = sm_count / 2 > 0 ? sm_count / 2 : 1;
  node_proj_kernel<<<dim3((unsigned)(cp < per ? cp : per), 2), kThreads, kSmem, st>>>(h, wn_img, bn, P, rows_a, rows_b);
  if (cq > 0)
    node_query_kernel<<<(unsigned)(cq < sm_count ? cq : sm_count), kThreads, kSmem, st>>>(h, wn_img + 4 * (size_t)kImgStride, bn + 512, q_mlp, q,
                                                                                         rows_a);
}
