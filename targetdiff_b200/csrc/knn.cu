// knn.cu -- fused per-graph k-NN -> dst-sorted fixed-degree neighbour list (CSR with constant row length k).
//
// Replaces torch_geometric.nn.knn_graph(x, k, batch, flow='source_to_target') -> torch_cluster.knn
// (reference call site models/uni_transformer.py:280).  Canonical semantics (SURVEY.md Appendix A.3):
//   d2 = ((dx*dx)+(dy*dy))+(dz*dz), every op rounded to fp32 (no FMA contraction); ascending d2, ties -> smaller
//   node index; self removed; graphs with <= k nodes give fewer edges (slots padded with -1).
// The (d2, index) order is realised with one 64-bit key  (float_as_uint(d2) << 32) | local_index : d2 >= 0 so the
// IEEE bit pattern is monotone, keys are unique, and "k+1 smallest keys" is exactly the canonical selection.
//
// cutoff_mode = 'hybrid' (reference models/common.py:165-212, add_p_index=True): protein destinations keep the k-NN over all atoms of
// the graph; a ligand destination gets every other ligand atom of its graph (ascending node index) followed by its k nearest PROTEIN
// atoms by the same (d2, index) key.  The reference ranks torch.norm distances with torch.topk, whose order among equal norms is
// unspecified, and distinct fp32 d2 can round to one norm: where such a tie falls at the k-th place the reference's choice differs
// (DESIGN.md section 2, restate.hybrid_graph_canonical).  Rows have `stride` >= k slots (the engine uses stride = k + max ligand atoms
// per graph - 1); unused slots are -1.
//
// Mapping: one CTA per (graph, chunk of queries); the graph's coordinates are staged once in shared memory
// (coalesced float4 loads); one warp per query holds the key row in shared memory, each lane tracks the minimum of
// its strided slice; k+1 rounds of a 64-bit warp-min pick the neighbours in order, only the winning lane rescans.
#include "tdiff_common.cuh"

#define KNN_WARPS 8

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = (w < v) ? w : v;
  }
  return v;
}

// One hybrid ligand row (warp-collective): other ligand atoms of the graph, then the k nearest protein atoms; `keys` = this warp's
// shared-memory key row, `spos` = the graph's staged coordinates (protein atoms first).
__device__ __forceinline__ void hybrid_ligand_row(const float4* spos, unsigned long long* keys, int qi, int np, int ng, int k, int stride, int base,
                                                  int lane, int* out) {
  const int nl = ng - np;
  for (int j = lane; j < nl; j += 32) {
    const int node = np + j;
    if (node != qi) out[j - (node > qi ? 1 : 0)] = base + node;
  }
  const float4 xq = spos[qi];
  unsigned long long lmin = ~0ull;
  for (int j = lane; j < np; j += 32) {
    const float4 xc = spos[j];
    const float dx = __fsub_rn(xq.x, xc.x), dy = __fsub_rn(xq.y, xc.y), dz = __fsub_rn(xq.z, xc.z);
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)j;
    keys[j] = key;
    lmin = key < lmin ? key : lmin;
  }
  __syncwarp();
  const int rounds = min(k, np);
  int written = nl - 1;
  for (int r = 0; r < rounds && written < stride; ++r) {
    const unsigned long long gmin = warp_min_u64(lmin);
    const int j = (int)(gmin & 0xffffffffu);
    if (lmin == gmin) {
      keys[j] = ~0ull;
      unsigned long long m = ~0ull;
      for (int jj = lane; jj < np; jj += 32) {
        const unsigned long long kv = keys[jj];
        m = kv < m ? kv : m;
      }
      lmin = m;
    }
    if (lane == 0) out[written] = base + j;
    ++written;
  }
  for (int w = written + lane; w < stride; w += 32) out[w] = -1;
  __syncwarp();
}

__global__ void __launch_bounds__(KNN_WARPS * 32)
knn_kernel(const float4* __restrict__ xm, const int* __restrict__ node_ptr, const int* __restrict__ prot_ptr, int k, int stride, int hybrid,
           int max_ng, int* __restrict__ src) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float4* spos = reinterpret_cast<float4*>(smem_raw);                                     // [max_ng]
  unsigned long long* skeys = reinterpret_cast<unsigned long long*>(spos + max_ng);       // [KNN_WARPS][max_ng]

  const int g = blockIdx.x;
  const int base = node_ptr[g];
  const int ng = node_ptr[g + 1] - base;
  const int np_h = hybrid ? prot_ptr[g + 1] - prot_ptr[g] : ng;          // hybrid: nodes >= np_h are ligand atoms
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = threadIdx.x; j < ng; j += blockDim.x) spos[j] = xm[base + j];
  __syncthreads();

  unsigned long long* keys = skeys + (size_t)warp * max_ng;
  const int rounds = min(k + 1, ng);
  // queries of this graph are spread over gridDim.y chunks and the CTA's warps
  for (int qi = blockIdx.y * KNN_WARPS + warp; qi < ng; qi += gridDim.y * KNN_WARPS) {
    if (qi >= np_h) {
      hybrid_ligand_row(spos, keys, qi, np_h, ng, k, stride, base, lane, src + (size_t)(base + qi) * stride);
      continue;
    }
    const float4 xq = spos[qi];
    unsigned long long lmin = ~0ull;
    for (int j = lane; j < ng; j += 32) {
      const float4 xc = spos[j];
      const float dx = __fsub_rn(xq.x, xc.x), dy = __fsub_rn(xq.y, xc.y), dz = __fsub_rn(xq.z, xc.z);
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)j;
      keys[j] = key;
      lmin = key < lmin ? key : lmin;
    }
    __syncwarp();
    int* out = src + (size_t)(base + qi) * stride;
    int written = 0;
    for (int r = 0; r < rounds; ++r) {
      const unsigned long long gmin = warp_min_u64(lmin);
      const int j = (int)(gmin & 0xffffffffu);
      if (lmin == gmin) {               // unique winner lane: retire the key and rescan its slice
        keys[j] = ~0ull;
        unsigned long long m = ~0ull;
        for (int jj = lane; jj < ng; jj += 32) {
          const unsigned long long kv = keys[jj];
          m = kv < m ? kv : m;
        }
        lmin = m;
      }
      if (j != qi && written < k) {
        if (lane == 0) out[written] = base + j;
        ++written;
      }
    }
    for (int w = written + lane; w < stride; w += 32) out[w] = -1;
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Incremental k-NN for the sampling loop.  Protein atoms never move (reference models/uni_transformer.py:205-206), so for a
// protein query the k+1 smallest keys among PROTEIN candidates are the same in every step: they are cached once per bound batch
// (sorted ascending, (k+1) keys per protein atom).  The exact per-step answer for such a query is then the k+1 smallest keys of
// {cached keys} U {keys of the graph's ligand atoms} -- any protein atom outside the cached set is beaten by k+1 protein atoms
// already.  With <= ~100 candidates the selection is done by rank counting (every lane reads all keys as shared-memory
// broadcasts) instead of k+1 serial arg-min rounds.  Ligand queries keep the full scan.  Keys, tie rule and output order are
// those of knn_kernel, so `src` is bit-identical (tests compare edge_index with the oracle).
// ---------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(KNN_WARPS * 32)
knn_protein_cache_kernel(const float4* __restrict__ xm, const int* __restrict__ node_ptr, const int* __restrict__ prot_ptr, int k, int max_ng,
                         unsigned long long* __restrict__ cache) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float4* spos = reinterpret_cast<float4*>(smem_raw);
  unsigned long long* skeys = reinterpret_cast<unsigned long long*>(spos + max_ng);
  const int g = blockIdx.x;
  const int base = node_ptr[g];
  const int np = prot_ptr[g + 1] - prot_ptr[g];            // protein atoms come first in a graph's node range
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = threadIdx.x; j < np; j += blockDim.x) spos[j] = xm[base + j];
  __syncthreads();
  unsigned long long* keys = skeys + (size_t)warp * max_ng;
  const int rounds = min(k + 1, np);
  for (int qi = blockIdx.y * KNN_WARPS + warp; qi < np; qi += gridDim.y * KNN_WARPS) {
    const float4 xq = spos[qi];
    unsigned long long lmin = ~0ull;
    for (int j = lane; j < np; j += 32) {
      const float4 xc = spos[j];
      const float dx = __fsub_rn(xq.x, xc.x), dy = __fsub_rn(xq.y, xc.y), dz = __fsub_rn(xq.z, xc.z);
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)j;
      keys[j] = key;
      lmin = key < lmin ? key : lmin;
    }
    __syncwarp();
    unsigned long long* out = cache + (size_t)(base + qi) * (k + 1);
    for (int r = 0; r < rounds; ++r) {
      const unsigned long long gmin = warp_min_u64(lmin);
      if (lmin == gmin) {
        keys[(int)(gmin & 0xffffffffu)] = ~0ull;
        unsigned long long m = ~0ull;
        for (int jj = lane; jj < np; jj += 32) {
          const unsigned long long kv = keys[jj];
          m = kv < m ? kv : m;
        }
        lmin = m;
      }
      if (lane == 0) out[r] = gmin;
    }
    for (int w = rounds + lane; w < k + 1; w += 32) out[w] = ~0ull;
    __syncwarp();
  }
}

__global__ void __launch_bounds__(KNN_WARPS * 32)
knn_update_kernel(const float4* __restrict__ xm, const int* __restrict__ node_ptr, const int* __restrict__ prot_ptr, int k, int stride, int hybrid,
                  int max_ng, const unsigned long long* __restrict__ cache, int* __restrict__ src) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float4* spos = reinterpret_cast<float4*>(smem_raw);
  unsigned long long* skeys = reinterpret_cast<unsigned long long*>(spos + max_ng);
  const int g = blockIdx.x;
  const int base = node_ptr[g];
  const int ng = node_ptr[g + 1] - base;
  const int np = prot_ptr[g + 1] - prot_ptr[g];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = threadIdx.x; j < ng; j += blockDim.x) spos[j] = xm[base + j];
  __syncthreads();
  unsigned long long* keys = skeys + (size_t)warp * max_ng;
  for (int qi = blockIdx.y * KNN_WARPS + warp; qi < ng; qi += gridDim.y * KNN_WARPS) {
    const float4 xq = spos[qi];
    int* out = src + (size_t)(base + qi) * stride;
    if (qi >= np && hybrid) {
      hybrid_ligand_row(spos, keys, qi, np, ng, k, stride, base, lane, out);
      continue;
    }
    if (qi < np) {
      // ---- protein query: cached protein keys + this step's ligand keys, selection by rank counting
      const int m = min(k + 1, np), n = m + (ng - np);
      const unsigned long long* crow = cache + (size_t)(base + qi) * (k + 1);
      for (int j = lane; j < m; j += 32) keys[j] = crow[j];
      for (int j = np + lane; j < ng; j += 32) {
        const float4 xc = spos[j];
        const float dx = __fsub_rn(xq.x, xc.x), dy = __fsub_rn(xq.y, xc.y), dz = __fsub_rn(xq.z, xc.z);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        keys[m + (j - np)] = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)j;
      }
      __syncwarp();
      const unsigned long long self = (unsigned long long)(unsigned)qi;          // d2 = 0 -> key = qi
      const int top = min(k + 1, n);
      for (int e0 = 0; e0 < n; e0 += 64) {                                         // two candidates per lane and pass
        const int ea = e0 + lane, eb = e0 + 32 + lane;
        const unsigned long long ka = ea < n ? keys[ea] : ~0ull, kb = eb < n ? keys[eb] : ~0ull;
        int ra = 0, rb = 0, rs = 0;
        for (int j = 0; j < n; ++j) {
          const unsigned long long kj = keys[j];                                   // broadcast read
          ra += kj < ka; rb += kj < kb; rs += kj < self;
        }
        // canonical rule: the k+1 smallest keys, self removed, first k kept
        if (ea < n && ra < top && ka != self) {
          const int pos = ra - (rs < ra ? 1 : 0);
          if (pos < k) out[pos] = base + (int)(ka & 0xffffffffu);
        }
        if (eb < n && rb < top && kb != self) {
          const int pos = rb - (rs < rb ? 1 : 0);
          if (pos < k) out[pos] = base + (int)(kb & 0xffffffffu);
        }
        if (e0 == 0) {
          int written = top - (rs < top ? 1 : 0);                                   // self is always a candidate (cached at d2 = 0)
          if (written > k) written = k;
          for (int w = written + lane; w < stride; w += 32) out[w] = -1;
        }
      }
      __syncwarp();
      continue;
    }
    // ---- ligand query: full scan of the graph (same procedure as knn_kernel)
    const int rounds = min(k + 1, ng);
    unsigned long long lmin = ~0ull;
    for (int j = lane; j < ng; j += 32) {
      const float4 xc = spos[j];
      const float dx = __fsub_rn(xq.x, xc.x), dy = __fsub_rn(xq.y, xc.y), dz = __fsub_rn(xq.z, xc.z);
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)j;
      keys[j] = key;
      lmin = key < lmin ? key : lmin;
    }
    __syncwarp();
    int written = 0;
    for (int r = 0; r < rounds; ++r) {
      const unsigned long long gmin = warp_min_u64(lmin);
      const int j = (int)(gmin & 0xffffffffu);
      if (lmin == gmin) {
        keys[j] = ~0ull;
        unsigned long long mm = ~0ull;
        for (int jj = lane; jj < ng; jj += 32) {
          const unsigned long long kv = keys[jj];
          mm = kv < mm ? kv : mm;
        }
        lmin = mm;
      }
      if (j != qi && written < k) {
        if (lane == 0) out[written] = base + j;
        ++written;
      }
    }
    for (int w = written + lane; w < stride; w += 32) out[w] = -1;
    __syncwarp();
  }
}

static void knn_grid(int n_graphs, int max_ng, dim3& grid, size_t& smem) {
  smem = (size_t)max_ng * sizeof(float4) + (size_t)KNN_WARPS * max_ng * sizeof(unsigned long long);
  int chunks = (max_ng + KNN_WARPS * 8 - 1) / (KNN_WARPS * 8);
  if (chunks < 1) chunks = 1;
  if ((long long)n_graphs * chunks > 65535LL * 8) chunks = 1;
  grid = dim3(n_graphs, chunks);
}

void td_launch_knn_cache(const float4* xm, const int* node_ptr, const int* prot_ptr, int n_graphs, int max_ng, int k, unsigned long long* cache,
                         cudaStream_t st) {
  if (n_graphs <= 0) return;
  dim3 grid; size_t smem;
  knn_grid(n_graphs, max_ng, grid, smem);
  static size_t opted[TD_MAX_DEVICES] = {0};
  if (smem > 48 * 1024) td_opt_in_smem(knn_protein_cache_kernel, smem, opted);
  knn_protein_cache_kernel<<<grid, KNN_WARPS * 32, smem, st>>>(xm, node_ptr, prot_ptr, k, max_ng, cache);
}

void td_launch_knn_update(const float4* xm, const int* node_ptr, const int* prot_ptr, int n_graphs, int max_ng, int k, int stride, int hybrid,
                          const unsigned long long* cache, int* src, cudaStream_t st) {
  if (n_graphs <= 0) return;
  dim3 grid; size_t smem;
  knn_grid(n_graphs, max_ng, grid, smem);
  static size_t opted[TD_MAX_DEVICES] = {0};
  if (smem > 48 * 1024) td_opt_in_smem(knn_update_kernel, smem, opted);
  knn_update_kernel<<<grid, KNN_WARPS * 32, smem, st>>>(xm, node_ptr, prot_ptr, k, stride, hybrid, max_ng, cache, src);
}

void td_launch_knn(const float4* xm, const int* node_ptr, const int* prot_ptr, int n_graphs, int max_ng, int k, int stride, int hybrid, int* src,
                   cudaStream_t st) {
  if (n_graphs <= 0) return;
  size_t smem = (size_t)max_ng * sizeof(float4) + (size_t)KNN_WARPS * max_ng * sizeof(unsigned long long);
  static size_t opted[TD_MAX_DEVICES] = {0};
  if (smem > 48 * 1024) td_opt_in_smem(knn_kernel, smem, opted);
  // enough chunks that small batches still fill the 148 SMs; each chunk re-stages the coordinates (cheap)
  int chunks = (max_ng + KNN_WARPS * 8 - 1) / (KNN_WARPS * 8);
  if (chunks < 1) chunks = 1;
  if ((long long)n_graphs * chunks > 65535LL * 8) chunks = 1;
  dim3 grid(n_graphs, chunks);
  knn_kernel<<<grid, KNN_WARPS * 32, smem, st>>>(xm, node_ptr, prot_ptr, k, stride, hybrid, max_ng, src);
}
