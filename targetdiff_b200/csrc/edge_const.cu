// edge_const.cu -- per-forward edge constants: 4-way edge type and the global edge gate e_w.
//
// Replaces (reference models/uni_transformer.py): _build_edge_type (:288-299) and the ew_net_type='global' gate
// e_w = sigmoid(MLP(20->128->1)(GaussianSmearing(|x_dst - x_src|)))  (:312-316), both evaluated once per forward on
// the forward's input coordinates and shared by all layers.
// One warp per edge slot; the 20->128 first layer lives in shared memory (k-major), LayerNorm by warp shuffles.
#include "tdiff_common.cuh"

#define EC_WARPS 8

// Phase 1, one warp per destination node.  `src_prev` (optional) is the neighbour list of the previous forward on the same batch: a
// node whose list is unchanged and that neither is a ligand atom nor has one among its neighbours keeps its edge types / gates
// (protein atoms never move, reference models/uni_transformer.py:205-206, so those edges' lengths are step-invariant).  All other
// nodes go to `work_list`; their edges are evaluated by edge_gate_kernel (phase 2), one warp per edge, so that the heavy part is
// load-balanced over the whole GPU instead of sitting in the few warps that happen to own ligand neighbourhoods.
__global__ void __launch_bounds__(EC_WARPS * 32)
edge_touch_kernel(const float4* __restrict__ xm, const int* __restrict__ src, int* __restrict__ src_prev, int have_prev, int n_nodes, int k,
                  unsigned char* __restrict__ rel_flag, unsigned char* __restrict__ touch_flag, unsigned char* __restrict__ etype,
                  int* __restrict__ work_list, int* __restrict__ n_work) {
  const int lane = threadIdx.x & 31;
  const int warp0 = blockIdx.x * EC_WARPS + (threadIdx.x >> 5), nwarps = gridDim.x * EC_WARPS;
  for (int node = warp0; node < n_nodes; node += nwarps) {
    const size_t e0 = (size_t)node * k;
    const float4 xd = xm[node];
    bool same = have_prev != 0, touch = xd.w != 0.0f;
    unsigned keep_mask = 0;          // bit j/32: slot j keeps its edge type and gate (same protein neighbour as in the previous forward)
    for (int j = lane; j < k; j += 32) {
      const int s = src[e0 + j];
      bool slot_same = false;
      if (src_prev) {
        slot_same = have_prev != 0 && src_prev[e0 + j] == s;
        same = same && slot_same;
        src_prev[e0 + j] = s;
      }
      const bool s_lig = s >= 0 && xm[s].w != 0.0f;
      if (slot_same && !s_lig && xd.w == 0.0f) keep_mask |= 1u << (j >> 5);
      touch = touch || s_lig;
      // "relevant" nodes = ligand atoms and their neighbours: the only rows the h2x sub-layers (and the last x2h) need
      if (rel_flag && xd.w != 0.0f && s >= 0) rel_flag[s] = 1;
    }
    if (rel_flag && xd.w != 0.0f && lane == 0) rel_flag[node] = 1;
    same = __all_sync(0xffffffffu, same);
    touch = __any_sync(0xffffffffu, touch);
    // "touched" = ligand atom or node with a ligand atom among its neighbours: the nodes whose features after the first x2h differ
    // from their ligand-free values (engine.cu, ligand-free cache)
    if (touch_flag && lane == 0) touch_flag[node] = touch ? 1 : 0;
    if (same && !touch) continue;
    // the node's edges are re-evaluated by edge_gate_kernel, except slots that still hold the same PROTEIN neighbour of a protein node:
    // neither atom moves (reference models/uni_transformer.py:205-206), so their type and gate are unchanged -- marked with bit 7
    if (etype)
      for (int j = lane; j < k; j += 32)
        if (keep_mask & (1u << (j >> 5))) etype[e0 + j] |= 0x80;
    if (lane == 0) work_list[atomicAdd(n_work, 1)] = node;
  }
}

// Phase 2, one warp per edge of the listed nodes: edge type and gate e_w = sigmoid(MLP(gaussians(|x_dst - x_src|))).
__global__ void __launch_bounds__(EC_WARPS * 32)
edge_gate_kernel(const float4* __restrict__ xm, const int* __restrict__ src, const int* __restrict__ work_list, const int* __restrict__ n_work,
                 int k, const float* __restrict__ offsets, float coeff, const float* __restrict__ w1t, const float* __restrict__ b1,
                 const float* __restrict__ ln_g, const float* __restrict__ ln_b, const float* __restrict__ w2, float b2,
                 unsigned char* __restrict__ etype, float* __restrict__ e_w, int gate_mode, int honour_keep) {
  __shared__ float s_w1t[TD_NG * TD_H];
  __shared__ float s_b1[TD_H], s_g[TD_H], s_b[TD_H], s_w2[TD_H];
  for (int i = threadIdx.x; i < TD_NG * TD_H; i += blockDim.x) s_w1t[i] = w1t[i];
  for (int i = threadIdx.x; i < TD_H; i += blockDim.x) {
    s_b1[i] = b1[i]; s_g[i] = ln_g[i]; s_b[i] = ln_b[i]; s_w2[i] = w2[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const float mu = offsets[lane < TD_NG ? lane : 0];
  const long long warp0 = (long long)blockIdx.x * EC_WARPS + (threadIdx.x >> 5), nwarps = (long long)gridDim.x * EC_WARPS;
  const long long n_items = (long long)(*n_work) * k;
  for (long long item = warp0; item < n_items; item += nwarps) {
    const int node = work_list[item / k];
    const size_t e = (size_t)node * k + (size_t)(item % k);
    const unsigned char keep = honour_keep ? etype[e] : 0;      // first forward of a batch: `etype` holds no marks yet (and no valid types)
    if (keep & 0x80) {               // unchanged protein-protein slot (edge_touch_kernel): keep type and gate, clear the mark
      if (lane == 0) etype[e] = keep & 0x7f;
      continue;
    }
    const int s = src[e];
    if (s < 0) {
      if (lane == 0) { etype[e] = 3; e_w[e] = 0.0f; }
      continue;
    }
    const float4 xd = xm[node], xs = xm[s];
    if (gate_mode != 0) {            // ew_net_type 'r' / 'm' / 'none': no global gate, only the edge type (the slot's gate defaults to 1)
      if (lane == 0) {
        const bool ns = xs.w != 0.0f, nd = xd.w != 0.0f;
        etype[e] = (unsigned char)(ns ? (nd ? 0 : 1) : (nd ? 2 : 3));
        e_w[e] = 1.0f;
      }
      continue;
    }
    const float dx = xd.x - xs.x, dy = xd.y - xs.y, dz = xd.z - xs.z;
    const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
    const float t = dist - mu;
    const float gj = expf(coeff * (t * t));
    float p[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) p[c] = s_b1[lane + 32 * c];
#pragma unroll
    for (int jj = 0; jj < TD_NG; ++jj) {
      const float g = __shfl_sync(0xffffffffu, gj, jj);
#pragma unroll
      for (int c = 0; c < 4; ++c) p[c] = fmaf(g, s_w1t[jj * TD_H + lane + 32 * c], p[c]);
    }
    ln_relu_128(p, s_g, s_b, lane);
    float acc = (p[0] * s_w2[lane] + p[1] * s_w2[lane + 32]) + (p[2] * s_w2[lane + 64] + p[3] * s_w2[lane + 96]);
    acc = warp_sum(acc) + b2;
    if (lane == 0) {
      const bool ns = xs.w != 0.0f, nd = xd.w != 0.0f;
      const int ty = ns ? (nd ? 0 : 1) : (nd ? 2 : 3);
      etype[e] = (unsigned char)ty;
      e_w[e] = 1.0f / (1.0f + expf(-acc));
    }
  }
}

void td_launch_edge_const(const float4* xm, const int* src, int* src_prev, int have_prev, int n_nodes, int k, const float* offsets, float coeff,
                          const float* w1t, const float* b1, const float* ln_g, const float* ln_b, const float* w2, float b2,
                          unsigned char* etype, float* e_w, unsigned char* rel_flag, unsigned char* touch_flag, int* work_list, int* n_work,
                          int gate_mode, cudaStream_t st) {
  if (n_nodes == 0) return;
  int blocks = (n_nodes + EC_WARPS - 1) / EC_WARPS;
  if (blocks > 148 * 8) blocks = 148 * 8;
  if (rel_flag) cudaMemsetAsync(rel_flag, 0, (size_t)n_nodes, st);
  cudaMemsetAsync(n_work, 0, sizeof(int), st);
  // gate_mode bit 0: no global gate (ew_net_type r / m / none); bit 1: developer switch, re-evaluate every slot of a listed node
  edge_touch_kernel<<<blocks, EC_WARPS * 32, 0, st>>>(xm, src, src_prev, have_prev, n_nodes, k, rel_flag, touch_flag, (gate_mode & 2) ? nullptr : etype,
                                                      work_list, n_work);
  edge_gate_kernel<<<148 * 8, EC_WARPS * 32, 0, st>>>(xm, src, work_list, n_work, k, offsets, coeff, w1t, b1, ln_g, ln_b, w2, b2, etype, e_w, gate_mode & 1,
                                                     (have_prev && !(gate_mode & 2)) ? 1 : 0);
}

// Per-layer edge length |x_dst - x_src| (reference models/uni_transformer.py:188-189) for every slot, from the layer's input
// coordinates; consumed by the tensor-core edge-MLP producers so that their metadata loads are plain coalesced streams.
// ew_net_type 'r' (:58-59,121-122): the two sub-layers' gates sigmoid(Linear(r_feat)) are evaluated here too -- r_feat is the
// (edge type one-hot) x (20 gaussians) outer product, so Linear(r_feat) = b + sum_j w[20 type + j] g_j(dist).
__global__ void edge_geom_kernel(const float4* __restrict__ xm, const int* __restrict__ src, const unsigned char* __restrict__ etype, long long n_slots,
                                 int k, float* __restrict__ dist, TdEwR ew) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_slots) return;
  const int s = src[e];
  float d = 0.0f;
  if (s >= 0) {
    const float4 xd = xm[e / k], xs = xm[s];
    const float dx = xd.x - xs.x, dy = xd.y - xs.y, dz = xd.z - xs.z;
    d = sqrtf(dx * dx + dy * dy + dz * dz);
  }
  dist[e] = d;
  if (ew.w_x2h) {
    float ax = ew.b_x2h, ah = ew.b_h2x;
    if (s >= 0) {
      const int ty = etype[e];
#pragma unroll 4
      for (int j = 0; j < TD_NG; ++j) {
        const float t = d - ew.offsets[j];
        const float g = expf(ew.coeff * (t * t));
        ax = fmaf(g, ew.w_x2h[ty * TD_NG + j], ax);
        ah = fmaf(g, ew.w_h2x[ty * TD_NG + j], ah);
      }
    }
    ew.out_x2h[e] = s >= 0 ? 1.0f / (1.0f + expf(-ax)) : 0.0f;
    ew.out_h2x[e] = s >= 0 ? 1.0f / (1.0f + expf(-ah)) : 0.0f;
  }
}

void td_launch_edge_geom(const float4* xm, const int* src, const unsigned char* etype, int n_nodes, int k, float* dist, const TdEwR& ew, cudaStream_t st) {
  const long long n = (long long)n_nodes * k;
  if (n > 0) edge_geom_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(xm, src, etype, n, k, dist, ew);
}

// Edge lengths of the slots of a list of destination rows (the ligand atoms), from the current coordinates, and optionally one 'r'
// gate set sigmoid(b + sum_j w[20 type + j] g_j(dist)) for them: the reference recomputes rel_x / dist after every h2x sub-layer
// (models/uni_transformer.py:207-208) and each h2x sub-layer has its own ew_net (:121-122).  Same arithmetic as edge_geom_kernel.
__global__ void edge_geom_rows_kernel(const float4* __restrict__ xm, const int* __restrict__ src, const unsigned char* __restrict__ etype,
                                      const int* __restrict__ rows, long long n_slots, int k, float* __restrict__ dist,
                                      const float* __restrict__ gate_w, float gate_b, const float* __restrict__ offsets, float coeff,
                                      float* __restrict__ gate) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_slots) return;
  const long long e = (long long)rows[t / k] * k + t % k;
  const int s = src[e];
  float d = 0.0f;
  if (s >= 0) {
    const float4 xd = xm[e / k], xs = xm[s];
    const float dx = xd.x - xs.x, dy = xd.y - xs.y, dz = xd.z - xs.z;
    d = sqrtf(dx * dx + dy * dy + dz * dz);
  }
  dist[e] = d;
  if (gate_w) {
    float a = gate_b;
    if (s >= 0) {
      const int ty = etype[e];
#pragma unroll 4
      for (int j = 0; j < TD_NG; ++j) {
        const float u = d - offsets[j];
        a = fmaf(expf(coeff * (u * u)), gate_w[ty * TD_NG + j], a);
      }
    }
    gate[e] = s >= 0 ? 1.0f / (1.0f + expf(-a)) : 0.0f;
  }
}

void td_launch_edge_geom_rows(const float4* xm, const int* src, const unsigned char* etype, const int* rows, int n_rows, int k, float* dist,
                              const float* gate_w, float gate_b, const float* offsets, float coeff, float* gate, cudaStream_t st) {
  const long long n = (long long)n_rows * k;
  if (n > 0) edge_geom_rows_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(xm, src, etype, rows, n, k, dist, gate_w, gate_b, offsets, coeff, gate);
}

// Compact the relevant-node flags into a list (order irrelevant: every row is processed independently); consumers bound by *n_rel.
__global__ void rel_compact_kernel(const unsigned char* __restrict__ flag, int n_nodes, int* __restrict__ rel_list, int* __restrict__ n_rel) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_nodes && flag[i]) rel_list[atomicAdd(n_rel, 1)] = i;
}
void td_launch_rel_compact(const unsigned char* flag, int n_nodes, int* rel_list, int* n_rel, cudaStream_t st) {
  if (n_nodes == 0) return;
  cudaMemsetAsync(n_rel, 0, sizeof(int), st);
  rel_compact_kernel<<<(n_nodes + 255) / 256, 256, 0, st>>>(flag, n_nodes, rel_list, n_rel);
}

// Class-sorted list of the dirty destinations of one x2h evaluation for the v4 edge kernel (ligand-free cache): the flagged PROTEIN nodes,
// padded with -1 to a multiple of `pad`, followed by the (already padded) list of all ligand nodes.  counts = {entries, protein part}.
__global__ void rel_rows_protein_kernel(const unsigned char* __restrict__ flag, const float4* __restrict__ xm, int n_nodes, int* __restrict__ rel_rows,
                                        int* __restrict__ rel_counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_nodes && flag[i] && xm[i].w == 0.0f) rel_rows[atomicAdd(&rel_counts[2], 1)] = i;
}
// list blockIdx.y (at rows + y * stride, counts + 4 y): its protein part (counts[2] entries) is written; pad it and append the ligand list
__global__ void rel_rows_finish_kernel(const int* __restrict__ lig_rows, int n_lig_rows, int pad, int* __restrict__ rows, long long stride,
                                       int* __restrict__ counts) {
  int* rel_rows = rows + (size_t)blockIdx.y * stride;
  int* rel_counts = counts + 4 * blockIdx.y;
  const int n_p = rel_counts[2], n_pp = (n_p + pad - 1) / pad * pad;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_pp - n_p) rel_rows[n_p + i] = -1;
  if (i < n_lig_rows) rel_rows[n_pp + i] = lig_rows[i];
  if (i == 0) { rel_counts[0] = n_pp + n_lig_rows; rel_counts[1] = n_pp; }
}
void td_launch_rel_rows(const unsigned char* rel_flag, const float4* xm, int n_nodes, const int* lig_rows, int n_lig_rows, int pad, int* rel_rows,
                        int* rel_counts, cudaStream_t st) {
  cudaMemsetAsync(rel_counts, 0, 4 * sizeof(int), st);
  if (n_nodes > 0) rel_rows_protein_kernel<<<(n_nodes + 255) / 256, 256, 0, st>>>(rel_flag, xm, n_nodes, rel_rows, rel_counts);
  const int n = n_lig_rows > pad ? n_lig_rows : pad;
  rel_rows_finish_kernel<<<(n + 255) / 256, 256, 0, st>>>(lig_rows, n_lig_rows, pad, rel_rows, 0, rel_counts);
}

// ---- backward cone of the sampling loop's last block (engine.cu).  A sampling step reads only the ligand rows of the network's output
// (type head) and the h2x sub-layers read h only on the relevant nodes R (ligand atoms and their neighbours).  x2h evaluation g of the
// block (G in all) reads h at its destinations and their sources, so it only needs the destinations
//   R_g = nodes within G - 1 - g hops of R, hops taken from a destination to its sources (R_{G-1} = R, R_{g-1} = R_g + src(R_g)),
// and its node GEMMs need the A blocks and q on R_g and the B blocks on R_{g-1}.  Rows outside these sets keep stale values.
// cone_lists_kernel, one CTA per graph (a graph's edges stay inside it): every node's hop distance from R in shared memory, then the
// protein nodes of 2 G lists, list t at rows + t * stride, its protein count in counts[4 t + 2]:
//   list 2 g      the destinations R_g of evaluation g (A blocks, q, edge MLPs), of those only the dirty ones for the first `n_dirty`
//                 (cached) evaluations;
//   list 2 g + 1  the nodes R_{g-1} (B blocks).
// rel_rows_finish_kernel then makes each a class-sorted list (every ligand atom is in every R_g and always dirty).  A graph's rows
// lie in the same order in both lists, so where R_g = R_{g-1} the two column groups of node_proj_kernel read the same h rows at about
// the same time.  Shared memory: the graph's distances (max_ng ints), then per list a counter and a base (4 G ints).
#define CONE_THREADS 512
__global__ void __launch_bounds__(CONE_THREADS)
cone_lists_kernel(const unsigned char* __restrict__ rel_flag, const int* __restrict__ src, const int* __restrict__ node_ptr,
                  const float4* __restrict__ xm, int n_nodes, int k, int G, int max_ng, const unsigned char* __restrict__ dirty, int n_dirty,
                  int* __restrict__ rows, long long stride, int* __restrict__ counts) {
  extern __shared__ int s_dist[];
  int* s_cnt = s_dist + max_ng;                  // [2 G]
  int* s_base = s_cnt + 2 * G;
  const int n0 = node_ptr[blockIdx.x], ng = node_ptr[blockIdx.x + 1] - n0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  constexpr int kFar = 1 << 30;
  for (int i = threadIdx.x; i < ng; i += blockDim.x) s_dist[i] = rel_flag[n0 + i] ? 0 : kFar;
  for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  // breadth-first rounds: round r gives the unvisited sources of the nodes at distance r distance r + 1.  Round r only writes r + 1, so a
  // node's `== r` test is stable (and warp-uniform) while other warps write.
  for (int r = 0; r < G; ++r) {
    bool grew = false;
    for (int i = warp; i < ng; i += nw) {
      if (s_dist[i] != r) continue;
      for (int j = lane; j < k; j += 32) {
        const int s = src[(size_t)(n0 + i) * k + j];
        if (s >= 0 && s_dist[s - n0] > r + 1) { s_dist[s - n0] = r + 1; grew = true; }
      }
    }
    if (!__syncthreads_or(grew)) break;
  }
  // two passes over the graph's nodes, 32 per warp: count every list's members, reserve the graph's ranges, write
  const unsigned lt = (1u << lane) - 1u;
  for (int pass = 0; pass < 2; ++pass) {
    for (int i0 = 32 * warp; i0 < ng; i0 += 32 * nw) {
      const int i = i0 + lane, n = n0 + i;
      const int d = i < ng ? s_dist[i] : kFar;
      const bool prot = i < ng && xm[n].w == 0.0f;
      for (int g = 0; g < G; ++g) {
        const bool a = prot && d <= G - 1 - g && (g >= n_dirty || dirty[(size_t)g * n_nodes + n]);
        const bool b = prot && d <= G - g;
        const unsigned ma = __ballot_sync(0xffffffffu, a), mb = __ballot_sync(0xffffffffu, b);
        int oa = 0, ob = 0;
        if (lane == 0) {
          if (ma) oa = atomicAdd(&s_cnt[2 * g], __popc(ma));
          if (mb) ob = atomicAdd(&s_cnt[2 * g + 1], __popc(mb));
        }
        if (pass == 0) continue;
        oa = __shfl_sync(0xffffffffu, oa, 0);
        ob = __shfl_sync(0xffffffffu, ob, 0);
        if (a) rows[(size_t)(2 * g) * stride + s_base[2 * g] + oa + __popc(ma & lt)] = n;
        if (b) rows[(size_t)(2 * g + 1) * stride + s_base[2 * g + 1] + ob + __popc(mb & lt)] = n;
      }
    }
    __syncthreads();
    if (pass == 0) {
      for (int t = threadIdx.x; t < 2 * G; t += blockDim.x) {
        s_base[t] = s_cnt[t] ? atomicAdd(&counts[4 * t + 2], s_cnt[t]) : 0;
        s_cnt[t] = 0;
      }
      __syncthreads();
    }
  }
}
void td_launch_cone_lists(const unsigned char* rel_flag, const int* src, const int* node_ptr, const float4* xm, int n_graphs, int max_ng, int n_nodes,
                          int k, int G, const unsigned char* dirty, int n_dirty, const int* lig_rows, int n_lig_rows, int pad, int* rows,
                          long long stride, int* counts, cudaStream_t st) {
  if (G <= 0) return;
  cudaMemsetAsync(counts, 0, (size_t)G * 8 * sizeof(int), st);
  const size_t smem = ((size_t)max_ng + 4 * (size_t)G) * sizeof(int);
  static size_t opted[TD_MAX_DEVICES] = {0};
  td_opt_in_smem(cone_lists_kernel, smem, opted);
  cone_lists_kernel<<<n_graphs, CONE_THREADS, smem, st>>>(rel_flag, src, node_ptr, xm, n_nodes, k, G, max_ng, dirty, n_dirty, rows, stride, counts);
  const int n = n_lig_rows > pad ? n_lig_rows : pad;
  rel_rows_finish_kernel<<<dim3((n + 255) / 256, 2 * G), 256, 0, st>>>(lig_rows, n_lig_rows, pad, rows, stride, counts);
}

// ---- ligand-free cache support (engine.cu): a node's features after x2h layer l equal their ligand-free values unless the node is
// "dirty": dirty_{l+1} = dirty_l  or  any neighbour in dirty_l   (dirty_1 = touched nodes, see edge_touch_kernel)
__global__ void dirty_propagate_kernel(const unsigned char* __restrict__ in, const int* __restrict__ src, int n_nodes, int k, unsigned char* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int node = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (node >= n_nodes) return;
  bool d = in[node] != 0;
  for (int j = lane; j < k && !d; j += 32) {
    const int s = src[(size_t)node * k + j];
    if (s >= 0 && in[s]) d = true;
  }
  d = __any_sync(0xffffffffu, d);
  if (lane == 0) out[node] = d ? 1 : 0;
}
void td_launch_dirty_propagate(const unsigned char* in, const int* src, int n_nodes, int k, unsigned char* out, cudaStream_t st) {
  if (n_nodes > 0) dirty_propagate_kernel<<<(n_nodes + 7) / 8, 256, 0, st>>>(in, src, n_nodes, k, out);
}
// clean protein nodes take their cached ligand-free features (one warp per node, 512 B rows)
__global__ void restore_clean_kernel(const unsigned char* __restrict__ dirty, const float4* __restrict__ xm, const float* __restrict__ h_free, int n_nodes,
                                     float* __restrict__ h) {
  const int lane = threadIdx.x & 31;
  const int node = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (node >= n_nodes || dirty[node] || xm[node].w != 0.0f) return;
  reinterpret_cast<float4*>(h + (size_t)node * TD_H)[lane] = reinterpret_cast<const float4*>(h_free + (size_t)node * TD_H)[lane];
}
void td_launch_restore_clean(const unsigned char* dirty, const float4* xm, const float* h_free, int n_nodes, float* h, cudaStream_t st) {
  if (n_nodes > 0) restore_clean_kernel<<<(n_nodes + 7) / 8, 256, 0, st>>>(dirty, xm, h_free, n_nodes, h);
}
