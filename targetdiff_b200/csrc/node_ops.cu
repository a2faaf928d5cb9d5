// node_ops.cu -- per-node work of one forward: embeddings, the node-side projections of the split first layers,
// the query MLPs, and the atom-type head.
//
// Reference lines restated: models/molopt_score_model.py:317-338 (embeddings + indicator column), :307-311,:352
// (v_inference head); models/uni_transformer.py:70,:132 (hq_func / xq_func); models/common.py:60-80 (MLP).
// The node projection is the exact first-layer split of SURVEY.md Appendix B:
//   W1 . [type | r_feat | h_dst | h_src] = W_t[:,type] + W_r . r_feat + (W_i h)[dst] + (W_j h)[src]
// so the two h-dependent terms become one dense [N,128] x [128,640] GEMM per sub-layer instead of per-edge work.
#include "tdiff_common.cuh"

// ---------------------------------------------------------------------------------------------- embeddings
__global__ void protein_embed_kernel(const float* __restrict__ feat, int n_protein, int fdim, const float* __restrict__ w,
                                     const float* __restrict__ b, const int* __restrict__ prot_node, float* __restrict__ h0) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n_protein * TD_H) return;
  const int p = (int)(i / TD_H), f = (int)(i % TD_H);
  float acc = 0.0f;
  if (f < TD_H - 1) {
    const float* fr = feat + (size_t)p * fdim;
    const float* wr = w + (size_t)f * fdim;
    for (int c = 0; c < fdim; ++c) acc = fmaf(fr[c], wr[c], acc);
    acc += b[f];
  }
  h0[(size_t)prot_node[p] * TD_H + f] = acc;     // indicator column (f == 127) = 0 for protein atoms
}

void td_launch_protein_embed(const float* feat, int n_protein, int fdim, const float* w, const float* b, const int* prot_node,
                             float* h0, cudaStream_t st) {
  if (n_protein == 0) return;
  long long n = (long long)n_protein * TD_H;
  protein_embed_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(feat, n_protein, fdim, w, b, prot_node, h0);
}

// h <- [protein: cached embedding | ligand: W_l[:, v] + b_l, indicator 1]; one float4 per thread.
__global__ void init_h_kernel(const float* __restrict__ h0, const float4* __restrict__ xm, const int* __restrict__ lig_v,
                              const int* __restrict__ node_lig, const float* __restrict__ wl_t, const float* __restrict__ bl,
                              const float* __restrict__ w_time, const float* __restrict__ time_norm, const int* __restrict__ lig_graph,
                              int n_nodes, float* __restrict__ h) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n_nodes * (TD_H / 4)) return;
  const int n = (int)(i / (TD_H / 4)), f4 = (int)(i % (TD_H / 4));
  float4 o;
  const int a = node_lig[n];
  if (a < 0) {
    o = *reinterpret_cast<const float4*>(h0 + (size_t)n * TD_H + 4 * f4);
  } else {
    const int v = lig_v[a];
    const float4 wv = *reinterpret_cast<const float4*>(wl_t + (size_t)v * TD_H + 4 * f4);
    const float4 bv = *reinterpret_cast<const float4*>(bl + 4 * f4);
    o.x = wv.x + bv.x; o.y = wv.y + bv.y; o.z = wv.z + bv.z; o.w = wv.w + bv.w;
    if (w_time) {                                // time_emb_mode 'simple': extra input column time_step / T (models/molopt_score_model.py:319-324)
      const float tn = time_norm[lig_graph[a]];
      const float4 wt = *reinterpret_cast<const float4*>(w_time + 4 * f4);
      o.x = fmaf(wt.x, tn, o.x); o.y = fmaf(wt.y, tn, o.y); o.z = fmaf(wt.z, tn, o.z); o.w = fmaf(wt.w, tn, o.w);
    }
    if (f4 == TD_H / 4 - 1) o.w = 1.0f;          // node_indicator column
  }
  *reinterpret_cast<float4*>(h + (size_t)n * TD_H + 4 * f4) = o;
}

void td_launch_init_h(const float* h0, const float4* xm, const int* lig_v, const int* node_lig, const float* wl_t, const float* bl,
                      const float* w_time, const float* time_norm, const int* lig_graph, int n_nodes, float* h, cudaStream_t st) {
  if (n_nodes == 0) return;
  long long n = (long long)n_nodes * (TD_H / 4);
  init_h_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(h0, xm, lig_v, node_lig, wl_t, bl, w_time, time_norm, lig_graph, n_nodes, h);
}

// out = a + b (x2h_out_fc glue: sum of the two halves of the node_output first Linear; residual add)
__global__ void add_rows_kernel(const float4* __restrict__ a, const float4* __restrict__ b, float4* __restrict__ out, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 x = a[i], y = b[i];
  out[i] = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
}
void td_launch_add_rows(const float* a, const float* b, float* out, long long n_floats, cudaStream_t st) {
  const long long n4 = n_floats / 4;
  if (n4 > 0) add_rows_kernel<<<(int)((n4 + 255) / 256), 256, 0, st>>>((const float4*)a, (const float4*)b, (float4*)out, n4);
}

// sampling loop, time embedding: every graph is at time step t_start - *step  ->  time_norm = t / T (fp32 division like the reference)
__global__ void set_time_kernel(const int* __restrict__ step, int t_start, int n_timesteps, int n_graphs, float* __restrict__ time_norm) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_graphs) time_norm[g] = (float)(t_start - *step) / (float)n_timesteps;
}
void td_launch_set_time(const int* step, int t_start, int n_timesteps, int n_graphs, float* time_norm, cudaStream_t st) {
  if (n_graphs > 0) set_time_kernel<<<(n_graphs + 255) / 256, 256, 0, st>>>(step, t_start, n_timesteps, n_graphs, time_norm);
}
// respaced chain: every graph is at time step time_seq[step]
__global__ void set_time_seq_kernel(const int* __restrict__ step, const int* __restrict__ time_seq, int n_timesteps, int n_graphs,
                                    float* __restrict__ time_norm) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_graphs) time_norm[g] = (float)time_seq[*step] / (float)n_timesteps;
}
void td_launch_set_time_seq(const int* step, const int* time_seq, int n_timesteps, int n_graphs, float* time_norm, cudaStream_t st) {
  if (n_graphs > 0) set_time_seq_kernel<<<(n_graphs + 255) / 256, 256, 0, st>>>(step, time_seq, n_timesteps, n_graphs, time_norm);
}

// ---------------------------------------------------------------------------------------------- node projection
// P[N,640] = h[N,128] . wn_t[128][640] + bn ; CTA tile 128 rows x 128 columns.
__global__ void __launch_bounds__(TD_GEMM_THREADS, 1)
node_proj_kernel(const float* __restrict__ h, int n_nodes, const float* __restrict__ wn_t, const float* __restrict__ bn,
                 float* __restrict__ P) {
  extern __shared__ __align__(16) float smem[];
  float* As = smem;                      // [128][TD_LDA]
  float* Bs = smem + 128 * TD_LDA;       // [128][128]
  const int row0 = blockIdx.x * 128, col0 = blockIdx.y * 128;
  const int tid = threadIdx.x;
  for (int i = tid; i < 128 * 32; i += TD_GEMM_THREADS) {
    const int r = i >> 5, c4 = i & 31;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < n_nodes) v = *reinterpret_cast<const float4*>(h + (size_t)(row0 + r) * TD_H + 4 * c4);
    *reinterpret_cast<float4*>(As + r * TD_LDA + 4 * c4) = v;
    *reinterpret_cast<float4*>(Bs + r * 128 + 4 * c4) = *reinterpret_cast<const float4*>(wn_t + (size_t)r * TD_NPROJ + col0 + 4 * c4);
  }
  __syncthreads();
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][8];
  tile_gemm_128(As, Bs, acc, ty, tx);
  const float4 bia0 = *reinterpret_cast<const float4*>(bn + col0 + 4 * tx);
  const float4 bia1 = *reinterpret_cast<const float4*>(bn + col0 + 64 + 4 * tx);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = row0 + ty + 32 * i;
    if (r < n_nodes) {
      float* o = P + (size_t)r * TD_NPROJ + col0;
      *reinterpret_cast<float4*>(o + 4 * tx) = make_float4(acc[i][0] + bia0.x, acc[i][1] + bia0.y, acc[i][2] + bia0.z, acc[i][3] + bia0.w);
      *reinterpret_cast<float4*>(o + 64 + 4 * tx) = make_float4(acc[i][4] + bia1.x, acc[i][5] + bia1.y, acc[i][6] + bia1.z, acc[i][7] + bia1.w);
    }
  }
}

void td_launch_node_proj(const float* h, int n_nodes, const float* wn_t, const float* bn, float* P, cudaStream_t st) {
  if (n_nodes == 0) return;
  const size_t smem = (size_t)(128 * TD_LDA + 128 * 128) * sizeof(float);
  static size_t opted[TD_MAX_DEVICES] = {0};
  td_opt_in_smem(node_proj_kernel, smem, opted);
  dim3 grid((n_nodes + 127) / 128, TD_NPROJ / 128);
  node_proj_kernel<<<grid, TD_GEMM_THREADS, smem, st>>>(h, n_nodes, wn_t, bn, P);
}

// ---------------------------------------------------------------------------------------------- query MLP tail
// q = relu(LN(P[:, 512:640])) . W2^T + b2    (first Linear already inside the node projection)
__global__ void __launch_bounds__(TD_GEMM_THREADS, 1)
node_q_kernel(const float* __restrict__ P, int n_nodes, TdMlp q, float* __restrict__ qout) {
  extern __shared__ __align__(16) float smem[];
  float* As = smem;
  float* Bs = smem + 128 * TD_LDA;
  const int row0 = blockIdx.x * 128;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 128 * 32; i += TD_GEMM_THREADS)
    *reinterpret_cast<float4*>(Bs + 4 * i) = *reinterpret_cast<const float4*>(q.w2t + 4 * i);
  for (int r = warp; r < 128; r += TD_GEMM_THREADS / 32) {
    float p[4] = {0.f, 0.f, 0.f, 0.f};
    if (row0 + r < n_nodes) {
      const float* pr = P + (size_t)(row0 + r) * TD_NPROJ + 512;
#pragma unroll
      for (int c = 0; c < 4; ++c) p[c] = pr[lane + 32 * c];
      ln_relu_128(p, q.ln_g, q.ln_b, lane);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) As[r * TD_LDA + lane + 32 * c] = p[c];
  }
  __syncthreads();
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][8];
  tile_gemm_128(As, Bs, acc, ty, tx);
  const float4 bia0 = *reinterpret_cast<const float4*>(q.b2 + 4 * tx);
  const float4 bia1 = *reinterpret_cast<const float4*>(q.b2 + 64 + 4 * tx);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = row0 + ty + 32 * i;
    if (r < n_nodes) {
      float* o = qout + (size_t)r * TD_H;
      *reinterpret_cast<float4*>(o + 4 * tx) = make_float4(acc[i][0] + bia0.x, acc[i][1] + bia0.y, acc[i][2] + bia0.z, acc[i][3] + bia0.w);
      *reinterpret_cast<float4*>(o + 64 + 4 * tx) = make_float4(acc[i][4] + bia1.x, acc[i][5] + bia1.y, acc[i][6] + bia1.z, acc[i][7] + bia1.w);
    }
  }
}

void td_launch_node_q(const float* P, int n_nodes, TdMlp q, float* qout, cudaStream_t st) {
  if (n_nodes == 0) return;
  const size_t smem = (size_t)(128 * TD_LDA + 128 * 128) * sizeof(float);
  static size_t opted[TD_MAX_DEVICES] = {0};
  td_opt_in_smem(node_q_kernel, smem, opted);
  node_q_kernel<<<(n_nodes + 127) / 128, TD_GEMM_THREADS, smem, st>>>(P, n_nodes, q, qout);
}

// ---------------------------------------------------------------------------------------------- atom-type head
// logits = W2 (softplus(W1 h + b1) - ln 2) + b2 for ligand atoms; one warp per atom, W1^T in shared memory.
#define HEAD_WARPS 8
__global__ void __launch_bounds__(HEAD_WARPS * 32)
head_kernel(const float* __restrict__ h, const int* __restrict__ lig_node, int n_lig, const float* __restrict__ w1t,
            const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2, int n_classes,
            float* __restrict__ logits) {
  extern __shared__ __align__(16) float smem[];
  float* s_w1t = smem;                          // [128][128]
  float* s_h = smem + 128 * 128;                // [HEAD_WARPS][128]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 128 * 32; i += blockDim.x)
    *reinterpret_cast<float4*>(s_w1t + 4 * i) = *reinterpret_cast<const float4*>(w1t + 4 * i);
  __syncthreads();
  float* hs = s_h + warp * TD_H;
  for (int a = blockIdx.x * HEAD_WARPS + warp; a < n_lig; a += gridDim.x * HEAD_WARPS) {
    const float* hr = h + (size_t)lig_node[a] * TD_H;
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 4; ++c) hs[lane + 32 * c] = hr[lane + 32 * c];
    __syncwarp();
    float y[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) y[c] = 0.0f;
    for (int kk = 0; kk < TD_H; ++kk) {
      const float hv = hs[kk];
#pragma unroll
      for (int c = 0; c < 4; ++c) y[c] = fmaf(hv, s_w1t[kk * TD_H + lane + 32 * c], y[c]);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float z = y[c] + b1[lane + 32 * c];
      const float sp = z > 20.0f ? z : log1pf(expf(z));        // F.softplus (beta=1, threshold=20)
      y[c] = sp - 0.6931471824645996f;                         // ShiftedSoftplus: fp32 log 2 (models/common.py:156-162)
    }
    for (int cls = 0; cls < n_classes; ++cls) {
      const float* wr = w2 + (size_t)cls * TD_H;
      float acc = (y[0] * wr[lane] + y[1] * wr[lane + 32]) + (y[2] * wr[lane + 64] + y[3] * wr[lane + 96]);
      acc = warp_sum(acc);
      if (lane == 0) logits[(size_t)a * n_classes + cls] = acc + b2[cls];
    }
  }
}

void td_launch_head(const float* h, const int* lig_node, int n_lig, const float* w1t, const float* b1, const float* w2, const float* b2,
                    int n_classes, float* logits, cudaStream_t st) {
  if (n_lig == 0) return;
  const size_t smem = (size_t)(128 * 128 + HEAD_WARPS * TD_H) * sizeof(float);
  static size_t opted[TD_MAX_DEVICES] = {0};
  td_opt_in_smem(head_kernel, smem, opted);
  int blocks = (n_lig + HEAD_WARPS - 1) / HEAD_WARPS;
  if (blocks > 148 * 2) blocks = 148 * 2;
  head_kernel<<<blocks, HEAD_WARPS * 32, smem, st>>>(h, lig_node, n_lig, w1t, b1, w2, b2, n_classes, logits);
}
