// aggregate.cu -- fused edge-message -> scatter_softmax -> scatter_sum attention aggregation (the HBM-bound kernel).
//
// Reference (models/uni_transformer.py):
//   x2h :73-83   alpha = scatter_softmax((q[dst]*k/sqrt(8)).sum(-1), dst);  out = scatter_sum(alpha[...,None]*v*e_w, dst) + h
//   h2x :131-140 v = xv[E,16]*e_w;  m = alpha*v[...,None]*(x[dst]-x[src]);  delta = scatter_sum(m, dst).mean(heads)
//   :205-206     x = x + delta * mask_ligand
// torch_scatter does this as 7 launches with atomics over an arbitrary index; here the k-NN list is dst-sorted with a
// fixed row length, so a destination's edges are one contiguous [deg,128] fp32 block: one warp per destination streams
// it with coalesced 512 B row reads (float4 per lane), the 16 per-head logits live 2 lanes per head (one xor-shuffle),
// softmax is an in-register online max/sum, and the result is one coalesced 512 B store.  No atomics, no re-reads.
//
// Algorithmic HBM bytes (SURVEY.md 8(d)): x2h  E*(512 k + 512 v + 4 e_w) + N*(512 q + 512 h + 512 out) = E*1028 + N*1536
//                                         h2x  E*(512 k + 64 v + 4 e_w + 4 src + 12 x_src) + N*(512 q + 12 x + 12 out + 1) = E*596 + N*537
#include "tdiff_common.cuh"

#define AGG_WARPS 8
#define AGG_CH 8          // edge rows in flight per warp (8 x 512 B k + 8 x 512 B v)

__device__ __forceinline__ float4 ldg_stream4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// logit of head lane/2 for one edge: sum_d (q_d*k_d)/sqrt(8), 4 terms per lane + the partner lane's 4
__device__ __forceinline__ float head_logit(const float4& q, const float4& k) {
  const float s8 = 2.8284271247461903f;   // float32(np.sqrt(8))
  float s = (__fdiv_rn(q.x * k.x, s8) + __fdiv_rn(q.y * k.y, s8)) + (__fdiv_rn(q.z * k.z, s8) + __fdiv_rn(q.w * k.w, s8));
  return s + __shfl_xor_sync(0xffffffffu, s, 1);
}

__global__ void __launch_bounds__(AGG_WARPS * 32)
aggregate_h_kernel(const float* __restrict__ kbuf, const float* __restrict__ vbuf, const float* __restrict__ e_w,
                   const int* __restrict__ src, const float* __restrict__ q, const float* __restrict__ h_in,
                   float* __restrict__ h_out, int n_nodes, int k) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * AGG_WARPS + (threadIdx.x >> 5);
  if (n >= n_nodes) return;
  const size_t e0 = (size_t)n * k;
  // degree = number of leading valid slots (absent edges are -1-padded at the tail)
  int deg = 0;
  for (int j = lane; j < k; j += 32) deg += (src[e0 + j] >= 0);
  deg = __reduce_add_sync(0xffffffffu, deg);
  const float4 q4 = *reinterpret_cast<const float4*>(q + (size_t)n * TD_H + 4 * lane);
  const float4 hin = *reinterpret_cast<const float4*>(h_in + (size_t)n * TD_H + 4 * lane);
  float m = -INFINITY, l = 0.0f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j0 = 0; j0 < deg; j0 += AGG_CH) {
    float4 kr[AGG_CH], vr[AGG_CH];
    float ew[AGG_CH];
#pragma unroll
    for (int c = 0; c < AGG_CH; ++c) {
      if (j0 + c < deg) {
        kr[c] = ldg_stream4(kbuf + (e0 + j0 + c) * TD_H + 4 * lane);
        vr[c] = ldg_stream4(vbuf + (e0 + j0 + c) * TD_H + 4 * lane);
        ew[c] = e_w[e0 + j0 + c];
      }
    }
#pragma unroll
    for (int c = 0; c < AGG_CH; ++c) {
      if (j0 + c < deg) {
        const float s = head_logit(q4, kr[c]);
        const float mn = fmaxf(m, s);
        const float sc = expf(m - mn);
        const float p = expf(s - mn);
        const float pw = p * ew[c];
        l = l * sc + p;
        acc.x = acc.x * sc + pw * vr[c].x;
        acc.y = acc.y * sc + pw * vr[c].y;
        acc.z = acc.z * sc + pw * vr[c].z;
        acc.w = acc.w * sc + pw * vr[c].w;
        m = mn;
      }
    }
  }
  float4 o = hin;
  if (deg > 0) {
    o.x += acc.x / l; o.y += acc.y / l; o.z += acc.z / l; o.w += acc.w / l;
  }
  *reinterpret_cast<float4*>(h_out + (size_t)n * TD_H + 4 * lane) = o;
}

void td_launch_aggregate_h(const float* kbuf, const float* vbuf, const float* e_w, const int* src, const float* q, const float* h_in,
                           float* h_out, int n_nodes, int k, cudaStream_t st) {
  if (n_nodes == 0) return;
  aggregate_h_kernel<<<(n_nodes + AGG_WARPS - 1) / AGG_WARPS, AGG_WARPS * 32, 0, st>>>(kbuf, vbuf, e_w, src, q, h_in, h_out, n_nodes, k);
}

// Coordinate update.  Rows = destinations to process: row a -> node row_nodes[a] (or a when row_nodes == NULL);
// kbuf/v16 are indexed by row (compact), src/e_w by node slot.  xm = (x, y, z, mask); xm_out may alias nothing in xm_in.
__global__ void __launch_bounds__(AGG_WARPS * 32)
aggregate_x_kernel(const float* __restrict__ kbuf, const float* __restrict__ v16, const float* __restrict__ e_w,
                   const int* __restrict__ src, const float* __restrict__ q, const float4* __restrict__ xm_in,
                   const int* __restrict__ row_nodes, float4* __restrict__ xm_out, int n_rows, int k) {
  const int lane = threadIdx.x & 31;
  const int a = blockIdx.x * AGG_WARPS + (threadIdx.x >> 5);
  if (a >= n_rows) return;
  const int n = row_nodes ? row_nodes[a] : a;
  const size_t e0 = (size_t)n * k;       // slot base (src, e_w)
  const size_t r0 = (size_t)a * k;       // row base (kbuf, v16)
  int deg = 0;
  for (int j = lane; j < k; j += 32) deg += (src[e0 + j] >= 0);
  deg = __reduce_add_sync(0xffffffffu, deg);
  const float4 q4 = *reinterpret_cast<const float4*>(q + (size_t)n * TD_H + 4 * lane);
  const float4 xd = xm_in[n];
  float m = -INFINITY, l = 0.0f;
  float ax = 0.f, ay = 0.f, az = 0.f;
  for (int j0 = 0; j0 < deg; j0 += AGG_CH) {
    float4 kr[AGG_CH];
    float vv[AGG_CH];
    float4 xs[AGG_CH];
#pragma unroll
    for (int c = 0; c < AGG_CH; ++c) {
      if (j0 + c < deg) {
        kr[c] = ldg_stream4(kbuf + (r0 + j0 + c) * TD_H + 4 * lane);
        vv[c] = v16[(r0 + j0 + c) * TD_HEADS + (lane >> 1)] * e_w[e0 + j0 + c];
        xs[c] = xm_in[src[e0 + j0 + c]];
      }
    }
#pragma unroll
    for (int c = 0; c < AGG_CH; ++c) {
      if (j0 + c < deg) {
        const float s = head_logit(q4, kr[c]);
        const float mn = fmaxf(m, s);
        const float sc = expf(m - mn);
        const float p = expf(s - mn);
        const float pv = p * vv[c];
        l = l * sc + p;
        ax = ax * sc + pv * (xd.x - xs[c].x);
        ay = ay * sc + pv * (xd.y - xs[c].y);
        az = az * sc + pv * (xd.z - xs[c].z);
        m = mn;
      }
    }
  }
  float dx = 0.f, dy = 0.f, dz = 0.f;
  if (deg > 0) {
    const float w = (lane & 1) ? 0.0f : 1.0f / l;      // each head is held by a lane pair: count it once
    dx = warp_sum(ax * w) * (1.0f / TD_HEADS);
    dy = warp_sum(ay * w) * (1.0f / TD_HEADS);
    dz = warp_sum(az * w) * (1.0f / TD_HEADS);
  }
  if (lane == 0) xm_out[n] = make_float4(xd.x + dx * xd.w, xd.y + dy * xd.w, xd.z + dz * xd.w, xd.w);
}

void td_launch_aggregate_x(const float* kbuf, const float* v16, const float* e_w, const int* src, const float* q, const float4* xm_in,
                           const int* row_nodes, float4* xm_out, int n_rows, int k, cudaStream_t st) {
  if (n_rows == 0) return;
  aggregate_x_kernel<<<(n_rows + AGG_WARPS - 1) / AGG_WARPS, AGG_WARPS * 32, 0, st>>>(kbuf, v16, e_w, src, q, xm_in, row_nodes, xm_out,
                                                                                   n_rows, k);
}

// ------------------------------------------------------------------------------------------------------------------------
// Variants that consume precomputed attention logits [rows,16] (written by the key-MLP epilogue of edge_mlp_v3.cu, so the
// [E,128] key tensor never reaches HBM).  Algorithmic HBM bytes: x2h  E*(64 logits + 512 v + 4 e_w) + N*(512 h + 512 out);
// h2x  E_l*(64 + 64 v + 4 e_w + 4 src + 12 x_src) + N_l*(12 x + 12 out + 1).
// ------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AGG_WARPS * 32)
aggregate_h_logits_kernel(const float* __restrict__ logits, const float* __restrict__ vbuf, const float* __restrict__ e_w,
                          const int* __restrict__ src, const float* __restrict__ h_in, float* __restrict__ h_out, TdRows dst, int k,
                          const float* __restrict__ ewm_w, float ewm_b) {
  const int lane = threadIdx.x & 31;
  const long long a = (long long)blockIdx.x * AGG_WARPS + (threadIdx.x >> 5);
  if (a >= (dst.d_n ? (long long)*dst.d_n : dst.n)) return;
  const int n = dst.list ? dst.list[a] : (int)a;
  if (n < 0) return;
  const size_t e0 = (size_t)n * k;
  int deg = 0;
  for (int j = lane; j < k; j += 32) deg += (src[e0 + j] >= 0);
  deg = __reduce_add_sync(0xffffffffu, deg);
  const float4 hin = *reinterpret_cast<const float4*>(h_in + (size_t)n * TD_H + 4 * lane);
  // ew_net_type 'm' (reference models/uni_transformer.py:60-61): the gate is sigmoid(Linear(value row)), evaluated on the fly
  float4 wm = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ewm_w) wm = *reinterpret_cast<const float4*>(ewm_w + 4 * lane);
  float m = -INFINITY, l = 0.0f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j0 = 0; j0 < deg; j0 += AGG_CH) {
    float4 vr[AGG_CH];
    float ew[AGG_CH], sg[AGG_CH];
#pragma unroll
    for (int c = 0; c < AGG_CH; ++c) {
      if (j0 + c < deg) {
        vr[c] = ldg_stream4(vbuf + (e0 + j0 + c) * TD_H + 4 * lane);
        sg[c] = logits[(e0 + j0 + c) * TD_HEADS + (lane >> 1)];
        ew[c] = e_w[e0 + j0 + c];
      }
    }
    if (ewm_w) {
#pragma unroll
      for (int c = 0; c < AGG_CH; ++c) {
        if (j0 + c < deg) {          // warp-uniform
          const float dot = warp_sum((vr[c].x * wm.x + vr[c].y * wm.y) + (vr[c].z * wm.z + vr[c].w * wm.w));
          ew[c] = 1.0f / (1.0f + expf(-(dot + ewm_b)));
        }
      }
    }
#pragma unroll
    for (int c = 0; c < AGG_CH; ++c) {
      if (j0 + c < deg) {
        const float s = sg[c];
        const float mn = fmaxf(m, s);
        const float sc = expf(m - mn);
        const float p = expf(s - mn);
        const float pw = p * ew[c];
        l = l * sc + p;
        acc.x = acc.x * sc + pw * vr[c].x;
        acc.y = acc.y * sc + pw * vr[c].y;
        acc.z = acc.z * sc + pw * vr[c].z;
        acc.w = acc.w * sc + pw * vr[c].w;
        m = mn;
      }
    }
  }
  float4 o = hin;
  if (deg > 0) {
    o.x += acc.x / l; o.y += acc.y / l; o.z += acc.z / l; o.w += acc.w / l;
  }
  *reinterpret_cast<float4*>(h_out + (size_t)n * TD_H + 4 * lane) = o;
}

void td_launch_aggregate_h_logits(const float* logits, const float* vbuf, const float* e_w, const int* src, const float* h_in, float* h_out,
                                  const TdRows& dst, int k, const float* ewm_w, float ewm_b, cudaStream_t st) {
  if (dst.n == 0) return;
  aggregate_h_logits_kernel<<<(unsigned)((dst.n + AGG_WARPS - 1) / AGG_WARPS), AGG_WARPS * 32, 0, st>>>(logits, vbuf, e_w, src, h_in, h_out, dst, k,
                                                                                                       ewm_w, ewm_b);
}

__global__ void __launch_bounds__(AGG_WARPS * 32)
aggregate_x_logits_kernel(const float* __restrict__ logits, const float* __restrict__ v16, const float* __restrict__ e_w,
                          const int* __restrict__ src, const float4* __restrict__ xm_in, const int* __restrict__ row_nodes,
                          float4* __restrict__ xm_out, int n_rows, int k) {
  const int lane = threadIdx.x & 31;
  const int a = blockIdx.x * AGG_WARPS + (threadIdx.x >> 5);
  if (a >= n_rows) return;
  const int n = row_nodes ? row_nodes[a] : a;
  const size_t e0 = (size_t)n * k, r0 = (size_t)a * k;
  int deg = 0;
  for (int j = lane; j < k; j += 32) deg += (src[e0 + j] >= 0);
  deg = __reduce_add_sync(0xffffffffu, deg);
  const float4 xd = xm_in[n];
  float m = -INFINITY, l = 0.0f;
  float ax = 0.f, ay = 0.f, az = 0.f;
  for (int j = 0; j < deg; ++j) {
    const float s = logits[(r0 + j) * TD_HEADS + (lane >> 1)];
    const float vv = v16[(r0 + j) * TD_HEADS + (lane >> 1)] * e_w[e0 + j];
    const float4 xs = xm_in[src[e0 + j]];
    const float mn = fmaxf(m, s);
    const float sc = expf(m - mn);
    const float p = expf(s - mn);
    const float pv = p * vv;
    l = l * sc + p;
    ax = ax * sc + pv * (xd.x - xs.x);
    ay = ay * sc + pv * (xd.y - xs.y);
    az = az * sc + pv * (xd.z - xs.z);
    m = mn;
  }
  float dx = 0.f, dy = 0.f, dz = 0.f;
  if (deg > 0) {
    const float w = (lane & 1) ? 0.0f : 1.0f / l;
    dx = warp_sum(ax * w) * (1.0f / TD_HEADS);
    dy = warp_sum(ay * w) * (1.0f / TD_HEADS);
    dz = warp_sum(az * w) * (1.0f / TD_HEADS);
  }
  if (lane == 0) xm_out[n] = make_float4(xd.x + dx * xd.w, xd.y + dy * xd.w, xd.z + dz * xd.w, xd.w);
}

void td_launch_aggregate_x_logits(const float* logits, const float* v16, const float* e_w, const int* src, const float4* xm_in,
                                  const int* row_nodes, float4* xm_out, int n_rows, int k, cudaStream_t st) {
  if (n_rows == 0) return;
  aggregate_x_logits_kernel<<<(n_rows + AGG_WARPS - 1) / AGG_WARPS, AGG_WARPS * 32, 0, st>>>(logits, v16, e_w, src, xm_in, row_nodes, xm_out,
                                                                                          n_rows, k);
}
