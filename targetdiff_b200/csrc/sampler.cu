// sampler.cu -- the per-step diffusion update fused into one kernel, plus small state/marshalling kernels.
//
// step_epilogue restates the loop body after the network call of ScorePosNet3D.sample_diffusion
// (reference models/molopt_score_model.py:667-693, C0 mode) and its helpers:
//   q_pos_posterior :424-428, extract :706-708, index_to_log_onehot :124-130 (clamp 1e-30), log_add_exp :173-175,
//   q_v_pred :383-392, q_v_pred_one_timestep :371-381, q_v_posterior :401-409, log_sample_categorical :160-166.
// The reference issues ~25 elementwise launches and 4 D2H copies per step; here it is one launch, trajectories are
// written straight into preallocated device buffers, and the step index lives in device memory so that the whole
// step can be replayed from a CUDA graph with zero host synchronisation.
#include "tdiff_common.cuh"
#include "sampler.cuh"

// ---------------------------------------------------------------------------------------- Philox4x32-10
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ key.x, lo1, hi0 ^ c.w ^ key.y, lo0);
    key.x += 0x9E3779B9u; key.y += 0xBB67AE85u;
  }
  return c;
}
__device__ __forceinline__ float u01(unsigned x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }   // [0,1), 24 bits

__device__ __forceinline__ float log_add_exp_f(float a, float b) {
  const float mx = fmaxf(a, b);
  return mx + logf(expf(a - mx) + expf(b - mx));
}

#define TD_LOG_EPS (-69.07755279f)   // logf(1e-30f): index_to_log_onehot's clamp (reference :124-130)

// log_add_exp(log_onehot(v)[c] + lam, l1m): class c's term of q(. | onehot(v)) in log space, the unnormalised form of q_v_pred and
// q_v_pred_one_timestep (reference :371-392)
__device__ __forceinline__ float log_q_onehot(int c, int v, float lam, float l1m) {
  return log_add_exp_f(((c == v) ? 0.0f : TD_LOG_EPS) + lam, l1m);
}

// lr = log_softmax of the type head's row lg[0 .. K); with kMask, the classes whose bit of `am` is clear enter as -inf (exp gives exactly
// 0 there, so every sum is unchanged when all are allowed) and leave as -inf
template <bool kMask>
__device__ __forceinline__ void log_softmax(const float* lg, int K, uint32_t am, float* lr) {
  float mx = -INFINITY;
  for (int c = 0; c < K; ++c) {
    lr[c] = (kMask && !((am >> c) & 1u)) ? -INFINITY : lg[c];
    mx = fmaxf(mx, lr[c]);
  }
  float se = 0.0f;
  for (int c = 0; c < K; ++c) se += expf(lr[c] - mx);
  const float lse = logf(se);
  for (int c = 0; c < K; ++c) lr[c] = (lr[c] - mx) - lse;
}

// One class of a Gumbel-max draw (log_sample_categorical, reference :160-166): class c with uniform u and log-probability lp replaces
// the best so far only on a strictly larger score, so that a tie goes to the lowest class, as the reference's argmax does
__device__ __forceinline__ void gumbel_max(float u, float lp, int c, float& best, int& vbest) {
  const float sc = -logf(-logf(u + 1e-30f) + 1e-30f) + lp;
  if (sc > best) { best = sc; vbest = c; }
}

// c x + d eps with every product and the sum rounded once, as the reference's perturbation (models/molopt_score_model.py:500-504)
__device__ __forceinline__ float4 forward_transition(float c, float d, const float4& x, const float nz[3]) {
  return make_float4(__fadd_rn(__fmul_rn(c, x.x), __fmul_rn(d, nz[0])), __fadd_rn(__fmul_rn(c, x.y), __fmul_rn(d, nz[1])),
                     __fadd_rn(__fmul_rn(c, x.z), __fmul_rn(d, nz[2])), 1.0f);
}

// Row s of the trajectories: pos_traj the centred x plus the graph's offset, v_traj the class v
__device__ __forceinline__ void write_traj(const TdStepArgs& A, int s, int a, const float4& x, int v) {
  if (A.pos_traj) {
    const float4 off = A.offset[A.lig_graph[a]];
    float* o = A.pos_traj + ((size_t)s * A.n_lig + a) * 3;
    o[0] = x.x + off.x; o[1] = x.y + off.y; o[2] = x.z + off.z;
  }
  if (A.v_traj) A.v_traj[(size_t)s * A.n_lig + a] = (long long)v;
}

// Philox domain words of the sampling chain's own stream ("pst\0", "vuni"; oracle/philox.py)
#define TD_STEP_POS_DOMAIN 0x70737400u
#define TD_STEP_TYPE_DOMAIN 0x76756e69u
// Philox domain words of the fixed-atom stream ("fxps", "fxtv"), distinct from the two above (oracle/fixed_atoms.py)
#define TD_FIX_POS_DOMAIN 0x66787073u
#define TD_FIX_TYPE_DOMAIN 0x66787476u
// Philox domain words of the start-ligand stream ("stps", "sttv"), distinct from the four above (oracle/start_ligand.py)
#define TD_START_POS_DOMAIN 0x73747073u
#define TD_START_TYPE_DOMAIN 0x73747476u

// Philox domain words of the likelihood stream ("lkps", "lktv"), distinct from the six above (oracle/likelihood.py)
#define TD_LK_POS_DOMAIN 0x6c6b7073u
#define TD_LK_TYPE_DOMAIN 0x6c6b7476u

// A random stream (Src) names its tapes, its Philox domain words and its draw layout: the tape row of draw d of row a, and its counter,
// lane 0 for positions and 1 + c/4 for class c.  TdDrawByRow is the layout of the step, fixed-atom and start streams: tape row
// d * Nl + a and counter (a, d, lane, domain).
struct TdDrawByRow {
  static __device__ __forceinline__ size_t row(const TdStepArgs& A, int a, int d) { return (size_t)d * A.n_lig + a; }
  static __device__ __forceinline__ uint4 counter(const TdStepArgs&, int a, int d, unsigned lane, unsigned domain) {
    return make_uint4((unsigned)a, (unsigned)d, lane, domain);
  }
};

// The chain's own stream: draw d = s is step s (steps already taken), whichever its kind (DESIGN.md section 1)
struct TdStepSource : TdDrawByRow {
  static constexpr unsigned kPosDomain = TD_STEP_POS_DOMAIN, kTypeDomain = TD_STEP_TYPE_DOMAIN;
  static __device__ __forceinline__ const float* pos_tape(const TdStepArgs& A) { return A.pos_noise; }
  static __device__ __forceinline__ const float* v_tape(const TdStepArgs& A) { return A.v_uniform; }
};

// Sources of forward_sample: x0 / v0, the tapes and the Philox domain words of the fixed-atom stream and of the start stream
struct TdFixedSource : TdDrawByRow {
  static constexpr unsigned kPosDomain = TD_FIX_POS_DOMAIN, kTypeDomain = TD_FIX_TYPE_DOMAIN;
  static __device__ __forceinline__ const float4* x0(const TdStepArgs& A) { return A.fix_pos; }
  static __device__ __forceinline__ const int* v0(const TdStepArgs& A) { return A.fix_v; }
  static __device__ __forceinline__ const float* pos_tape(const TdStepArgs& A) { return A.fix_pos_noise; }
  static __device__ __forceinline__ const float* v_tape(const TdStepArgs& A) { return A.fix_v_uniform; }
};
struct TdStartSource : TdDrawByRow {   // the start ligand is the chain's own state before the start draw
  static constexpr unsigned kPosDomain = TD_START_POS_DOMAIN, kTypeDomain = TD_START_TYPE_DOMAIN;
  static __device__ __forceinline__ const float4* x0(const TdStepArgs& A) { return A.lig_pos; }
  static __device__ __forceinline__ const int* v0(const TdStepArgs& A) { return A.lig_v; }
  static __device__ __forceinline__ const float* pos_tape(const TdStepArgs& A) { return A.start_pos_noise; }
  static __device__ __forceinline__ const float* v_tape(const TdStepArgs& A) { return A.start_v_uniform; }
};
// Likelihood scoring: the clean ligand is the ligand state; `d` is the atom's index j within its graph g, so that the counter
// (j, k_g, t_g << 8 | lane, domain) does not depend on where the graph sits in the batch.  The tape is [Nl, .] in batch order.
struct TdLikelihoodSource {
  static constexpr unsigned kPosDomain = TD_LK_POS_DOMAIN, kTypeDomain = TD_LK_TYPE_DOMAIN;
  static __device__ __forceinline__ const float4* x0(const TdStepArgs& A) { return A.lig_pos; }
  static __device__ __forceinline__ const int* v0(const TdStepArgs& A) { return A.lig_v; }
  static __device__ __forceinline__ const float* pos_tape(const TdStepArgs& A) { return A.lk_pos_noise; }
  static __device__ __forceinline__ const float* v_tape(const TdStepArgs& A) { return A.lk_v_uniform; }
  static __device__ __forceinline__ size_t row(const TdStepArgs&, int a, int) { return (size_t)a; }
  static __device__ __forceinline__ uint4 counter(const TdStepArgs& A, int a, int d, unsigned lane, unsigned domain) {
    const int g = A.lig_graph[a];
    return make_uint4((unsigned)d, A.lk_key[g], ((unsigned)A.lk_t[g] << 8) | lane, domain);
  }
};

// Every random number of the sampler is drawn by draw_normal3 and draw_uniform4, from draw d of row a of the stream Src: a tape row, or
// Philox4x32-10 on Src's counter under the sampler's key (seed mod 2^32, seed >> 32).
template <class Src>
__device__ __forceinline__ uint4 philox_draw(const TdStepArgs& A, int a, int d, unsigned lane, unsigned domain) {
  return philox4x32_10(Src::counter(A, a, d, lane, domain), make_uint2((unsigned)A.seed, (unsigned)(A.seed >> 32)));
}
// nz = three standard normals: row Src::row(a, d) of the position tape [., 3], or Box-Muller on counter (a, d, 0, position domain) with
// u0, u2 in (0, 1] and u1, u3 in [0, 1).
template <class Src>
__device__ __forceinline__ void draw_normal3(const TdStepArgs& A, int a, int d, float nz[3]) {
  if (Src::pos_tape(A)) {
    const float* pn = Src::pos_tape(A) + Src::row(A, a, d) * 3;
    nz[0] = pn[0]; nz[1] = pn[1]; nz[2] = pn[2];
  } else {
    const uint4 r0 = philox_draw<Src>(A, a, d, 0u, Src::kPosDomain);
    const float u0 = 1.0f - u01(r0.x), u1 = u01(r0.y), u2 = 1.0f - u01(r0.z), u3 = u01(r0.w);
    const float ra = sqrtf(-2.0f * logf(u0)), rb = sqrtf(-2.0f * logf(u2));
    nz[0] = ra * cospif(2.0f * u1); nz[1] = ra * sinpif(2.0f * u1); nz[2] = rb * cospif(2.0f * u3);
  }
}
// u[j] = the uniform of class c0 + j (c0 a multiple of 4): the type tape [., K] for c0 + j < K, or the four words of counter
// (a, d, 1 + c0/4, type domain)
template <class Src>
__device__ __forceinline__ void draw_uniform4(const TdStepArgs& A, int a, int d, int c0, float u[4]) {
  const int K = A.n_classes;
  if (Src::v_tape(A)) {
    const float* vu = Src::v_tape(A) + Src::row(A, a, d) * K;
    for (int j = 0; j < 4 && c0 + j < K; ++j) u[j] = vu[c0 + j];
  } else {
    const uint4 r = philox_draw<Src>(A, a, d, 1u + (unsigned)(c0 >> 2), Src::kTypeDomain);
    u[0] = u01(r.x); u[1] = u01(r.y); u[2] = u01(r.z); u[3] = u01(r.w);
  }
}

// Row `a`: a sample of q(x_tm | x0) and q(v_tm | v0) with x0 / v0 from `Src`, from draw `d` of its stream or tapes; x0 / v0 exactly
// when tm < 0.  Position sqrt(ac) x0 + sqrt(1 - ac) eps (forward_transition); type: Gumbel-max over the unnormalised
// q_v_pred(log_onehot(v0), tm) (q_v_sample, :394-398).  With pos_only the type is left as it is.  For a fixed atom (TdFixedSource,
// DESIGN.md section 1) d = 0 is the draw before the first step and d = j + 1 the draw after step j.
template <class Src>
__device__ __forceinline__ void forward_sample(const TdStepArgs& A, int a, int d, int tm, float4& x, int& v) {
  const float4 x0 = Src::x0(A)[a];
  if (tm < 0) {
    x = make_float4(x0.x, x0.y, x0.z, 1.0f);
    if (!A.pos_only) v = Src::v0(A)[a];
    return;
  }
  float nz[3];
  draw_normal3<Src>(A, a, d, nz);
  const float acv = A.ac[tm];
  x = forward_transition(sqrtf(acv), sqrtf(1.0f - acv), x0, nz);
  if (A.pos_only) return;
  const int K = A.n_classes, v0 = Src::v0(A)[a];
  const float lca = A.lca_v[tm], l1mca = A.l1mca_v[tm] - A.log_k;
  float best = -INFINITY;
  int vbest = 0;
  for (int c0 = 0; c0 < K; c0 += 4) {
    float u[4];
    draw_uniform4<Src>(A, a, d, c0, u);
    for (int j = 0; j < 4 && c0 + j < K; ++j) gumbel_max(u[j], log_q_onehot(c0 + j, v0, lca, l1mca), c0 + j, best, vbest);
  }
  v = vbest;
}

// The step's x0 prediction of ligand row `a` at network time t, centred frame: the node array's row in C0 mode; in 'noise' mode
// x0 = sqrt(1/ac) x_t - sqrt(1/ac - 1) (pred - x_t)   (reference :419-422,663-666).  Shared by step_epilogue_kernel and
// clash_guidance_kernel, so that a row guidance leaves alone has the same bits in a guided and an unguided step.
__device__ __forceinline__ float4 td_pred_x0(const TdStepArgs& A, int a, int t, const float4& xt) {
  float4 x0 = A.xm_final[A.lig_node[a]];
  if (A.mean_noise) {
    const float ra = A.sra[t], rm = A.srm1[t];
    x0.x = ra * xt.x - rm * (x0.x - xt.x);
    x0.y = ra * xt.y - rm * (x0.y - xt.y);
    x0.z = ra * xt.z - rm * (x0.z - xt.z);
  }
  return x0;
}

// kSeq = true runs step s of a respaced chain (DESIGN.md section 1): the network saw t = seq_t[s], and the state moves to p = seq_p[s]
// with the per-step coefficients seq_*[s]; kSeq = false is the default chain t = t_start - s, p = t - 1 on the checkpoint's tables.  A
// guided step (clash guidance) runs these same instances with xm_final = the guided predictions and mean_noise = 0: the guidance kernel
// has already converted them.  kMask = true (element constraints, DESIGN.md section 1): bit c of allowed[a] set = class c allowed for
// row a.  The type head's log_softmax runs over the allowed classes only, and on the decoder step (p < 0) the posterior's forbidden
// classes are -inf before its normalisation, so that it is renormalised over the allowed set and the Gumbel-max draw can only pick an
// allowed class.  kMask = false never reads `allowed`.  Fixed rows (fix_mask) are overwritten after the update.
template <bool kSeq, bool kMask>
__global__ void step_epilogue_kernel(TdStepArgs A, const uint32_t* __restrict__ allowed) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A.n_lig) return;
  const int s = *A.step;                       // steps done so far
  const int t = kSeq ? A.seq_t[s] : A.t_start - s;   // current timestep (reference :649-651)
  const int p = kSeq ? A.seq_p[s] : t - 1;           // the time this step moves to
  const int K = A.n_classes;
  const bool fixed = A.fix_mask && A.fix_mask[a];

  // ---- positions: posterior mean + noise (reference :673-679)
  float nz[3];
  draw_normal3<TdStepSource>(A, a, s, nz);
  const float4 xt = A.lig_pos[a];
  const float4 x0 = td_pred_x0(A, a, t, xt);
  const float c0 = kSeq ? A.seq_c0[s] : A.c0[t], ct = kSeq ? A.seq_ct[s] : A.ct[t];
  const float sig = ((t == 0) ? 0.0f : 1.0f) * expf(0.5f * (kSeq ? A.seq_logvar[s] : A.logvar[t]));
  float4 xn;
  xn.x = (c0 * x0.x + ct * xt.x) + sig * nz[0];
  xn.y = (c0 * x0.y + ct * xt.y) + sig * nz[1];
  xn.z = (c0 * x0.z + ct * xt.z) + sig * nz[2];
  xn.w = 1.0f;
  // a fixed row is overwritten after the update: q(x_p | x0_f) from draw s + 1, or x0_f itself after t = 0
  int vfix = 0;
  if (fixed) forward_sample<TdFixedSource>(A, a, s + 1, p, xn, vfix);
  A.lig_pos[a] = xn;

  int vnew = A.lig_v[a];
  if (!A.pos_only) {
    // ---- atom types: categorical posterior in log space (reference :682-685)
    float lr[TD_CMAX];
    const uint32_t am = kMask ? allowed[a] : 0u;
    log_softmax<kMask>(A.logits + (size_t)a * K, K, am, lr);
    const int tm1 = kSeq ? (p > 0 ? p : 0) : (t > 0 ? t - 1 : 0);
    const float lca = A.lca_v[tm1], l1mca = A.l1mca_v[tm1] - A.log_k;
    const float la = kSeq ? A.seq_la[s] : A.la_v[t], l1ma = (kSeq ? A.seq_l1ma[s] : A.l1ma_v[t]) - A.log_k;
    const int vcur = vnew;
    float un_lp[TD_CMAX];
    float m2 = -INFINITY;
    for (int c = 0; c < K; ++c) {
      un_lp[c] = log_add_exp_f(lr[c] + lca, l1mca) + log_q_onehot(c, vcur, la, l1ma);
      if (kMask && p < 0 && !((am >> c) & 1u)) un_lp[c] = -INFINITY;       // decoder step: renormalised over the allowed set
      m2 = fmaxf(m2, un_lp[c]);
    }
    float s2 = 0.0f;
    for (int c = 0; c < K; ++c) s2 += expf(un_lp[c] - m2);
    const float lse2 = m2 + logf(s2);                                      // torch.logsumexp
    float best = -INFINITY;
    vnew = 0;
    float* o0 = A.v0_traj ? A.v0_traj + ((size_t)s * A.n_lig + a) * K : nullptr;
    float* ot = A.vt_traj ? A.vt_traj + ((size_t)s * A.n_lig + a) * K : nullptr;
    for (int c0 = 0; c0 < K; c0 += 4) {
      float u[4];
      draw_uniform4<TdStepSource>(A, a, s, c0, u);
      for (int j = 0; j < 4 && c0 + j < K; ++j) {
        const int c = c0 + j;
        const float lp = un_lp[c] - lse2;
        gumbel_max(u[j], lp, c, best, vnew);
        if (o0) o0[c] = lr[c];
        if (ot) ot[c] = lp;
      }
    }
    if (fixed) vnew = vfix;                    // v0_traj / vt_traj above keep the model's own opinion of the row
    A.lig_v[a] = vnew;
  }
  write_traj(A, s, a, xn, vnew);
}

__global__ void advance_step_kernel(int* step) { *step += 1; }

template <bool kMask>
static void launch_step_epilogue(const TdStepArgs& A, const uint32_t* allowed, int grid, cudaStream_t st) {
  if (A.seq_t) step_epilogue_kernel<true, kMask><<<grid, 128, 0, st>>>(A, allowed);
  else step_epilogue_kernel<false, kMask><<<grid, 128, 0, st>>>(A, allowed);
}
void td_launch_step_epilogue(const TdStepArgs& A, const uint32_t* allowed, cudaStream_t st) {
  if (A.n_lig > 0) {
    const int grid = (A.n_lig + 127) / 128;
    if (allowed) launch_step_epilogue<true>(A, allowed, grid, st);
    else launch_step_epilogue<false>(A, nullptr, grid, st);
  }
  advance_step_kernel<<<1, 1, 0, st>>>(A.step);
}

// ---------------------------------------------------------------------------------------- clash guidance
// Clash guidance (DESIGN.md section 1), before the epilogue of a denoising step: for ligand row a of graph g with the step's x0
// prediction y (td_pred_x0), and each protein atom p of g at its bound position x_p, r = y - x_p, d = |r|; a pair contributes when
// 0 < d < radius, and the guided prediction is y + strength * sum (radius - d) r / d over the contributing pairs, or y itself, bit for
// bit, when none contributes.  It is written to row lig_node[a] of G.guided, a node-indexed array, which the unchanged epilogue then
// reads as its xm_final.  One CTA per graph: the graph's protein coordinates pass through shared memory in chunks of
// TD_GUIDE_CHUNK atoms; one warp per ligand atom, lane l summing the protein atoms j = l, l + 32, ... of the graph in order, then a
// fixed shuffle tree.  The order of every sum depends on the graph's own atoms only, so a graph gets the same bits in any batch.
#define TD_GUIDE_CHUNK 1024
#define TD_GUIDE_WARPS 8
__global__ void __launch_bounds__(TD_GUIDE_WARPS * 32) clash_guidance_kernel(TdStepArgs A, TdGuideArgs G) {
  __shared__ float sx[TD_GUIDE_CHUNK], sy[TD_GUIDE_CHUNK], sz[TD_GUIDE_CHUNK];
  const int g = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int p0 = G.node_ptr[g], np = G.prot_ptr[g + 1] - G.prot_ptr[g];       // protein nodes p0 .. p0 + np - 1 lead the graph
  const int lb = G.node_ptr[g] - G.prot_ptr[g], le = G.node_ptr[g + 1] - G.prot_ptr[g + 1];
  if (lb >= le) return;
  const int s = *A.step;
  const int t = A.seq_t ? A.seq_t[s] : A.t_start - s;
  const float rho = G.radius, lam = G.strength;
  const int nchunk = (np + TD_GUIDE_CHUNK - 1) / TD_GUIDE_CHUNK;
  auto stage = [&](int c) {
    __syncthreads();
    for (int j = threadIdx.x; j < TD_GUIDE_CHUNK && c * TD_GUIDE_CHUNK + j < np; j += blockDim.x) {
      const float4 x = G.prot_xm[p0 + c * TD_GUIDE_CHUNK + j];
      sx[j] = x.x; sy[j] = x.y; sz[j] = x.z;
    }
    __syncthreads();
  };
  if (nchunk == 1) stage(0);
  for (int base = lb; base < le; base += TD_GUIDE_WARPS) {      // every warp runs every round: the staging barriers are uniform
    const int a = base + warp;
    const bool live = a < le;
    float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live) y = td_pred_x0(A, a, t, A.lig_pos[a]);
    float ax = 0.f, ay = 0.f, az = 0.f;
    unsigned hit = 0;
    for (int c = 0; c < nchunk; ++c) {
      if (nchunk > 1) stage(c);
      const int n = min(TD_GUIDE_CHUNK, np - c * TD_GUIDE_CHUNK);
      if (!live) continue;
      for (int j = lane; j < n; j += 32) {
        const float rx = y.x - sx[j], ry = y.y - sy[j], rz = y.z - sz[j];
        const float d = sqrtf(rx * rx + ry * ry + rz * rz);
        if (d > 0.f && d < rho) {
          const float w = (rho - d) / d;
          ax += w * rx; ay += w * ry; az += w * rz;
          hit = 1;
        }
      }
    }
    if (!live) continue;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ax += __shfl_xor_sync(0xffffffffu, ax, o);
      ay += __shfl_xor_sync(0xffffffffu, ay, o);
      az += __shfl_xor_sync(0xffffffffu, az, o);
    }
    if (__any_sync(0xffffffffu, hit) && lane == 0) {
      y.x = y.x + lam * ax; y.y = y.y + lam * ay; y.z = y.z + lam * az;
    }
    if (lane == 0) G.guided[A.lig_node[a]] = y;
  }
}
void td_launch_clash_guidance(const TdStepArgs& A, const TdGuideArgs& G, int n_graphs, cudaStream_t st) {
  if (A.n_lig > 0 && n_graphs > 0) clash_guidance_kernel<<<n_graphs, TD_GUIDE_WARPS * 32, 0, st>>>(A, G);
}

// ---------------------------------------------------------------------------------------- connectivity guidance
// Connectivity guidance (DESIGN.md section 1), before the epilogue of a denoising step and after clash guidance when both are on.  Graph
// g's ligand rows i = 0 .. n-1 (within-graph indices) sit at q_i: the held row's target x0_f (fix_pos) when fix_mask marks it, the
// step's x0 prediction y_i (td_pred_x0) otherwise.  Rows i, j are bonded when |q_i - q_j| < radius.  With one component every row keeps
// y.  Otherwise each component C without a held row takes its closest outside pair (i in C, j not in C, smallest d, then lowest (i, j))
// and moves rigidly: every row a of C gets y_a + f (q_j - q_i), f = (strength * w * (d - length)) / d, w = 1 when j's component holds a
// held row and 1/2 otherwise; components with a held row keep y.  Every distance, comparison and the shift are explicitly rounded fp32
// operations (no contraction), so a float32 restatement makes the same decisions, and every decision reads the graph's own rows only.
// One CTA per graph, rows in shared memory; components by hook-and-compress union-find (roots end as the lowest index of their
// component); the closest pair of each component as a 64-bit atomicMin key (d^2 bits << 32 | i << 16 | j).  Writes row lig_node[a] of
// C.guided for every ligand row, held rows included (the epilogue overwrites those as before).
#define TD_CONNECT_THREADS 256
__device__ __forceinline__ float connect_dist2(const float* sx, const float* sy, const float* sz, int i, int j) {
  const float dx = __fsub_rn(sx[j], sx[i]), dy = __fsub_rn(sy[j], sy[i]), dz = __fsub_rn(sz[j], sz[i]);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
__global__ void __launch_bounds__(TD_CONNECT_THREADS) connect_guidance_kernel(TdStepArgs A, TdConnectArgs C) {
  __shared__ float sx[TD_CONNECT_MAX], sy[TD_CONNECT_MAX], sz[TD_CONNECT_MAX];
  __shared__ int par[TD_CONNECT_MAX];
  __shared__ unsigned long long key[TD_CONNECT_MAX];
  __shared__ unsigned char row_held[TD_CONNECT_MAX], comp_held[TD_CONNECT_MAX];
  __shared__ int changed, n_comp;
  const int g = blockIdx.x, tid = threadIdx.x;
  const int lb = C.node_ptr[g] - C.prot_ptr[g], n = C.node_ptr[g + 1] - C.prot_ptr[g + 1] - lb;
  const int s = *A.step;
  const int t = A.seq_t ? A.seq_t[s] : A.t_start - s;
  // the engine refuses a chain with more than TD_CONNECT_MAX ligand atoms in a graph; a graph of one atom is one component
  const bool multi_possible = n >= 2 && n <= TD_CONNECT_MAX;
  if (multi_possible) {
    for (int i = tid; i < n; i += blockDim.x) {
      const int a = lb + i;
      const bool h = A.fix_mask && A.fix_mask[a];
      const float4 q = h ? A.fix_pos[a] : td_pred_x0(A, a, t, A.lig_pos[a]);
      sx[i] = q.x; sy[i] = q.y; sz[i] = q.z;
      par[i] = i; key[i] = ~0ull; row_held[i] = h; comp_held[i] = 0;
    }
    if (tid == 0) { changed = 0; n_comp = 0; }
    __syncthreads();
    const float rho = C.radius;
    volatile int* vp = par;
    for (;;) {
      // hook: for every bonded pair in different trees, the higher root points to the lower one.  Parents only decrease and always
      // point within a component; a hook lost to a concurrent one leaves `changed` set, so the pair is seen again next round
      for (int k = tid; k < n * n; k += blockDim.x) {
        const int i = k / n, j = k - i * n;
        if (j <= i || !(__fsqrt_rn(connect_dist2(sx, sy, sz, i, j)) < rho)) continue;
        int ri = i, rj = j;
        while (vp[ri] != ri) ri = vp[ri];
        while (vp[rj] != rj) rj = vp[rj];
        if (ri != rj) {
          atomicMin(&par[max(ri, rj)], min(ri, rj));
          changed = 1;
        }
      }
      __syncthreads();
      const bool again = changed;
      // compress: every row points at its root
      for (int i = tid; i < n; i += blockDim.x) {
        int r = vp[i];
        while (vp[r] != r) r = vp[r];
        vp[i] = r;
      }
      __syncthreads();
      if (!again) break;
      if (tid == 0) changed = 0;
      __syncthreads();
    }
    for (int i = tid; i < n; i += blockDim.x) {
      if (row_held[i]) comp_held[par[i]] = 1;
      if (par[i] == i) atomicAdd(&n_comp, 1);
    }
    __syncthreads();
    if (n_comp > 1) {
      for (int k = tid; k < n * n; k += blockDim.x) {
        const int i = k / n, j = k - i * n;
        if (par[i] == par[j]) continue;
        const float d2 = connect_dist2(sx, sy, sz, i, j);
        atomicMin(&key[par[i]], ((unsigned long long)__float_as_uint(d2) << 32) | ((unsigned)i << 16) | (unsigned)j);
      }
      __syncthreads();
    }
  }
  const bool shift = multi_possible && n_comp > 1;
  const float lam = C.strength, bl = C.length;
  for (int i = tid; i < n; i += blockDim.x) {
    const int a = lb + i;
    float4 y = td_pred_x0(A, a, t, A.lig_pos[a]);
    if (shift && !comp_held[par[i]]) {
      const unsigned long long k = key[par[i]];
      const int ci = (int)((k >> 16) & 0xffffu), cj = (int)(k & 0xffffu);
      const float d = __fsqrt_rn(__uint_as_float((unsigned)(k >> 32)));
      const float w = comp_held[par[cj]] ? 1.0f : 0.5f;
      const float f = __fdiv_rn(__fmul_rn(__fmul_rn(lam, w), __fsub_rn(d, bl)), d);
      y.x = __fadd_rn(y.x, __fmul_rn(f, __fsub_rn(sx[cj], sx[ci])));
      y.y = __fadd_rn(y.y, __fmul_rn(f, __fsub_rn(sy[cj], sy[ci])));
      y.z = __fadd_rn(y.z, __fmul_rn(f, __fsub_rn(sz[cj], sz[ci])));
    }
    C.guided[A.lig_node[a]] = y;
  }
}
void td_launch_connect_guidance(const TdStepArgs& A, const TdConnectArgs& C, int n_graphs, cudaStream_t st) {
  if (A.n_lig > 0 && n_graphs > 0) connect_guidance_kernel<<<n_graphs, TD_CONNECT_THREADS, 0, st>>>(A, C);
}

// Re-noising step s of a time path (tdiff_sample_path, DESIGN.md section 1): the state moves up from t = seq_t[s] to p = seq_p[s] > t
// with the forward process, no network.  The step tables hold c = sqrt(abar_p / abar_t) in seq_c0, d = sqrt(1 - abar_p / abar_t) in
// seq_ct, lambda = log of the type schedule's transition probability t -> p in seq_la and log(1 - e^lambda + 1e-40) in seq_l1ma.  A row
// that is not fixed: x_p = c x_t + d eps (forward_transition), and a Gumbel-max draw over the unnormalised log q(v_p | v_t) =
// log_add_exp(log_onehot(v_t) + lambda, l1ma - log K) (q_v_sample's form); with pos_only the type stays.  Fixed rows: q(x_p | x0_f),
// q(v_p | v0_f) from draw s + 1, as after a denoising step.  The random stream is the denoising step's, draw s of TdStepSource.
// Trajectories: pos_traj / v_traj the new state, vt_traj the normalised log q(v_p | v_t), v0_traj a copy of entry s - 1 (the latest
// network prediction).
__global__ void renoise_kernel(TdStepArgs A) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A.n_lig) return;
  const int s = *A.step;
  const int p = A.seq_p[s];
  const int K = A.n_classes;
  const bool fixed = A.fix_mask && A.fix_mask[a];
  float4 xn;
  int vnew = A.lig_v[a];
  if (!fixed) {
    float nz[3];
    draw_normal3<TdStepSource>(A, a, s, nz);
    xn = forward_transition(A.seq_c0[s], A.seq_ct[s], A.lig_pos[a], nz);
  } else {
    forward_sample<TdFixedSource>(A, a, s + 1, p, xn, vnew);
  }
  if (!A.pos_only) {
    const float la = A.seq_la[s], l1ma = A.seq_l1ma[s] - A.log_k;
    const int vcur = A.lig_v[a];
    float lq[TD_CMAX];
    float mx = -INFINITY;
    for (int c = 0; c < K; ++c) {
      lq[c] = log_q_onehot(c, vcur, la, l1ma);
      mx = fmaxf(mx, lq[c]);
    }
    float se = 0.0f;
    for (int c = 0; c < K; ++c) se += expf(lq[c] - mx);
    const float lse = mx + logf(se);                                       // torch.logsumexp
    float* ot = A.vt_traj ? A.vt_traj + ((size_t)s * A.n_lig + a) * K : nullptr;
    float* o0 = A.v0_traj ? A.v0_traj + ((size_t)s * A.n_lig + a) * K : nullptr;
    const float* p0 = o0 ? o0 - (size_t)A.n_lig * K : nullptr;
    float best = -INFINITY;
    int vbest = 0;
    for (int c0 = 0; c0 < K; c0 += 4) {
      float u[4];
      draw_uniform4<TdStepSource>(A, a, s, c0, u);
      for (int j = 0; j < 4 && c0 + j < K; ++j) {
        const int c = c0 + j;
        gumbel_max(u[j], lq[c], c, best, vbest);
        if (ot) ot[c] = lq[c] - lse;
        if (o0) o0[c] = p0[c];
      }
    }
    if (!fixed) vnew = vbest;
    A.lig_v[a] = vnew;
  }
  A.lig_pos[a] = xn;
  write_traj(A, s, a, xn, vnew);
}

void td_launch_renoise(const TdStepArgs& A, cudaStream_t st) {
  if (A.n_lig > 0) renoise_kernel<<<(A.n_lig + 127) / 128, 128, 0, st>>>(A);
  advance_step_kernel<<<1, 1, 0, st>>>(A.step);
}

// fixed rows <- q(x_{T-1} | x0_f), q(v_{T-1} | v0_f) from draw 0, once before the first step of a chain
__global__ void fixed_init_kernel(TdStepArgs A) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A.n_lig || !A.fix_mask[a]) return;
  float4 x;
  int v = A.lig_v[a];
  forward_sample<TdFixedSource>(A, a, 0, A.t_start, x, v);
  A.lig_pos[a] = x;
  A.lig_v[a] = v;
}
void td_launch_fixed_init(const TdStepArgs& A, cudaStream_t st) {
  if (A.n_lig > 0) fixed_init_kernel<<<(A.n_lig + 127) / 128, 128, 0, st>>>(A);
}

// start chain (tdiff_set_start), once before its first step, in place of fixed_init_kernel: every row <- a sample at t_start.  Fixed
// rows as fixed_init_kernel gives them (draw 0 of the fixed-atom stream); the others from the start stream with their own state, the
// start ligand, as x0 / v0 -- counters (a, 0, 0, "stps") and (a, 0, 1 + c/4, "sttv"), or the start tape pos [Nl,3], v [Nl,K].
__global__ void start_init_kernel(TdStepArgs A) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A.n_lig) return;
  float4 x;
  int v = A.lig_v[a];
  if (A.fix_mask && A.fix_mask[a]) forward_sample<TdFixedSource>(A, a, 0, A.t_start, x, v);
  else forward_sample<TdStartSource>(A, a, 0, A.t_start, x, v);
  A.lig_pos[a] = x;
  A.lig_v[a] = v;
}
void td_launch_start_init(const TdStepArgs& A, cudaStream_t st) {
  if (A.n_lig > 0) start_init_kernel<<<(A.n_lig + 127) / 128, 128, 0, st>>>(A);
}

// ---------------------------------------------------------------------------------------- likelihood scoring
// tdiff_likelihood_terms (DESIGN.md section 1): graph g at t_g.  Before the forward: x0 / v0 saved to scratch, every row <- a sample of
// q(x_t | x0), q(v_t | v0) at t_g (forward_sample on the likelihood stream or tape), time_norm[g] = t_g / T divided in fp32.
__global__ void likelihood_init_kernel(TdLikelihoodArgs L) {
  const TdStepArgs& A = L.A;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (L.time_norm && i < L.n_graphs) L.time_norm[i] = __fdiv_rn((float)A.lk_t[i], (float)L.n_timesteps);
  if (i >= A.n_lig) return;
  const int g = A.lig_graph[i];
  const int j = i - (L.node_ptr[g] - L.prot_ptr[g]);
  L.x0[i] = A.lig_pos[i];
  L.v0[i] = A.lig_v[i];
  float4 x;
  int v = A.lig_v[i];
  forward_sample<TdLikelihoodSource>(A, i, j, A.lk_t[g], x, v);
  A.lig_pos[i] = x;
  A.lig_v[i] = v;
}
void td_launch_likelihood_init(const TdLikelihoodArgs& L, cudaStream_t st) {
  const int n = L.A.n_lig > L.n_graphs ? L.A.n_lig : L.n_graphs;
  if (n > 0) likelihood_init_kernel<<<(n + 127) / 128, 128, 0, st>>>(L);
}

// After the forward: the per-atom terms of graph g, restated op by op from the reference (models/molopt_score_model.py:133-155
// normal_kl / log_normal / categorical_kl / log_categorical, :401-409 q_v_posterior, :411-438 the priors, :470-489 compute_pos_Lt /
// compute_v_Lt, :588-617 likelihood_estimation), their means over the graph's ligand atoms (summed in atom order in fp32, then divided
// by the count, as scatter_mean on CPU; 0 for a graph without ligand atoms), and the ligand state restored to x0 / v0.  One block per
// graph: each chunk of 128 atoms puts its terms in shared memory and thread 0 adds them up in order.
__global__ void __launch_bounds__(128) likelihood_epilogue_kernel(TdLikelihoodArgs L) {
  const TdStepArgs& A = L.A;
  __shared__ float terms[4][128];
  const int g = blockIdx.x, tid = threadIdx.x;
  const int b = L.node_ptr[g] - L.prot_ptr[g], e = L.node_ptr[g + 1] - L.prot_ptr[g + 1];
  const int t = A.lk_t[g], T = L.n_timesteps, K = A.n_classes;
  const float log_sqrt_2pi = 0.918938533f;                                 // np.log(np.sqrt(2 * np.pi)) in fp32
  const float log_2 = 0.693147181f;                                        // np.log(2.) in fp32
  float sum[4] = {0.f, 0.f, 0.f, 0.f};
  for (int base = b; base < e; base += 128) {
    const int a = base + tid;
    if (a < e) {
      const float4 x0 = L.x0[a], xt = A.lig_pos[a], px = L.xm_final[L.lig_node[a]];
      const int v0 = L.v0[a], vt = A.lig_v[a];
      const float x0v[3] = {x0.x, x0.y, x0.z}, xtv[3] = {xt.x, xt.y, xt.z}, pxv[3] = {px.x, px.y, px.z};
      // ---- positions: q_pos_posterior of the model's x0 and of the true x0, each product and sum rounded once (:424-428)
      const float c0 = L.c0[t], ct = L.ct[t], lv = L.logvar[t];
      float tp = 0.f;
      if (t > 0) {                 // normal_kl(mean_true, lv, mean_model, lv) / log 2 (compute_pos_Lt, :470-482)
        for (int d = 0; d < 3; ++d) {
          const float ctx = __fmul_rn(ct, xtv[d]);
          const float df = __fadd_rn(__fmul_rn(c0, x0v[d]), ctx) - __fadd_rn(__fmul_rn(c0, pxv[d]), ctx);
          tp += 0.5f * ((((-1.0f + lv) - lv) + expf(lv - lv)) + __fmul_rn(__fmul_rn(df, df), expf(-lv)));
        }
        tp = tp / log_2;
      } else {                     // decoder: -log_normal(x0, mean_model, 0.5 lv), in nats
        const float ls = 0.5f * lv, var2 = 2.0f * expf(ls * 2.0f);
        float lp = 0.f;
        for (int d = 0; d < 3; ++d) {
          const float df = x0v[d] - __fadd_rn(__fmul_rn(c0, pxv[d]), __fmul_rn(ct, xtv[d]));
          lp += ((-__fmul_rn(df, df)) / var2 - ls) - log_sqrt_2pi;
        }
        tp = -lp;
      }
      // ---- types: q_v_posterior of log_softmax(logits) and of log_onehot(v0) given v_t (:401-409), at t - 1 clamped to 0
      float lr[TD_CMAX], um[TD_CMAX], ut[TD_CMAX];
      log_softmax<false>(L.logits + (size_t)a * K, K, 0u, lr);
      const int tm1 = t > 0 ? t - 1 : 0;
      const float lca = A.lca_v[tm1], l1mca = A.l1mca_v[tm1] - A.log_k;
      const float la = L.la_v[t], l1ma = L.l1ma_v[t] - A.log_k;
      float mm = -INFINITY, mt = -INFINITY;
      for (int c = 0; c < K; ++c) {
        const float q1 = log_q_onehot(c, vt, la, l1ma);
        um[c] = log_add_exp_f(lr[c] + lca, l1mca) + q1;
        ut[c] = log_q_onehot(c, v0, lca, l1mca) + q1;
        mm = fmaxf(mm, um[c]); mt = fmaxf(mt, ut[c]);
      }
      float sm = 0.f, st = 0.f;
      for (int c = 0; c < K; ++c) { sm += expf(um[c] - mm); st += expf(ut[c] - mt); }
      const float lsm = mm + logf(sm), lst = mt + logf(st);                // torch.logsumexp
      float tv = 0.f;
      if (t > 0) {                 // categorical_kl(log_true, log_model)
        for (int c = 0; c < K; ++c) {
          const float lt = ut[c] - lst;
          tv += __fmul_rn(expf(lt), lt - (um[c] - lsm));
        }
      } else {                     // -log_categorical(log_onehot(v0), log_model): the clamped entries weigh exp(log 1e-30)
        const float w_eps = expf(TD_LOG_EPS);
        for (int c = 0; c < K; ++c) tv += __fmul_rn((c == v0) ? 1.0f : w_eps, um[c] - lsm);
        tv = -tv;
      }
      // ---- priors at T - 1 with the ligand's own types (kl_pos_prior / kl_v_prior, :411-438)
      const float acT = A.ac[T - 1];
      const float sa = sqrtf(acT), lv2 = logf(sqrtf(1.0f - acT));
      float pp = 0.f;
      for (int d = 0; d < 3; ++d) {
        const float m = __fmul_rn(sa, x0v[d]);
        pp += 0.5f * ((((-1.0f + lv2) - 0.0f) + expf(0.0f - lv2)) + __fmul_rn(__fmul_rn(0.0f - m, 0.0f - m), expf(-lv2)));
      }
      const float lcaT = A.lca_v[T - 1], l1mcaT = A.l1mca_v[T - 1] - A.log_k, log_half = -logf((float)K);
      float pv = 0.f;
      for (int c = 0; c < K; ++c) {
        const float lq = log_q_onehot(c, v0, lcaT, l1mcaT);
        pv += __fmul_rn(expf(lq), lq - log_half);
      }
      terms[0][tid] = tp; terms[1][tid] = tv; terms[2][tid] = pp; terms[3][tid] = pv;
      if (L.atom_kl_pos) L.atom_kl_pos[a] = tp;
      if (L.atom_kl_v) L.atom_kl_v[a] = tv;
      if (L.xt) { L.xt[3 * a] = xt.x; L.xt[3 * a + 1] = xt.y; L.xt[3 * a + 2] = xt.z; }
      if (L.vt) L.vt[a] = (long long)vt;
      A.lig_pos[a] = x0;
      A.lig_v[a] = v0;
    }
    __syncthreads();
    if (tid == 0) {
      const int n = min(128, e - base);
      for (int i = 0; i < n; ++i) { sum[0] += terms[0][i]; sum[1] += terms[1][i]; sum[2] += terms[2][i]; sum[3] += terms[3][i]; }
    }
    __syncthreads();
  }
  if (tid != 0) return;
  const float cnt = (float)(e - b > 0 ? e - b : 1);
  if (L.kl_pos) L.kl_pos[g] = sum[0] / cnt;
  if (L.kl_v) L.kl_v[g] = sum[1] / cnt;
  if (L.prior_pos) L.prior_pos[g] = sum[2] / cnt;
  if (L.prior_v) L.prior_v[g] = sum[3] / cnt;
}
void td_launch_likelihood_epilogue(const TdLikelihoodArgs& L, cudaStream_t st) {
  if (L.n_graphs > 0) likelihood_epilogue_kernel<<<L.n_graphs, 128, 0, st>>>(L);
}

// fixed set in (tdiff_set_fixed): positions and classes are read at masked rows only; lab frame -> centred like set_ligand_kernel
__global__ void set_fixed_kernel(const unsigned char* __restrict__ mask, const float* __restrict__ pos, const long long* __restrict__ v,
                                 const int* __restrict__ lig_graph, const float4* __restrict__ offset, int apply_center, int n, int n_classes,
                                 unsigned char* __restrict__ fix_mask, float4* __restrict__ fix_pos, int* __restrict__ fix_v, int* __restrict__ err) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  const unsigned char m = mask[a] ? 1 : 0;
  fix_mask[a] = m;
  if (!m) { fix_pos[a] = make_float4(0.f, 0.f, 0.f, 1.0f); fix_v[a] = 0; return; }
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  if (apply_center) o = offset[lig_graph[a]];
  fix_pos[a] = make_float4(pos[3 * a] - o.x, pos[3 * a + 1] - o.y, pos[3 * a + 2] - o.z, 1.0f);
  const long long vv = v[a];
  if (vv < 0 || vv >= n_classes) { atomicExch(err, 1); fix_v[a] = 0; }
  else fix_v[a] = (int)vv;
}
void td_launch_set_fixed(const unsigned char* mask, const float* pos, const long long* v, const int* lig_graph, const float4* offset,
                         int apply_center, int n, int n_classes, unsigned char* fix_mask, float4* fix_pos, int* fix_v, int* err,
                         cudaStream_t st) {
  if (n > 0) set_fixed_kernel<<<(n + 255) / 256, 256, 0, st>>>(mask, pos, v, lig_graph, offset, apply_center, n, n_classes, fix_mask, fix_pos,
                                                               fix_v, err);
}

// type mask in (tdiff_set_type_mask): every row needs a class and no bit at or above n_classes; only checked, the caller copies
__global__ void check_type_mask_kernel(const uint32_t* __restrict__ allowed, int n, int n_classes, int* __restrict__ err) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  const uint32_t m = allowed[a];
  const uint32_t outside = n_classes >= 32 ? 0u : ~((1u << n_classes) - 1u);
  if (m == 0u || (m & outside)) atomicExch(err, 1);
}
void td_launch_check_type_mask(const uint32_t* allowed, int n, int n_classes, int* err, cudaStream_t st) {
  if (n > 0) check_type_mask_kernel<<<(n + 255) / 256, 256, 0, st>>>(allowed, n, n_classes, err);
}

// ---------------------------------------------------------------------------------------- state marshalling
// per-graph protein centroid, sequential fp32 sum in atom order then / count == torch_scatter.scatter_mean on CPU
// (reference models/molopt_score_model.py:115)
__global__ void segment_mean3_kernel(const float* __restrict__ pos, const int* __restrict__ seg_ptr, int n_seg, float4* __restrict__ out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_seg) return;
  float sx = 0.f, sy = 0.f, sz = 0.f;
  const int b = seg_ptr[g], e = seg_ptr[g + 1];
  for (int i = b; i < e; ++i) { sx += pos[3 * i]; sy += pos[3 * i + 1]; sz += pos[3 * i + 2]; }
  float cnt = (float)(e - b);
  if (cnt < 1.0f) cnt = 1.0f;
  out[g] = make_float4(sx / cnt, sy / cnt, sz / cnt, 0.0f);
}
void td_launch_segment_mean3(const float* pos, const int* seg_ptr, int n_seg, float4* out, cudaStream_t st) {
  if (n_seg > 0) segment_mean3_kernel<<<(n_seg + 127) / 128, 128, 0, st>>>(pos, seg_ptr, n_seg, out);
}

// protein atoms -> node array (both ping-pong buffers), centred
__global__ void place_protein_kernel(const float* __restrict__ pos, const int* __restrict__ prot_node, const int* __restrict__ prot_graph,
                                     const float4* __restrict__ offset, int n, float4* __restrict__ xm0, float4* __restrict__ xm1) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const float4 o = offset[prot_graph[p]];
  const float4 v = make_float4(pos[3 * p] - o.x, pos[3 * p + 1] - o.y, pos[3 * p + 2] - o.z, 0.0f);
  xm0[prot_node[p]] = v;
  xm1[prot_node[p]] = v;
}
void td_launch_place_protein(const float* pos, const int* prot_node, const int* prot_graph, const float4* offset, int n, float4* xm0,
                             float4* xm1, cudaStream_t st) {
  if (n > 0) place_protein_kernel<<<(n + 255) / 256, 256, 0, st>>>(pos, prot_node, prot_graph, offset, n, xm0, xm1);
}

// ligand state in  (lab frame -> centred float4, int64 -> int32, range check like reference :125)
__global__ void set_ligand_kernel(const float* __restrict__ pos, const long long* __restrict__ v, const int* __restrict__ lig_graph,
                                  const float4* __restrict__ offset, int apply_center, int n, int n_classes, float4* __restrict__ lig_pos,
                                  int* __restrict__ lig_v, int* __restrict__ err) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  if (apply_center) o = offset[lig_graph[a]];
  lig_pos[a] = make_float4(pos[3 * a] - o.x, pos[3 * a + 1] - o.y, pos[3 * a + 2] - o.z, 1.0f);
  if (v) {
    const long long vv = v[a];
    if (vv < 0 || vv >= n_classes) { atomicExch(err, 1); lig_v[a] = 0; }      // never store an index that would read out of bounds
    else lig_v[a] = (int)vv;
  }
}
void td_launch_set_ligand(const float* pos, const long long* v, const int* lig_graph, const float4* offset, int apply_center, int n,
                          int n_classes, float4* lig_pos, int* lig_v, int* err, cudaStream_t st) {
  if (n > 0) set_ligand_kernel<<<(n + 255) / 256, 256, 0, st>>>(pos, v, lig_graph, offset, apply_center, n, n_classes, lig_pos, lig_v, err);
}

__global__ void get_ligand_kernel(const float4* __restrict__ lig_pos, const int* __restrict__ lig_v, const int* __restrict__ lig_graph,
                                  const float4* __restrict__ offset, int add_offset, int n, float* __restrict__ pos, long long* __restrict__ v) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  if (pos) {
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (add_offset) o = offset[lig_graph[a]];
    const float4 p = lig_pos[a];
    pos[3 * a] = p.x + o.x; pos[3 * a + 1] = p.y + o.y; pos[3 * a + 2] = p.z + o.z;
  }
  if (v) v[a] = (long long)lig_v[a];
}
void td_launch_get_ligand(const float4* lig_pos, const int* lig_v, const int* lig_graph, const float4* offset, int add_offset, int n,
                          float* pos, long long* v, cudaStream_t st) {
  if (n > 0) get_ligand_kernel<<<(n + 255) / 256, 256, 0, st>>>(lig_pos, lig_v, lig_graph, offset, add_offset, n, pos, v);
}

// ligand atoms parked far from every pocket (distinct points; ligand-free cache construction, engine.cu)
__global__ void park_ligand_kernel(float4* __restrict__ lig_pos, int* __restrict__ lig_v, int n) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  lig_pos[a] = make_float4(1.0e6f + 64.0f * (float)(a & 4095), 1.0e6f + 64.0f * (float)((a >> 12) & 4095), 1.0e6f, 1.0f);
  lig_v[a] = 0;
}
void td_launch_park_ligand(float4* lig_pos, int* lig_v, int n, cudaStream_t st) {
  if (n > 0) park_ligand_kernel<<<(n + 255) / 256, 256, 0, st>>>(lig_pos, lig_v, n);
}

// ligand rows of the node array <- ligand state (start of every forward)
__global__ void scatter_ligand_pos_kernel(const float4* __restrict__ lig_pos, const int* __restrict__ lig_node, int n, float4* __restrict__ xm) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a < n) xm[lig_node[a]] = lig_pos[a];
}
void td_launch_scatter_ligand_pos(const float4* lig_pos, const int* lig_node, int n, float4* xm, cudaStream_t st) {
  if (n > 0) scatter_ligand_pos_kernel<<<(n + 255) / 256, 256, 0, st>>>(lig_pos, lig_node, n, xm);
}

// float4 node rows -> packed [n,3] (all nodes when idx == NULL, else gathered rows)
__global__ void gather_xyz_kernel(const float4* __restrict__ xm, const int* __restrict__ idx, int n, float* __restrict__ out) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n) return;
  const float4 p = xm[idx ? idx[a] : a];
  out[3 * a] = p.x; out[3 * a + 1] = p.y; out[3 * a + 2] = p.z;
}
void td_launch_gather_xyz(const float4* xm, const int* idx, int n, float* out, cudaStream_t st) {
  if (n > 0) gather_xyz_kernel<<<(n + 255) / 256, 256, 0, st>>>(xm, idx, n, out);
}

__global__ void pack_xyzm_kernel(const float* __restrict__ x, const unsigned char* __restrict__ mask, int n, float4* __restrict__ xm) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a < n) xm[a] = make_float4(x[3 * a], x[3 * a + 1], x[3 * a + 2], (mask && mask[a]) ? 1.0f : 0.0f);
}
void td_launch_pack_xyzm(const float* x, const unsigned char* mask, int n, float4* xm, cudaStream_t st) {
  if (n > 0) pack_xyzm_kernel<<<(n + 255) / 256, 256, 0, st>>>(x, mask, n, xm);
}

// ---------------------------------------------------------------------------------------- edge_index export
// slots [N*k] (-1 padded) -> compact int64 [2,E] in slot order (dst ascending, then distance ascending):
// exactly PyG knn_graph(flow='source_to_target') row0 = src, row1 = dst.  Single-CTA scan over per-node degrees.
__global__ void __launch_bounds__(1024)
edge_count_scan_kernel(const int* __restrict__ src, int n_nodes, int k, long long* __restrict__ node_off, long long* __restrict__ total) {
  __shared__ long long part[1024];
  const int tid = threadIdx.x;
  const int per = (n_nodes + 1023) / 1024;
  const int b = min(tid * per, n_nodes), e = min(b + per, n_nodes);
  long long s = 0;
  for (int n = b; n < e; ++n) {
    int d = 0;
    for (int j = 0; j < k; ++j) d += (src[(size_t)n * k + j] >= 0);
    s += d;
  }
  part[tid] = s;
  __syncthreads();
  if (tid == 0) {
    long long run = 0;
    for (int i = 0; i < 1024; ++i) { const long long v = part[i]; part[i] = run; run += v; }
    *total = run;
  }
  __syncthreads();
  long long run = part[tid];
  for (int n = b; n < e; ++n) {
    node_off[n] = run;
    int d = 0;
    for (int j = 0; j < k; ++j) d += (src[(size_t)n * k + j] >= 0);
    run += d;
  }
}
__global__ void edge_compact_kernel(const int* __restrict__ src, const float* __restrict__ e_w, int n_nodes, int k,
                                    const long long* __restrict__ node_off, const long long* __restrict__ total,
                                    long long* __restrict__ edge_index, float* __restrict__ ew_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n_nodes * k) return;
  const int n = (int)(i / k), j = (int)(i % k);
  const int s = src[i];
  if (s < 0) return;
  const long long E = *total;
  const long long pos = node_off[n] + j;       // valid slots are leading
  if (edge_index) { edge_index[pos] = s; edge_index[E + pos] = n; }
  if (ew_out) ew_out[pos] = e_w[i];
}
void td_launch_edge_count_scan(const int* src, int n_nodes, int k, long long* node_off, long long* total, cudaStream_t st) {
  edge_count_scan_kernel<<<1, 1024, 0, st>>>(src, n_nodes, k, node_off, total);
}
void td_launch_edge_compact(const int* src, const float* e_w, int n_nodes, int k, const long long* node_off, const long long* total,
                            long long* edge_index, float* ew_out, cudaStream_t st) {
  const long long n = (long long)n_nodes * k;
  if (n > 0) edge_compact_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(src, e_w, n_nodes, k, node_off, total, edge_index, ew_out);
}
