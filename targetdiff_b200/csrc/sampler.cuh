// sampler.cuh -- argument block of the fused step epilogue and the marshalling launchers (sampler.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct TdStepArgs {
  int n_lig, n_classes, t_start, pos_only;
  int* step;                       // device: steps already done in this chain (advanced by the launcher's tail kernel)
  const int* lig_node;             // [Nl] node index of each ligand atom
  const int* lig_graph;            // [Nl] graph id
  const float4* xm_final;          // node array after the last layer (predicted x0 in the centred frame)
  const float* logits;             // [Nl,K]
  const float4* offset;            // [B] pocket centroids
  const float *c0, *ct, *logvar;   // posterior_mean_c0_coef, posterior_mean_ct_coef, posterior_logvar [T]
  const float *sra, *srm1;         // sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod [T] (model_mean_type 'noise')
  int mean_noise;                  // 1: the network output is x_t + predicted noise direction (reference :663-666)
  const float *la_v, *l1ma_v, *lca_v, *l1mca_v;   // log_alphas_v, log_one_minus_alphas_v, and their cumprod versions [T]
  float log_k;                     // float32(np.log(num_classes))
  const float* pos_noise;          // tape [S,Nl,3] or NULL (Philox)
  const float* v_uniform;          // tape [S,Nl,K] or NULL (Philox)
  unsigned long long seed;
  float4* lig_pos;                 // in/out [Nl] centred ligand positions
  int* lig_v;                      // in/out [Nl]
  float* pos_traj;                 // [S,Nl,3] or NULL
  long long* v_traj;               // [S,Nl] or NULL
  float* v0_traj;                  // [S,Nl,K] or NULL
  float* vt_traj;                  // [S,Nl,K] or NULL
  // fixed atoms (tdiff_set_fixed); fix_mask == NULL: none
  const unsigned char* fix_mask;   // [Nl] 1 = the row is held to the forward process of (fix_pos, fix_v)
  const float4* fix_pos;           // [Nl] target positions x0_f, centred frame
  const int* fix_v;                // [Nl] target classes v0_f
  const float* ac;                 // alphas_cumprod [T]
  const float* fix_pos_noise;      // fixed-atom tape [S+1,Nl,3] or NULL (Philox, FIX_POS domain)
  const float* fix_v_uniform;      // fixed-atom tape [S+1,Nl,K] or NULL (Philox, FIX_TYPE domain)
  // respaced chain (tdiff_sample_seq) or time path (tdiff_sample_path); seq_t == NULL: the default chain, t = t_start - step, and the
  // kernel takes that path only.  A re-noising step (p > t) keeps c, d, lambda, l1ma in seq_c0, seq_ct, seq_la, seq_l1ma (renoise_kernel)
  const int* seq_t;                // [S] tau_s, the time the network sees at step s
  const int* seq_p;                // [S] the time step s moves to: tau_{s+1}, or tau_{S-1} - 1 at the last step
  const float *seq_c0, *seq_ct, *seq_logvar;   // [S] position posterior of the jump t -> p (the checkpoint's tables at t on unit steps)
  const float *seq_la, *seq_l1ma;  // [S] lambda = log of the type schedule's transition probability p -> t, log(1 - e^lambda + 1e-40)
  // start chain (tdiff_set_start): the start draw's tape, read by start_init_kernel only
  const float* start_pos_noise;    // [Nl,3] or NULL (Philox, START_POS domain)
  const float* start_v_uniform;    // [Nl,K] or NULL (Philox, START_TYPE domain)
  // likelihood scoring (tdiff_likelihood_terms): per-graph timestep and draw key, the noising draw's tape; read by likelihood kernels only
  const int* lk_t;                 // [B] t_g in 0..T-1
  const unsigned* lk_key;          // [B] k_g
  const float* lk_pos_noise;       // [Nl,3] or NULL (Philox, LK_POS domain)
  const float* lk_v_uniform;       // [Nl,K] or NULL (Philox, LK_TYPE domain)
};

// likelihood scoring (DESIGN.md section 1): the noising draw (TdStepArgs A) and the epilogue's own tables and outputs
struct TdLikelihoodArgs {
  TdStepArgs A;                    // n_lig, n_classes, seed, ac, lca_v, l1mca_v, log_k, lig_pos, lig_v, lig_graph, lk_*
  int n_graphs, n_timesteps;
  const int *node_ptr, *prot_ptr;  // [B+1]: graph g's ligand atoms are node_ptr[g] - prot_ptr[g] .. node_ptr[g+1] - prot_ptr[g+1] - 1
  const float4* xm_final;          // node array after the forward (predicted x0, centred)
  const int* lig_node;             // [Nl]
  const float* logits;             // [Nl,K]
  const float *c0, *ct, *logvar;   // posterior_mean_c0_coef, posterior_mean_ct_coef, posterior_logvar [T]
  const float *la_v, *l1ma_v;      // log_alphas_v, log_one_minus_alphas_v [T]
  float4* x0;                      // scratch [Nl]: the clean ligand, restored into lig_pos by the epilogue
  int* v0;                         // scratch [Nl]
  float* time_norm;                // [B] t_g / T, or NULL (no time embedding)
  float *kl_pos, *kl_v, *prior_pos, *prior_v;   // [B] or NULL
  float *atom_kl_pos, *atom_kl_v;  // [Nl] or NULL
  float* xt;                       // [Nl,3] centred x_t, or NULL
  long long* vt;                   // [Nl] v_t, or NULL
};

// clash guidance (DESIGN.md section 1): the batch layout, the bound protein coordinates and the guided x0 predictions
struct TdGuideArgs {
  const int *node_ptr, *prot_ptr;  // [B+1]: graph g's protein atoms are nodes node_ptr[g] .. node_ptr[g] + prot_ptr[g+1] - prot_ptr[g] - 1
  const float4* prot_xm;           // node array whose protein rows hold the bound, centred protein positions (xm0)
  float4* guided;                  // out [N], node-indexed: row lig_node[a] <- the guided x0 prediction of ligand row a
  float radius, strength;          // rho > 0 (A), lambda > 0
};

// connectivity guidance (DESIGN.md section 1): the batch layout, the bond radius, bond length and strength, and the guided x0
// predictions.  The kernel reads each row's prediction through td_pred_x0 of its TdStepArgs, so after clash guidance (xm_final =
// guided, mean_noise = 0) it reads and rewrites the guided rows in place
#define TD_CONNECT_MAX 1024        // ligand atoms per graph (TDIFF_CONNECT_MAX_ATOMS): within-graph indices fit the key's 16-bit fields
struct TdConnectArgs {
  const int *node_ptr, *prot_ptr;  // [B+1]: graph g's ligand rows are node_ptr[g] - prot_ptr[g] .. node_ptr[g+1] - prot_ptr[g+1] - 1
  float4* guided;                  // out [N], node-indexed: row lig_node[a] <- the guided x0 prediction of ligand row a
  float radius, length, strength;  // rho > 0, 0 < b < rho (A), lambda > 0
};

// allowed: [Nl] class bit masks of the element constraint (tdiff_set_type_mask), or NULL for the unconstrained step
void td_launch_step_epilogue(const TdStepArgs& A, const uint32_t* allowed, cudaStream_t st);
void td_launch_check_type_mask(const uint32_t* allowed, int n, int n_classes, int* err, cudaStream_t st);
void td_launch_clash_guidance(const TdStepArgs& A, const TdGuideArgs& G, int n_graphs, cudaStream_t st);
void td_launch_connect_guidance(const TdStepArgs& A, const TdConnectArgs& C, int n_graphs, cudaStream_t st);
void td_launch_renoise(const TdStepArgs& A, cudaStream_t st);
void td_launch_fixed_init(const TdStepArgs& A, cudaStream_t st);
void td_launch_start_init(const TdStepArgs& A, cudaStream_t st);
void td_launch_likelihood_init(const TdLikelihoodArgs& L, cudaStream_t st);
void td_launch_likelihood_epilogue(const TdLikelihoodArgs& L, cudaStream_t st);
void td_launch_set_fixed(const unsigned char* mask, const float* pos, const long long* v, const int* lig_graph, const float4* offset,
                         int apply_center, int n, int n_classes, unsigned char* fix_mask, float4* fix_pos, int* fix_v, int* err,
                         cudaStream_t st);
void td_launch_segment_mean3(const float* pos, const int* seg_ptr, int n_seg, float4* out, cudaStream_t st);
void td_launch_place_protein(const float* pos, const int* prot_node, const int* prot_graph, const float4* offset, int n, float4* xm0,
                             float4* xm1, cudaStream_t st);
void td_launch_park_ligand(float4* lig_pos, int* lig_v, int n, cudaStream_t st);
void td_launch_set_ligand(const float* pos, const long long* v, const int* lig_graph, const float4* offset, int apply_center, int n,
                          int n_classes, float4* lig_pos, int* lig_v, int* err, cudaStream_t st);
void td_launch_get_ligand(const float4* lig_pos, const int* lig_v, const int* lig_graph, const float4* offset, int add_offset, int n,
                          float* pos, long long* v, cudaStream_t st);
void td_launch_scatter_ligand_pos(const float4* lig_pos, const int* lig_node, int n, float4* xm, cudaStream_t st);
void td_launch_gather_xyz(const float4* xm, const int* idx, int n, float* out, cudaStream_t st);
void td_launch_pack_xyzm(const float* x, const unsigned char* mask, int n, float4* xm, cudaStream_t st);
void td_launch_edge_count_scan(const int* src, int n_nodes, int k, long long* node_off, long long* total, cudaStream_t st);
void td_launch_edge_compact(const int* src, const float* e_w, int n_nodes, int k, const long long* node_off, const long long* total,
                            long long* edge_index, float* ew_out, cudaStream_t st);
