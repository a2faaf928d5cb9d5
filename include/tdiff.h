/* tdiff.h -- C-ABI of libtdiff.so: the H100 (sm_90a) engine for targetdiff's denoising-sampling hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8(b)).  The reference is pure Python; the "FFI" a maintainer
 * binds is ctypes (see INTEGRATION.md).  Each entry point names the reference interface it replaces
 * (paths relative to the reference tree).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch types.
 *   - `d_` arguments are DEVICE pointers owned by the caller; `h_` arguments are HOST pointers.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream).  Calls are asynchronous on it
 *     unless stated otherwise.
 *   - every function returns 0 on success or a negative TDIFF_E* code; tdiff_last_error() gives the text.
 *     Nothing throws across the ABI.  One engine per device; an engine is not thread-safe.
 *   - there is NO CPU fallback: without a CUDA device tdiff_create fails with TDIFF_ECUDA.
 *   - node order everywhere is the reference's `compose_context` order (models/common.py:120-137):
 *     per graph, protein atoms (input order) then ligand atoms (input order).  `batch_protein`/`batch_ligand`
 *     must be sorted ascending (they are in scripts/sample_diffusion.py:42,50), expressed here as per-graph counts.
 */
#ifndef TDIFF_H_
#define TDIFF_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define TDIFF_API __attribute__((visibility("default")))
#else
#define TDIFF_API
#endif

#define TDIFF_OK 0
#define TDIFF_EINVAL (-1)   /* bad argument / unsupported configuration */
#define TDIFF_ECUDA (-2)    /* CUDA runtime error (no device, launch failure, out of memory) */
#define TDIFF_ESTATE (-3)   /* call order violated (e.g. forward before bind_batch) */
#define TDIFF_EWEIGHT (-4)  /* missing / mis-shaped state_dict entry */

typedef struct tdiff_engine tdiff_engine;

/* Model hyper-parameters: the keys of reference configs/training.yml:9-42 that shape the network
 * (read at models/molopt_score_model.py:13-33,205-305).  Unsupported values are rejected with TDIFF_EINVAL. */
typedef struct tdiff_config {
  int32_t hidden_dim;        /* 128 (only value supported by the kernels) */
  int32_t n_heads;           /* 16 */
  int32_t num_layers;        /* 9 (any >= 1) */
  int32_t knn;               /* k of the k-NN graph, 1..64 (32 default, 48 stress) */
  int32_t num_r_gaussian;    /* 20 (the reference's fixed offsets, models/common.py:15) */
  int32_t num_classes;       /* ligand_atom_feature_dim, 13 */
  int32_t protein_feat_dim;  /* protein_atom_feature_dim, 27 */
  int32_t num_timesteps;     /* num_diffusion_timesteps, 1000 */
  int32_t model_mean_type;   /* 0 = 'C0' (network predicts x0), 1 = 'noise' (x0 from the predicted displacement,
                              * reference models/molopt_score_model.py:419-422,663-666) */
  int32_t num_blocks;        /* 0 or 1: one block; n > 1: the k-NN graph is rebuilt from the updated coordinates and the SAME layers run
                              * again, n times in total (models/uni_transformer.py:306-321) */
  int32_t ew_net_type;       /* edge gate: 0 'global' (one MLP gate per forward, :312-316), 1 'r' (per sub-layer Linear(r_feat) -> sigmoid,
                              * :58-59,121-122), 2 'm' (x2h: Linear(value) -> sigmoid, h2x: 1, :60-61,123-124), 3 'none' (1) */
  int32_t x2h_out_fc;        /* 1: node_output MLP on [aggregate | h] before the residual (:39-40,80-81) */
  int32_t time_emb;          /* 0: time_emb_dim = 0; 1: time_emb_mode 'simple', one extra ligand input column time_step / T
                              * (models/molopt_score_model.py:319-324); 'sin' cannot run in the reference itself (:325-326) */
  int32_t cutoff_mode;       /* 0 'knn' (models/uni_transformer.py:279-280); 1 'hybrid' (:281-283 -> models/common.py:165-212, add_p_index):
                              * a ligand destination gets every other ligand atom of its graph + its knn nearest protein atoms, protein
                              * destinations keep the k-NN over all atoms.  Needs knn + max ligand atoms per graph - 1 <= 64 slots and
                              * >= knn protein atoms per graph (checked at tdiff_bind_batch).  'radius' is a dead path in the reference */
  int32_t sublayers;         /* layer form of every attention layer (models/uni_transformer.py:143-210; keys num_x2h, num_h2x, sync_twoup
                              * of configs/training.yml:38-42).  0: the reference default, num_x2h = num_h2x = 1, sync_twoup = False;
                              * otherwise 1 << 24 | sync_twoup << 16 | num_h2x << 8 | num_x2h, with num_x2h, num_h2x in 0..16 and
                              * sync_twoup in 0..1.  A layer runs num_x2h feature updates in sequence on the layer's input coordinates,
                              * then num_h2x coordinate updates, each reading the x2h output (sync_twoup = 0) or the layer's input h
                              * (sync_twoup = 1) and the edge lengths of the coordinates the previous one moved; the layer's h is the
                              * x2h output.  State_dict keys ...x2h_layers.i.* / ...h2x_layers.i.* for every i (TDIFF_EWEIGHT if absent) */
  int32_t reserved[1];       /* must be 0 */
} tdiff_config;

/* One state_dict entry (reference key name, fp32, host memory).  SURVEY.md Appendix D lists the 384 keys. */
typedef struct tdiff_tensor {
  const char* name;
  const float* data;
  int64_t numel;
} tdiff_tensor;

/* ---- engine life cycle ------------------------------------------------------------------------------
 * Replaces: ScorePosNet3D.__init__ + load_state_dict (models/molopt_score_model.py:200-311,
 * scripts/sample_diffusion.py:158-163).  Copies and re-packs the weights for the kernels (first-layer split of the
 * [128,340] edge-MLP matrices into type / gaussian / h_dst / h_src blocks, transposes for the GEMM B operand). */
TDIFF_API int tdiff_create(const tdiff_config* cfg, const tdiff_tensor* h_state_dict, int n_entries, int device, tdiff_engine** out);
TDIFF_API void tdiff_destroy(tdiff_engine* e);
TDIFF_API const char* tdiff_last_error(void);
TDIFF_API const char* tdiff_version(void);

/* ---- batch binding -----------------------------------------------------------------------------------
 * Replaces: Batch.from_data_list(...).to(device) + center_pos + the step-invariant half of forward
 * (scripts/sample_diffusion.py:42, models/molopt_score_model.py:110-120,333-347).
 * h_protein_counts / h_ligand_counts: atoms per graph [n_graphs].  d_protein_pos [Np,3], d_protein_feat [Np,F] fp32.
 * center_mode: 0 'none', 1 'protein' (subtract the per-graph protein centroid; scatter_mean semantics).
 * State across calls: a bind clears the ligand state, the fixed set and its tape, the start and its tapes, and every cache of the
 * previous batch, and sets the time (tdiff_set_time) to 0; a refused bind (TDIFF_EINVAL) changes nothing, and the batch bound before
 * stays usable.  tdiff_set_ligand replaces the ligand state; a chain advances it and leaves the time at its last step's; tdiff_forward
 * reads both and changes neither.  The fixed set, the start and the borrowed
 * tapes persist across chains and tdiff_set_ligand until they are cleared or the next bind.  The caches (the previous forward's graph
 * and edge gates, the ligand-free features built by the first chain, the protein-only neighbour keys) are exact: a call gives the same
 * bits on a reused engine as on a fresh one bound to the same batch and given the same ligand state. */
TDIFF_API int tdiff_bind_batch(tdiff_engine* e, int n_graphs, const int32_t* h_protein_counts, const int32_t* h_ligand_counts,
                     const float* d_protein_pos, const float* d_protein_feat, int center_mode, void* stream);

/* Set the ligand state.  d_ligand_pos [Nl,3] fp32 (lab frame if apply_center!=0, already centred otherwise),
 * d_ligand_v [Nl] int64 class indices (checked < num_classes like models/molopt_score_model.py:125). */
TDIFF_API int tdiff_set_ligand(tdiff_engine* e, const float* d_ligand_pos, const int64_t* d_ligand_v, int apply_center, void* stream);
/* Read the ligand state back; add_offset!=0 adds the pocket centroid (models/molopt_score_model.py:695). */
TDIFF_API int tdiff_get_ligand(tdiff_engine* e, float* d_ligand_pos, int64_t* d_ligand_v, int add_offset, void* stream);
/* Per-graph centring offset [n_graphs,3] (zeros for center_mode 0). */
TDIFF_API int tdiff_get_offset(tdiff_engine* e, float* d_offset, void* stream);

/* Time step of every graph for the next tdiff_forward, as time_step / num_timesteps (fp32, device, [n_graphs]); only read when the
 * engine was created with time_emb = 1 (models/molopt_score_model.py:319-324).  tdiff_sample sets it itself every step. */
TDIFF_API int tdiff_set_time(tdiff_engine* e, const float* d_time_norm, void* stream);

/* ---- one network evaluation ----------------------------------------------------------------------------
 * Replaces: ScorePosNet3D.forward (models/molopt_score_model.py:313-368) for time_emb_dim=0 on the bound batch and
 * current ligand state.  Outputs (any may be NULL): d_pred_pos [Nl,3] (centred frame), d_pred_logits [Nl,K],
 * d_final_h [N,128] (composed node order).  fix_x!=0 freezes coordinates (fetch_embedding, :619-631).
 * Does not modify the ligand state. */
TDIFF_API int tdiff_forward(tdiff_engine* e, float* d_pred_pos, float* d_pred_logits, float* d_final_h, int fix_x, void* stream);

/* tdiff_forward plus the per-block outputs of forward(..., return_all=True) (models/molopt_score_model.py:360-367,
 * models/uni_transformer.py:303-327), for B = num_blocks: d_block_pos [(B+1),Nl,3] the ligand coordinates before block 0 and after
 * every block, d_block_logits [(B+1),Nl,K] the v_inference head applied to the ligand rows of h at the same points (entry 0: the
 * initial embeddings).  Entry B equals d_pred_pos / d_pred_logits.  Either may be NULL; the other outputs as tdiff_forward. */
TDIFF_API int tdiff_forward_blocks(tdiff_engine* e, float* d_pred_pos, float* d_pred_logits, float* d_final_h, int fix_x, float* d_block_pos,
                                   float* d_block_logits, void* stream);

/* Graph of the most recent forward: number of edges, and edge_index as int64 [2,E] (row 0 = src/neighbour,
 * row 1 = dst/query), bit-compatible with PyG knn_graph(flow='source_to_target') (models/uni_transformer.py:280).
 * tdiff_num_edges synchronises the stream. */
TDIFF_API int64_t tdiff_num_edges(tdiff_engine* e, void* stream);
TDIFF_API int tdiff_get_edge_index(tdiff_engine* e, int64_t* d_edge_index, void* stream);
/* Intermediate state of the most recent forward for parity tests: x after layer `layer` ([N,3]); e_w per edge
 * (compacted, [E]). */
TDIFF_API int tdiff_get_edge_weight(tdiff_engine* e, float* d_e_w, void* stream);
TDIFF_API int tdiff_get_node_pos(tdiff_engine* e, float* d_x, void* stream);

/* ---- the sampling loop ---------------------------------------------------------------------------------
 * Replaces: ScorePosNet3D.sample_diffusion's loop body x num_steps (models/molopt_score_model.py:649-693), C0 mode.
 * Time sequence t = T-1 ... T-num_steps (:649).  Noise: if d_pos_noise/d_v_uniform are non-NULL they are the tape
 * ([num_steps,Nl,3] / [num_steps,Nl,K], reference draw order randn_like then rand_like); otherwise counter-based
 * Philox4x32-10 keyed by `seed`.  Trajectory outputs (each may be NULL), written on device, zero host syncs:
 *   d_pos_traj [S,Nl,3] fp32 (lab frame, :691-692), d_v_traj [S,Nl] int64 (:693),
 *   d_v0_traj [S,Nl,K] (log_softmax of logits, :687), d_vt_traj [S,Nl,K] (log posterior, :688).
 * pos_only!=0 keeps atom types fixed (:681).  The ligand state is advanced in place (read it with tdiff_get_ligand).
 * The whole step is captured once into a CUDA graph and replayed. */
TDIFF_API int tdiff_sample(tdiff_engine* e, int num_steps, const float* d_pos_noise, const float* d_v_uniform, uint64_t seed,
                 float* d_pos_traj, int64_t* d_v_traj, float* d_v0_traj, float* d_vt_traj, int pos_only, void* stream);

/* Fixed atoms (fragment-conditioned sampling; an extension beyond the reference, DESIGN.md section 1).  Ligand atoms with
 * d_mask[a] != 0 are held to the forward process of a target (x0_f, v0_f) through every later tdiff_sample: before the first step
 * they are set to a sample of q(x_{T-1} | x0_f), q(v_{T-1} | v0_f); after the step at time t (whose network sees every atom and
 * whose posterior update runs for every row) they are overwritten with a fresh sample of q(x_{t-1} | x0_f), q(v_{t-1} | v0_f), or
 * with x0_f, v0_f exactly after t = 0.  Position sqrt(alphas_cumprod) x0_f + sqrt(1 - alphas_cumprod) eps; type Gumbel-max over
 * q_v_pred(log_onehot(v0_f)).  d_pos_traj / d_v_traj record the state after the overwrite, d_v0_traj / d_vt_traj what the network and
 * the posterior produced.  With pos_only the types of every row are left as they are.  tdiff_forward and the other calls ignore it.
 * d_mask [Nl] uint8, or NULL to clear the set; d_pos0 [Nl,3] fp32 (lab frame if apply_center != 0, centred otherwise) and d_v0 [Nl]
 * int64 are read at masked rows only (class >= num_classes -> TDIFF_EINVAL and no fixed set, until a valid call sets one; synchronises
 * the stream).  Before tdiff_bind_batch ->
 * TDIFF_ESTATE; tdiff_bind_batch clears the set.  Costs one extra launch per chain and none per step.
 * Noise: without tapes, draw d (d = 0 before the first step, d = j + 1 after step j) comes from the same Philox key as the sampler
 * on its own counters (a, d, 0, 0x66787073) for positions and (a, d, 1 + c/4, 0x66787476) for class c; the free atoms' stream is
 * unchanged.  tdiff_set_fixed_tape gives those draws as a tape instead: d_pos_noise [S+1,Nl,3], d_v_uniform [S+1,Nl,K] (NULL under
 * pos_only) for the next chains of num_steps = S (borrowed pointers, NULL clears, tdiff_bind_batch clears).  With a fixed set, a chain
 * takes either both tapes or neither (TDIFF_EINVAL otherwise), so the two sources of noise are never mixed. */
TDIFF_API int tdiff_set_fixed(tdiff_engine* e, const uint8_t* d_mask, const float* d_pos0, const int64_t* d_v0, int apply_center,
                              void* stream);
TDIFF_API int tdiff_set_fixed_tape(tdiff_engine* e, const float* d_pos_noise, const float* d_v_uniform);

/* Respaced sampling (an extension beyond the reference, DESIGN.md section 1): the chain of tdiff_sample on a time sequence
 * h_time_seq[0..S-1] (host memory, S = num_steps), integers tau_0 > tau_1 > ... > tau_{S-1} >= 0 with tau_0 = T - 1 and 1 <= S <= T.
 * Step s evaluates the network at t = tau_s, exactly as tdiff_sample does at t, and moves the state to time p = tau_{s+1}, or to
 * p = tau_{S-1} - 1 at the last step (the decoder step, sigma = 0, when tau_{S-1} = 0: a sequence that ends at 0 finishes the molecule).
 *   Unit steps (p = t - 1) use the checkpoint's tables at t, so T-1, ..., 0 is tdiff_sample(T) and T-1, ..., T-S is tdiff_sample(S),
 *   bit for bit.
 *   Jump steps (p < t - 1) use the exact posteriors q(x_p | x_t, x0), q(v_p | v_t, v0).  With abar = alphas_cumprod, a = abar_t / abar_p:
 *     x_p = c0 x0 + ct x_t + sigma eps, c0 = sqrt(abar_p) (1 - a) / (1 - abar_t), ct = sqrt(a) (1 - abar_p) / (1 - abar_t),
 *     sigma^2 = (1 - abar_p) (1 - a) / (1 - abar_t);
 *     log q(v_p | v_t, v0) = normalise[log_add_exp(log v0 + lcabar_v[p], l1mcabar_v[p] - log K)
 *                                      + log_add_exp(log v_t + lambda, log(1 - e^lambda + 1e-40) - log K)],
 *     lambda = sum_{i = p+1..t} log_alphas_v[i].
 *   The host computes these in double from the fp32 'betas' (1 - abar = -expm1(sum log1p(-beta))) and 'log_alphas_v' tables and
 *   rounds each to fp32 once; the tables are uploaded before the chain (one stream synchronisation).
 * Everything else is tdiff_sample's: tapes [S,Nl,...] and Philox counters keyed by the step index s, trajectories [S,...] (entry s is
 * the state after step s, at time p), the same launches per step, one captured graph.  Fixed atoms (tdiff_set_fixed): after step s
 * the fixed rows get a sample at p from draw s + 1 (the fixed tape is [S+1,Nl,...]), or x0_f / v0_f after the step at tau_{S-1} = 0.
 * A time embedding sees tau_s / T.  A NULL, empty, too long, not strictly decreasing or negative sequence, or one not starting at
 * T - 1 -> TDIFF_EINVAL. */
TDIFF_API int tdiff_sample_seq(tdiff_engine* e, const int32_t* h_time_seq, int num_steps, const float* d_pos_noise, const float* d_v_uniform,
                               uint64_t seed, float* d_pos_traj, int64_t* d_v_traj, float* d_v0_traj, float* d_vt_traj, int pos_only,
                               void* stream);

/* Resampled sampling on a time path (an extension beyond the reference, DESIGN.md section 1; RePaint, Lugmayr et al. 2022): the chain
 * may re-noise the ligand with the forward process between denoising steps.  A time path tau_0, ..., tau_{S-1} has every tau_s in
 * 0..T-1, tau_0 = T - 1 (t_start while a start is armed, tdiff_set_start), tau_{s+1} != tau_s, tau_1 < tau_0 when S > 1, and
 * 1 <= S <= TDIFF_PATH_MAX_PER_T * T.  Step s moves the state from t = tau_s to p = tau_{s+1}, or to tau_{S-1} - 1 at the last step.
 *   Denoising step (p < t): tdiff_sample_seq's step, bit for bit (network at t, unit or jump posterior, fixed rows resampled at p); a
 *   strictly decreasing path is tdiff_sample_seq's chain.
 *   Re-noising step (p > t): no network and no time-embedding update.  Every row that is not fixed: x_p = c x_t + d eps with
 *   c = sqrt(abar_p / abar_t), d = sqrt(1 - abar_p / abar_t) computed in double (log(abar_p / abar_t) = sum_{i = t+1..p} log1p(-beta_i),
 *   1 - abar_p / abar_t = -expm1 of it), rounded to fp32 once each, each product and the sum rounded once; the type by Gumbel-max over
 *   log q(v_p | v_t) = log_add_exp(log_onehot(v_t) + lambda, log(1 - e^lambda + 1e-40) - log K), lambda = sum_{i = t+1..p}
 *   log_alphas_v[i] (log_alphas_v[p] and log_one_minus_alphas_v[p] on a unit step, p = t + 1), log_onehot clamped at 1e-30; with
 *   pos_only the type stays.  Fixed rows (tdiff_set_fixed) get a sample of q(x_p | x0_f), q(v_p | v0_f) from draw s + 1, as after a
 *   denoising step.  2 launches.
 * Noise: step s of either kind reads row s of the tapes [S,Nl,...], or the Philox counters of step s, so a path of S steps uses the
 * stream of any S-step chain; the fixed tape is [S+1,Nl,...].  Trajectories [S,...], entry s the state after step s: pos_traj and
 * v_traj the state (fixed rows as held); vt_traj the normalised log-probabilities the type was drawn from; v0_traj the network's
 * log_softmax at denoising steps, and after a re-noising step a copy of entry s - 1 (the latest network prediction).
 * Works with tdiff_set_fixed, tdiff_set_start, tapes, pos_only, the time embedding and every layer form.  A NULL or empty path, a
 * wrong tau_0, equal neighbours, a time outside 0..T-1, an upward first step or a path over the limit -> TDIFF_EINVAL. */
#define TDIFF_PATH_MAX_PER_T 64
TDIFF_API int tdiff_sample_path(tdiff_engine* e, const int32_t* h_time_path, int num_steps, const float* d_pos_noise, const float* d_v_uniform,
                                uint64_t seed, float* d_pos_traj, int64_t* d_v_traj, float* d_v0_traj, float* d_vt_traj, int pos_only,
                                void* stream);

/* Clash guidance (an extension beyond the reference, DESIGN.md section 1): at every denoising step of every following chain
 * (tdiff_sample, tdiff_sample_seq, the denoising steps of tdiff_sample_path), the step's x0 prediction y of each ligand atom (after the
 * 'noise' mean type's conversion; centred frame) is replaced by
 *   y + strength * sum_p (radius - d) (y - x_p) / d,   d = |y - x_p|,
 * over the protein atoms p of the same graph at their bound positions x_p with 0 < d < radius -- y - (strength / 2) grad E(y) for
 * E(y) = sum_p max(0, radius - |y - x_p|)^2.  An atom without such a pair keeps y bit for bit.  The step then runs unchanged on the
 * guided prediction (posterior, noise, types, fixed-row overwrite, trajectories); fixed rows are guided and then overwritten as before.
 * fp32; every sum runs over the graph's own protein atoms in bind order, so a graph gets the same bits in any batch.  No random numbers
 * are drawn.  One more launch per denoising step; re-noising steps, tdiff_forward, tdiff_forward_blocks and tdiff_likelihood_terms
 * ignore the setting.  strength == 0 turns guidance off (radius is then ignored); strength > 0 needs a finite radius > 0 (Angstrom).  A
 * negative or non-finite strength, or a bad radius with strength > 0 -> TDIFF_EINVAL and the previous setting stays.  The setting
 * belongs to the handle: it refers to no batch rows, so it survives tdiff_bind_batch.  Off on a new handle. */
TDIFF_API int tdiff_set_clash_guidance(tdiff_engine* e, float radius, float strength);

/* Connectivity guidance (an extension beyond the reference, DESIGN.md section 1): at every denoising step of every following chain
 * (tdiff_sample, tdiff_sample_seq, the denoising steps of tdiff_sample_path; after clash guidance when both are on), the step's x0
 * predictions y of each graph's ligand atoms (centred frame) are moved so that the molecule's separate pieces come closer.  Ligand atoms
 * a, c of a graph are bonded when |q_a - q_c| < radius, where q is y, or the target position x0_f for a fixed row (tdiff_set_fixed).
 * With one connected component every atom keeps y bit for bit.  Otherwise each component C finds its closest outside pair (i in C,
 * j not in C; smallest d = |q_i - q_j|, then the lowest within-graph (i, j)); a component with a fixed row stays, and every other one
 * moves rigidly: each of its atoms gets y + f (q_j - q_i), f = (strength * w * (d - bond_length)) / d, w = 1 when j's component has a
 * fixed row and 1/2 otherwise, all shifts from the unshifted predictions.  d^2 = (dx dx + dy dy) + dz dz, d = sqrt(d^2), every comparison,
 * f and each coordinate of the shift are explicitly rounded fp32 operations, and every decision reads the graph's own atoms, so a graph
 * gets the same bits in any batch.  The step then runs unchanged on the guided prediction; fixed rows keep their prediction and are
 * overwritten as before.  No random numbers are drawn.  One more launch per denoising step; re-noising steps, tdiff_forward,
 * tdiff_forward_blocks and tdiff_likelihood_terms ignore the setting.  A chain with more than TDIFF_CONNECT_MAX_ATOMS ligand atoms in a
 * graph while guidance is on -> TDIFF_EINVAL before anything runs.  strength == 0 turns guidance off (radius and bond_length are then
 * ignored); strength > 0 needs finite radius > 0 and 0 < bond_length < radius (Angstrom).  A negative or non-finite strength, or a bad
 * radius or bond length with strength > 0 -> TDIFF_EINVAL and the previous setting stays.  The setting belongs to the handle: it
 * survives tdiff_bind_batch.  Off on a new handle. */
#define TDIFF_CONNECT_MAX_ATOMS 1024
TDIFF_API int tdiff_set_connect_guidance(tdiff_engine* e, float radius, float bond_length, float strength);

/* Element constraints (an extension beyond the reference, DESIGN.md section 1): d_allowed [Nl] uint32 (device), bit c of row a set =
 * class c allowed for ligand atom a.  At every denoising step of every following chain (tdiff_sample, tdiff_sample_seq, the denoising
 * steps of tdiff_sample_path, with or without clash guidance) the type head's log_softmax runs over the allowed classes only (the
 * others get log v0_hat = -inf: the prediction conditioned on v0 in the set), and the posterior runs unchanged on it.  On the decoder
 * step (target time p < 0: t = 0 of the default chain, or a sequence or path ending at 0) the posterior is also renormalised over the
 * allowed set, so that the draw picks an allowed class.  The intermediate states are drawn from the whole posterior (the forward
 * marginals have mass on every class), so a chain that stops before t = 0 may end in a forbidden class.  v0_traj holds the conditioned
 * log v0_hat and vt_traj the distribution each state was drawn from, -inf at forbidden entries where that is their value.  A mask
 * that allows every class gives the unconstrained chain's bits.  No random numbers are drawn; no launch is added per step.  Fixed rows
 * (tdiff_set_fixed) are overwritten as before.  Re-noising steps, the start and fixed-row draws, tdiff_forward, tdiff_forward_blocks
 * and tdiff_likelihood_terms ignore the mask.  NULL clears it.  A row without a class or with a bit at or above num_classes ->
 * TDIFF_EINVAL and the previous mask stays (synchronises the stream).  A chain with pos_only while a mask is set -> TDIFF_EINVAL.
 * Before tdiff_bind_batch -> TDIFF_ESTATE; tdiff_bind_batch clears the mask. */
TDIFF_API int tdiff_set_type_mask(tdiff_engine* e, const uint32_t* d_allowed, void* stream);

/* Start-ligand sampling (an extension beyond the reference, DESIGN.md section 1): arms the next chains to start from the current ligand
 * state (the start ligand x0, v0, centred like any ligand) noised to the start time t_start in 0..T-1, and to run the reverse chain
 * from there; t_start = -1 clears it.  The current ligand state is the one tdiff_set_ligand set or, after a chain, that chain's
 * output: a second chain without tdiff_set_ligand in between re-noises the first chain's result, not the start ligand.  Set the
 * start ligand again before each chain to draw several samples from it.  While a start is armed:
 *   the chain runs through tdiff_sample_seq only, and its time sequence must begin at tau_0 = t_start (the unit sequence
 *   t_start, ..., 0 has t_start + 1 steps; a respaced one is allowed); tdiff_sample -> TDIFF_EINVAL.  Without a start
 *   tdiff_sample_seq keeps requiring tau_0 = T - 1.
 *   Before the first step, one launch (in place of the fixed set's) replaces every row: fixed rows (tdiff_set_fixed) by the sample
 *   the fixed set gives them at t_start (draw 0 of the fixed-atom stream or tape); the others by a sample of q(x_{t_start} | x0),
 *   q(v_{t_start} | v0) -- sqrt(alphas_cumprod[t_start]) x0 + sqrt(1 - alphas_cumprod[t_start]) eps with each product and the sum
 *   rounded once, and Gumbel-max over q_v_pred(log_onehot(v0), t_start) -- the fixed set's formulas.  With pos_only the types stay
 *   as set.  The steps are tdiff_sample_seq's, with the same launches.
 * Noise: without tapes, the start draw of atom a comes from the sampler's Philox key on its own counters (a, 0, 0, 0x73747073 "stps")
 * for positions and (a, 0, 1 + c/4, 0x73747476 "sttv") for class c; the sampler's and the fixed set's streams are unchanged.
 * d_pos_noise [Nl,3] and d_v_uniform [Nl,K] (NULL under pos_only) give the start draw as a tape instead (borrowed pointers).  A chain
 * takes either all of its tapes (step, fixed, start) or none (TDIFF_EINVAL otherwise).  Before tdiff_bind_batch -> TDIFF_ESTATE;
 * t_start outside -1..T-1 -> TDIFF_EINVAL; tdiff_bind_batch clears the start. */
TDIFF_API int tdiff_set_start(tdiff_engine* e, int t_start, const float* d_pos_noise, const float* d_v_uniform);

/* Likelihood scoring (the variational bound of scripts/likelihood_est_diffusion.py, batched over graphs; DESIGN.md section 1).  The
 * current ligand state is the clean ligand (x0, v0); bind with center_mode 1 ('protein') as the reference's likelihood_estimation does.
 * Graph g is scored at h_time_steps[g] = t_g in 0..T-1 (host memory):
 *   x_t = sqrt(abar) x0 + sqrt(1 - abar) eps, abar = alphas_cumprod[t_g], each product and the sum rounded once, and v_t by Gumbel-max
 *   over q_v_pred(log_onehot(v0), t_g) -- the formulas and guards of the fixed set's and the start's draws;
 *   the forward (fix_x = 0) on (x_t, v_t), a time embedding seeing t_g / T divided in fp32;
 *   per ligand atom, the reference's terms (models/molopt_score_model.py:588-617): positions KL(q(x_{t-1} | x_t, x0) || p) / log 2 for
 *   t_g > 0 and the decoder NLL (in nats) at t_g = 0; types categorical_kl(log_true, log_model) for t_g > 0 and
 *   -log_categorical(log_onehot(v0), log_model) at t_g = 0; and the prior terms at T - 1 (kl_pos_prior, kl_v_prior, :411-438) with the
 *   ligand's own types, for every graph;
 *   per graph, the mean of each term over its ligand atoms (summed in atom order in fp32; 0 for a graph without ligand atoms).
 * Outputs (device, each may be NULL): d_kl_pos, d_kl_v, d_prior_pos, d_prior_v [B]; d_atom_kl_pos, d_atom_kl_v [Nl]; d_xt [Nl,3]
 * (centred frame) and d_vt [Nl] int64, the sampled state.  The ligand state is restored to x0, v0; the time embedding is left at t_g / T;
 * the call's forward is the most recent one for tdiff_num_edges / tdiff_get_edge_index (the graph of x_t).  The fixed set and an armed
 * start are ignored, as tdiff_forward ignores them.
 * Noise: without a tape, atom j (its index within graph g) draws from the sampler's Philox key on counters (j, k_g, t_g << 8, 0x6c6b7073
 * "lkps") for positions and (j, k_g, t_g << 8 | (1 + c/4), 0x6c6b7476 "lktv") for class c, so that a graph's draws, and with them its
 * terms, do not depend on the rest of the batch.  h_keys [B] gives k_g (host memory; NULL: k_g = g).  d_pos_noise [Nl,3] and
 * d_v_uniform [Nl,K] replace the draws (both or neither).  Launches: the forward's plus 2.  No host synchronisation beyond the pageable
 * H2D copy of t_g and k_g.  Before bind or set_ligand -> TDIFF_ESTATE; a t_g outside 0..T-1, one half of the tape, or an engine with
 * model_mean_type 1 ('noise', for which the reference raises) -> TDIFF_EINVAL. */
TDIFF_API int tdiff_likelihood_terms(tdiff_engine* e, const int32_t* h_time_steps, const uint32_t* h_keys, const float* d_pos_noise,
                                     const float* d_v_uniform, uint64_t seed, float* d_kl_pos, float* d_kl_v, float* d_prior_pos,
                                     float* d_prior_v, float* d_atom_kl_pos, float* d_atom_kl_v, float* d_xt, int64_t* d_vt, void* stream);

/* Same loop through HOST buffers (the end-to-end path: H2D of the inputs, the chain, D2H of the results, all on
 * `stream`, synchronised before returning).  Equivalent of the device-facing part of sample_diffusion_ligand
 * (scripts/sample_diffusion.py:42-112) for one batch.  h_out_* may be NULL. */
TDIFF_API int tdiff_sample_host(tdiff_engine* e, int n_graphs, const int32_t* h_protein_counts, const int32_t* h_ligand_counts,
                      const float* h_protein_pos, const float* h_protein_feat, const float* h_ligand_pos,
                      const int64_t* h_ligand_v, int center_mode, int num_steps, const float* h_pos_noise,
                      const float* h_v_uniform, uint64_t seed, float* h_out_pos, int64_t* h_out_v, float* h_pos_traj,
                      int64_t* h_v_traj, float* h_v0_traj, float* h_vt_traj, int pos_only, void* stream);

/* ---- stand-alone graph / scatter operators (the reference's native seam, SURVEY.md 8(b)) ----------------
 * tdiff_knn_graph replaces torch_geometric.nn.knn_graph(x, k, batch, flow='source_to_target')
 * (models/uni_transformer.py:280): d_x [N,3], h_graph_counts [n_graphs] nodes per graph (batch sorted).
 * Outputs: d_src_slots [N*k] int32 (neighbour of node i in slots i*k.., ascending (d2,index), -1 padded when the graph
 * has <= k nodes), d_edge_index int64 [2, *n_edges] compacted (may be NULL).  h_n_edges receives E (synchronises). */
TDIFF_API int tdiff_knn_graph(const float* d_x, int n_nodes, const int32_t* h_graph_counts, int n_graphs, int k,
                    int32_t* d_src_slots, int64_t* d_edge_index, int64_t* h_n_edges, void* stream);

/* Fused scatter_softmax -> scatter_sum over a dst-sorted fixed-degree neighbour list (replaces
 * models/uni_transformer.py:73-83): logits[e,h] = sum_d (q[dst,h,d]*k[e,h,d]/sqrt(8)); alpha = softmax over the
 * edges of dst; out[dst] = h_in[dst] + sum_e alpha*v[e]*e_w[e].   d_k,d_v [N*kk,128], d_q,d_h_in,d_h_out [N,128],
 * d_src_slots [N*kk] (-1 = absent edge), d_e_w [N*kk]. */
TDIFF_API int tdiff_attn_aggregate_h(const float* d_k, const float* d_v, const float* d_e_w, const int32_t* d_src_slots,
                           const float* d_q, const float* d_h_in, float* d_h_out, int n_nodes, int kk, void* stream);
/* Coordinate variant (replaces models/uni_transformer.py:131-140 and :205-206): v [N*kk,16] per-head scalars,
 * message alpha*v*e_w*(x[dst]-x[src]), mean over heads, x_out = x + delta*mask.  d_x, d_x_out [N,3]; d_mask [N] uint8. */
TDIFF_API int tdiff_attn_aggregate_x(const float* d_k, const float* d_v16, const float* d_e_w, const int32_t* d_src_slots,
                           const float* d_q, const float* d_x, const uint8_t* d_mask, float* d_x_out, int n_nodes, int kk,
                           void* stream);
/* scatter_mean(src [M,3], index [M] sorted, dim=0) given per-segment counts (models/molopt_score_model.py:115). */
TDIFF_API int tdiff_scatter_mean3(const float* d_src, const int32_t* h_counts, int n_segments, float* d_out, void* stream);

/* Bond-count stability screen of generated molecules (the step after the sampling path: utils/evaluation/analyze.py:106-143
 * `check_stability`, called per molecule by scripts/evaluate_diffusion.py:78-84).  d_pos [n_atoms,3] fp32, d_atomic_num [n_atoms] int32
 * (atomic numbers, utils/transforms.py `get_atomic_number_from_index`), h_counts [n_mol] atoms per molecule.  Outputs (device):
 * d_nr_bonds [n_atoms] summed bond orders (may be NULL), d_stable_atoms [n_mol], d_mol_stable [n_mol] (1 = every atom stable).
 * hs != 0 requires bonds == valence instead of 0 < bonds <= valence.  An atomic number outside the reference's table -> TDIFF_EINVAL
 * (KeyError in the reference).  Synchronises the stream. */
TDIFF_API int tdiff_check_stability(const float* d_pos, const int32_t* d_atomic_num, const int32_t* h_counts, int n_mol, int hs,
                                    int32_t* d_nr_bonds, int32_t* d_stable_atoms, uint8_t* d_mol_stable, void* stream);

/* ---- instrumentation ------------------------------------------------------------------------------------
 * Number of kernel launches issued by this engine since creation (graph replays count their nodes). */
TDIFF_API int64_t tdiff_launch_count(tdiff_engine* e);
/* Edge-MLP execution mode of this engine (env TDIFF_EDGE_MLP at creation): 0 FP32 FFMA ("simt"), 2 wgmma bf16x2 split with keys in HBM
 * ("tc3v2"), 3 wgmma bf16x3 split ("tc6"), 5 wgmma bf16x2 split, gaussian block on the tensor core and attention logits fused into the
 * key-MLP epilogue (default, "tc3"). */
TDIFF_API int tdiff_edge_mlp_mode(tdiff_engine* e);
/* Time (ms, CUDA events on `stream`) and count of the attention-aggregate launches accumulated while profiling is on. */
TDIFF_API int tdiff_profile(tdiff_engine* e, int enable);
TDIFF_API int tdiff_profile_read(tdiff_engine* e, double* ms_aggregate_h, int64_t* n_aggregate_h, double* ms_aggregate_x,
                       int64_t* n_aggregate_x, double* ms_edge_mlp, int64_t* n_edge_mlp, double* ms_total);
/* Node lists of the last sampling step's backward cone (DESIGN.md section 4.3), copied to the host by synchronous copies (call once
 * the step's stream has finished).  h_dims = {G x2h evaluations of the last block, row stride}; then, where not NULL, 2 G class-sorted
 * lists: h_counts [2G,4] = {entries, protein part, protein nodes, -}, h_rows [2G,stride] (-1 = padding; order within a class
 * unspecified); list 2g holds the destinations of evaluation g, list 2g+1 the nodes whose B blocks it computes.  TDIFF_ESTATE when no
 * sampling step has built them since the batch was bound. */
TDIFF_API int tdiff_get_cone(tdiff_engine* e, int32_t* h_dims, int32_t* h_counts, int32_t* h_rows);

#ifdef __cplusplus
}
#endif
#endif /* TDIFF_H_ */
