/* b200nerf.h -- C ABI of libb200nerf.so, the sm_90a backend of NeuRAD's volumetric-rendering hot path.
 *
 * The reference (georghess/neurad-studio) has no FFI of its own: its backend seam is the string flag
 * `NeuRADModelConfig.implementation` (nerfstudio/models/neurad.py:146) that selects tiny-cuda-nn or torch
 * inside HashEncoding / SHEncoding / MLP, and the module-level plugin API Field / Sampler / Renderer /
 * Model.get_nff_outputs.  This header is the C boundary a third backend ("b200") binds: every entry point
 * names the reference interface it replaces.  Conventions (SURVEY.md section 8b):
 *
 *   - The caller (PyTorch) owns every buffer.  All `const float*` / `float*` arguments are DEVICE pointers to
 *     contiguous fp32 arrays unless the name ends in `_host`.  Index outputs are int32.
 *   - `stream` is a `cudaStream_t` passed as `void*` (NULL = the legacy default stream).
 *   - Every function returns 0 on success and a negative code on failure; `b200nerf_last_error()` returns a
 *     thread-local message.  The library never aborts and has no CPU fallback.
 *   - A `b200nerf_ctx` is bound to one device; several contexts (one per GPU) may coexist in one process.
 *     One host thread drives one context at a time (same contract as the reference's single-threaded model).
 *   - Large tables (hash grids, embeddings) are referenced zero-copy and must outlive their use; small tensors
 *     (MLP weights, decoders, actor trajectories) are repacked into library-owned device memory by the
 *     `b200nerf_set_*` calls, so call those again after the parameters change.
 *   - No allocation happens inside `*_fwd` calls.
 */
#ifndef B200NERF_H_
#define B200NERF_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200NERF_VERSION 100
#define B200NERF_MAX_LEVELS 16

enum {
  B200NERF_OK = 0,
  B200NERF_ERR_INVALID = -1,     /* bad argument / unsupported configuration */
  B200NERF_ERR_CUDA = -2,        /* CUDA runtime error (message has the cudaError string) */
  B200NERF_ERR_STATE = -3,       /* a required b200nerf_set_* call is missing */
  B200NERF_ERR_UNSUPPORTED = -4  /* valid in the reference, not implemented here yet */
};

typedef struct b200nerf_ctx b200nerf_ctx;

/* field selector: NeuRADModel.field / NeuRADModel.proposal_fields[0|1] (neurad.py:180-184, 236-247) */
enum { B200NERF_FIELD_MAIN = 0, B200NERF_FIELD_PROP0 = 1, B200NERF_FIELD_PROP1 = 2 };

/* HashEncoding hyper-parameters + its `scalings` buffer (field_components/encodings.py:326-352). */
typedef struct {
  int32_t num_levels;
  int32_t features_per_level;
  int32_t log2_hashmap_size;
  float scalings[B200NERF_MAX_LEVELS];
} b200nerf_grid_desc;

/* tiny-cuda-nn `HashGrid` encoding layout -- what `HashEncoding(implementation="tcnn")` instantiates (encoding_config at
 * field_components/encodings.py:386-401: n_levels, n_features_per_level, log2_hashmap_size, base_resolution = min_res,
 * per_level_scale = growth_factor; `n_input_dims` 3, or 4 for the shared actor grid, neurad_encoding.py:110-131).  The caller
 * computes the per-level constants (neurad-studio_b200/tcnn_compat.py: grid_layout): position scale (pos = fma(x, scale,
 * 0.5)), vertices per axis, first entry and entry count in the flat parameter vector, and whether the level indexes linearly
 * (res^n_dims fits) or hashes.  `scalings` is HashEncoding.scalings, which NeuRAD's anti-aliasing weights use in both modes
 * (neurad_encoding.py:297-304).  PARITY UNPINNED: tiny-cuda-nn is absent here (oracle/tcnn_oracle.py). */
typedef struct {
  int32_t num_levels;
  int32_t features_per_level;
  int32_t n_input_dims;
  float scale[B200NERF_MAX_LEVELS];
  uint32_t resolution[B200NERF_MAX_LEVELS];
  uint32_t offset[B200NERF_MAX_LEVELS];
  uint32_t size[B200NERF_MAX_LEVELS];
  uint8_t dense[B200NERF_MAX_LEVELS];
  float scalings[B200NERF_MAX_LEVELS];
} b200nerf_tcnn_grid_desc;

const char* b200nerf_last_error(void);
int b200nerf_version(void);

int b200nerf_create(int device_ordinal, b200nerf_ctx** out);
int b200nerf_destroy(b200nerf_ctx* ctx);

/* ---- parameters --------------------------------------------------------------------------------------- */

/* The stream the b200nerf_set_* entry points issue their packing kernels and device-to-device copies on (default: the
 * legacy default stream).  Bind the stream the parameters were last written on -- e.g. torch's current stream after an
 * optimizer step -- and renders launched on the same stream see the new parameters in order; nothing synchronises the
 * device (b200nerf_set_rgb_decoder alone waits for this stream before it returns). */
int b200nerf_set_param_stream(b200nerf_ctx* ctx, void* stream);

/* NeuRADHashEncoding of one field (field_components/neurad_encoding.py:85-131): the static grid
 * `static_grid.hash_table` [L*T, F] and, in torch mode, one 3-D grid per actor `actor_grids[i].hash_table`.
 * `actor_tables_host` is a HOST array of `n_actors` device pointers (NULL when n_actors == 0).
 * `static_scale` = scene_box.aabb.max() (neurad.py:182); `actor_scale` = ActorSettings.actor_scale. */
int b200nerf_set_field_grids(b200nerf_ctx* ctx, int field, const b200nerf_grid_desc* static_desc,
                             const float* static_table, const b200nerf_grid_desc* actor_desc,
                             const float* const* actor_tables_host, int n_actors, float static_scale,
                             float actor_scale);

/* The same field from a tcnn-trained checkpoint (SURVEY 8f row f3): `static_params` is `hashgrid.static_grid.tcnn_encoding
 * .params` (flat fp32 master copy, rounded to fp16-representable values by the caller: tiny-cuda-nn casts to half at forward
 * time), `actor_params` the ONE 4-D grid `hashgrid.actor_grids[0].tcnn_encoding.params` shared by all actors
 * (neurad_encoding.py:270-281; NULL when n_actors == 0).  Selects the tcnn kernels for the fused renderer: the main field and
 * the proposal fields used for sampling must then all be bound through this entry point; the SH basis follows tiny-cuda-nn's
 * convention (evaluated at the direction, Condon-Shortley signs).  Bias-free FullyFusedMLP weights are passed to
 * b200nerf_set_main_mlps / b200nerf_set_lidar_decoder with zero biases (tcnn_compat.py unpacks and un-pads them). */
int b200nerf_set_field_grids_tcnn(b200nerf_ctx* ctx, int field, const b200nerf_tcnn_grid_desc* static_desc,
                                  const float* static_params, const b200nerf_tcnn_grid_desc* actor_desc,
                                  const float* actor_params, int n_actors, float static_scale, float actor_scale);

/* Stage operator: tcnn.Encoding{HashGrid}.forward, x [P, n_input_dims] in [0,1] -> out [P, L*F] (level-major). */
int b200nerf_tcnn_hashgrid_fwd(b200nerf_ctx* ctx, const b200nerf_tcnn_grid_desc* desc, const float* params, const float* x,
                               float* out, int64_t n_points, void* stream);

/* NeuRADProposalField.density_decoder = nn.Linear(L*F, 1, bias=False) (fields/neurad_field.py:201). */
int b200nerf_set_proposal_decoder(b200nerf_ctx* ctx, int field, const float* weight, int in_dim);

/* NeuRADField.mlp_geo (in->hidden->1+nff), mlp_feature (nff+16 ->hidden->hidden->nff) as nn.Linear [out,in]
 * weights + biases (fields/neurad_field.py:98-117, field_components/mlp.py:142-157), and the SDF slope
 * `beta = |sdf_to_density.beta| + beta_min` (model_components/utils.py:24-41). */
int b200nerf_set_main_mlps(b200nerf_ctx* ctx, const float* geo_w0, const float* geo_b0, const float* geo_w1,
                           const float* geo_b1, const float* feat_w0, const float* feat_b0, const float* feat_w1,
                           const float* feat_b1, const float* feat_w2, const float* feat_b2, float beta);

/* NeuRADModel.lidar_decoder: MLP 48->32->32->2 (neurad.py:217-224). */
int b200nerf_set_lidar_decoder(b200nerf_ctx* ctx, const float* w0, const float* b0, const float* w1,
                               const float* b1, const float* w2, const float* b2);

/* NeuRADModel.appearance_embedding [num_embeds, dim] with temporal interpolation (neurad.py:187-196,
 * 423-441).  Zero-copy. */
int b200nerf_set_appearance(b200nerf_ctx* ctx, const float* embedding, int num_embeds, int dim,
                            int embeds_per_sensor, float duration);

/* The same embedding with use_temporal_appearance = False (neurad.py:190-195, 440): one row per sensor, and a ray's
 * appearance columns are row `sensor_idx` copied.  Rays without sensor_idx use sensor 0 (the viewer's fallback sensor,
 * neurad.py:425-428), as with b200nerf_set_appearance; sensor indices must be in [0, num_embeds), nothing checks them
 * on the device.  Zero-copy; replaces a binding of b200nerf_set_appearance and vice versa. */
int b200nerf_set_appearance_per_sensor(b200nerf_ctx* ctx, const float* embedding, int num_embeds, int dim);

/* DynamicActors buffers/parameters (model_components/dynamic_actors.py:109-170): unique_timestamps [T],
 * actor_rotations_6d [T,A,6], actor_positions [T,A,3], actor_present_at_time [T,A] (uint8), actor_sizes
 * [A,3]; `padding_host` = actor_bbox_padding (3 floats, host).  n_actors == 0 disables the actor branch. */
int b200nerf_set_actors(b200nerf_ctx* ctx, int n_actors, int n_times, const float* timestamps,
                        const float* rotations_6d, const float* positions, const uint8_t* present,
                        const float* sizes, const float* padding_host);

/* SamplingSettings + ProposalNetworkSampler / PDFSampler constants (neurad.py:101-117,
 * ray_samplers.py:255-376, 569-666).  `u1_host` / `u2_host` are PDFSampler's eval-mode quantiles
 * `linspace(0, 1-1/nb, nb) + 1/(2nb)` for nb = n_prop1+1 and nb = n_nerf+1 (computed by the caller with
 * torch.linspace so they are bit-identical to the reference's).  `density_field_of_round[i]` selects which
 * proposal field round i evaluates: the reference's `density_fns` closures bind late (neurad.py:248), so
 * BOTH rounds evaluate proposal_fields[1]; pass {B200NERF_FIELD_PROP1, B200NERF_FIELD_PROP1} for drop-in
 * behaviour. */
int b200nerf_set_sampling(b200nerf_ctx* ctx, int n_prop0, int n_prop1, int n_nerf, float power_lambda,
                          float power_scaling, float sky_distance, float histogram_padding,
                          const float* u1_host, const float* u2_host, const int* density_field_of_round,
                          float camera_area_scale);

/* ---- the fused path: NeuRADModel.get_nff_outputs (neurad.py:368-421), eval mode ------------------------ */

/* A flat RayBundle (cameras/rays.py:252-275).  Optional members may be NULL. */
typedef struct {
  const float* origins;      /* [N,3] */
  const float* directions;   /* [N,3] */
  const float* pixel_area;   /* [N]   (unscaled; camera rays are scaled by camera_area_scale in-kernel,
                                       NeuRADModel._scale_pixel_area neurad.py:702-709) */
  const float* times;        /* [N]   */
  const float* nears;        /* [N] or NULL -> 0 (neurad.py:449) */
  const float* fars;         /* [N] or NULL -> 1e6, clamped to sky_distance (neurad.py:445-448) */
  const int64_t* sensor_idx; /* [N] or NULL -> fallback sensor 0 (metadata["sensor_idxs"], neurad.py:424-427) */
  const uint8_t* is_lidar;   /* [N] or NULL -> all camera rays (metadata["is_lidar"]) */
  int32_t image_width;       /* 0: no hint.  W > 0: the bundle is a row-major image (or stack of images) with W rays
                                per row; the kernel then walks it in 32x8-pixel tiles (a warp = an 8x4 patch) so that
                                the rays of a warp are neighbours in BOTH image directions.  Results are written at
                                the rays' own indices, i.e. the output order is unchanged. */
} b200nerf_rays;

typedef struct {
  float* features;       /* [N, nff_out_dim + appearance_dim] rendered features ++ appearance embedding */
  float* depth;          /* [N] */
  float* accumulation;   /* [N] */
  float* prop_depth_0;   /* [N] */
  float* prop_depth_1;   /* [N] */
  float* intensity;      /* [N] or NULL: sigmoid(lidar_decoder(features)[0]) (neurad.py:350-357) */
  float* ray_drop_logit; /* [N] or NULL */
} b200nerf_outputs;

/* Peer gather fused into the render epilogue (multi-GPU, one process per GPU): when set, every rendered ray's
 * {features, depth, accumulation} row is ALSO stored, from inside the render kernel, at row `row_offset + ray` of each
 * peer's buffer -- plain st.global on peer-mapped (NVLink / NVSwitch) addresses, e.g. the `buffer_ptrs` of a
 * torch.distributed._symmetric_memory rendezvous.  This replaces the per-image all-gather: the transfer overlaps the
 * rendering tile by tile and no NCCL kernel has to wait for the (persistent, all-SM) render kernel to drain.  The
 * caller still needs a cross-rank barrier before reading.  `self_rank`'s entry is skipped when it equals the local
 * `b200nerf_outputs` slice.  A "peer" may also be pinned, device-mapped HOST memory: the results then stream to the
 * host over PCIe while the kernel is still rendering (no separate device->host copy).  Reference counterpart: none (the reference renders on one device per process,
 * pipelines/ad_pipeline.py:197-306). */
#define B200NERF_MAX_PEERS 16
typedef struct {
  int32_t n_peers;   /* 0 disables */
  int32_t self_rank; /* index into the arrays below that is this rank (skipped), or -1 */
  int64_t row_offset;
  float* features[B200NERF_MAX_PEERS];     /* [rows, nff_out_dim + appearance_dim] */
  float* depth[B200NERF_MAX_PEERS];        /* [rows] */
  float* accumulation[B200NERF_MAX_PEERS]; /* [rows] */
} b200nerf_peer_outputs;

/* Applies to subsequent b200nerf_nff_render_fwd calls of this context; NULL clears it. */
int b200nerf_set_peer_outputs(b200nerf_ctx* ctx, const b200nerf_peer_outputs* peers);

/* Optional per-stage dump used by the parity tests (any member may be NULL). */
typedef struct {
  float* prop_weights_0; /* [N, n_prop0] */
  float* prop_weights_1; /* [N, n_prop1] */
  float* bins_s_1;       /* [N, n_prop1+1] spacing-domain bin edges after resampling round 1 */
  float* bins_e_1;       /* [N, n_prop1+1] euclidean */
  float* bins_s_2;       /* [N, n_nerf+1] */
  float* bins_e_2;       /* [N, n_nerf+1] */
  int32_t* inds_1;       /* [N, n_prop1+1] searchsorted(cdf, u, right) */
  int32_t* inds_2;       /* [N, n_nerf+1] */
  float* sdf;            /* [N, n_nerf] */
  float* alpha;          /* [N, n_nerf] */
  float* field_feature;  /* [N, n_nerf, nff_out_dim] */
  float* weights;        /* [N, n_nerf] (after the sky top-up) */
  int32_t* actor_id_0;   /* [N, n_prop0] actor index per sample or -1 */
  int32_t* actor_id_1;   /* [N, n_prop1] */
  int32_t* actor_id_main;/* [N, n_nerf] */
} b200nerf_trace;

int b200nerf_nff_render_fwd(b200nerf_ctx* ctx, const b200nerf_rays* rays, int64_t n_rays,
                            const b200nerf_outputs* out, const b200nerf_trace* trace, void* stream);

/* ---- stage-level operators (the reference's per-module API) -------------------------------------------- */

/* HashEncoding.forward / pytorch_fwd (encodings.py:425-471): x [P,3] in [0,1] -> out [P, L*F].
 * `indices` (optional) receives the 8 hashed table rows per level, [P, L, 8], in the reference's corner
 * order hashed_0..hashed_7 (encodings.py:436-443). */
int b200nerf_hashgrid_fwd(b200nerf_ctx* ctx, const b200nerf_grid_desc* desc, const float* table, const float* x,
                          float* out, int32_t* indices, int64_t n_points, void* stream);

/* SHEncoding(levels=4).forward (encodings.py:797-805, utils/math.py:31-94): dirs [P,3] -> [P,16]. */
int b200nerf_sh4_fwd(b200nerf_ctx* ctx, const float* dirs, float* out, int64_t n_points, void* stream);

/* MLP.forward (field_components/mlp.py:142-183; the tcnn FullyFusedMLP role, mlp.py:103-113) for NeuRAD's tiny
 * MLPs on the wgmma tensor cores with the 3xTF32 split (fp32-level accuracy): x [n_rows, in_dim] -> y [n_rows,
 * out_dims[n_layers-1]]; ReLU between layers, none at the output.  `weights_host` / `biases_host` are HOST arrays
 * of `n_layers` device pointers in nn.Linear layout ([out,in] / [out]; biases_host or its entries may be NULL).
 * Limits: 1..3 layers, every width <= 64 (<= 48: 48-column tile; wider, e.g. BASELINE config 1's 32 -> 64 -> 4:
 * 64-column tile). */
int b200nerf_mlp_fwd(b200nerf_ctx* ctx, const float* x, int64_t n_rows, int in_dim, int n_layers,
                     const float* const* weights_host, const float* const* biases_host, const int* out_dims_host,
                     float* y, void* stream);
/* The same forward for TRAINING: additionally stores the pre-activations of the hidden layers, hidden_pre_host[l]
 * [n_rows, out_dims[l]] for l < n_layers - 1 (a HOST array of device pointers; entries may be NULL), which the backward
 * (b200nerf_linear_wgrad on ReLU(pre-activation), b200nerf_relu_bwd) needs -- what torch autograd keeps for
 * MLP.forward (mlp.py:142-183) instead of recomputing it. */
int b200nerf_mlp_fwd_train(b200nerf_ctx* ctx, const float* x, int64_t n_rows, int in_dim, int n_layers,
                           const float* const* weights_host, const float* const* biases_host, const int* out_dims_host,
                           float* y, float* const* hidden_pre_host, void* stream);
/* Input gradient of one Linear layer of those MLPs (autograd of F.linear + ReLU, mlp.py:170-178):
 *   dx [n_rows, dx_dim] = dy [n_rows, dy_dim] @ weight_t^T,   weight_t = the layer's nn.Linear weight TRANSPOSED, [dx_dim, dy_dim]
 * and, when relu_z [n_rows, dx_dim] (the pre-activation that fed this layer through ReLU) is given, dx *= (relu_z > 0).
 * Same wgmma 3xTF32 operator as b200nerf_mlp_fwd. */
int b200nerf_mlp_dgrad(b200nerf_ctx* ctx, const float* dy, int64_t n_rows, int dy_dim, const float* weight_t, int dx_dim,
                       const float* relu_z, float* dx, void* stream);

/* ---- module-level seams: the reference's Field / Sampler / Encoding nn.Modules as stand-alone operators ----
 * (SURVEY.md 8b).  The fused b200nerf_nff_render_fwd never materialises a per-sample tensor; these do, because the
 * reference's modules hand [N,S,...] tensors to each other.  They use the parameters bound with b200nerf_set_*. */

/* Frustums.get_fast_isotropic_gaussian(num_multisamples=1) (cameras/rays.py:109-124): per-ray origins/directions
 * [N,3], pixel_area [N] (already scaled), euclidean bin edges [N,S+1] -> mean [N,S,3], std [N,S]. */
int b200nerf_isotropic_gaussian_fwd(b200nerf_ctx* ctx, const float* origins, const float* directions,
                                    const float* pixel_area, const float* bins_e, int64_t n_rays, int n_samples,
                                    float* mean, float* std, void* stream);

/* NeuRADHashEncoding.forward(positions: GaussiansStd, times, directions) (field_components/neurad_encoding.py:150-187)
 * of field `field`: scene contraction, static grid, dynamic-actor assignment at each ray's time, per-actor grids
 * (zero padded to the static width), anti-aliasing rescale.  mean [N,S,3], std [N,S], times [N] (the reference
 * reads times[:,0]; may be NULL without actors), flip [N] (+1 / -1) or NULL = the training-mode random actor flip
 * drawn by the caller (:212-219), directions [N,3] (directions_per_ray != 0) or [N,S,3] or NULL.
 * Outputs (each optional): features [N*S, L*F]; density [N,S] = trunc_exp(density_decoder(features))
 * (NeuRADProposalField.get_density, fields/neurad_field.py:208-213); directions_out [N,S,3] (box frame and
 * renormalised for samples inside an actor, :203-209); actor_id [N,S] (actor index or -1). */
int b200nerf_neurad_encoding_fwd(b200nerf_ctx* ctx, int field, const float* mean, const float* std, const float* times,
                                 const float* flip, const float* directions, int directions_per_ray, int64_t n_rays, int n_samples,
                                 float* features, float* density, float* directions_out, int32_t* actor_id,
                                 void* stream);

/* NeuRADField.forward between and after its two MLPs (fields/neurad_field.py:139-149):
 *   mid : geo_out [P, G+1] = (sdf | geo_embedding), directions [P,3] -> mlp_feature_in [P, G+16] =
 *         [geo_embedding | SHEncoding(4)(get_normalized_directions(d))]
 *   tail: feature [P,G] = geo_embedding + mlp_feature_out; sdf [P] = geo_out[:,0]; alpha [P] = sigmoid(-sdf * beta)
 *         with beta = |sdf_to_density.beta| + 1e-4 (model_components/utils.py:29-41).  sdf / alpha may be NULL.
 * The MLPs themselves run through b200nerf_mlp_fwd (wgmma). */
int b200nerf_field_mid_fwd(b200nerf_ctx* ctx, const float* geo_out, const float* directions, int64_t n_points,
                           int geo_feat_dim, float* mlp_feature_in, void* stream);
int b200nerf_field_tail_fwd(b200nerf_ctx* ctx, const float* geo_out, const float* mlp_feature_out, int64_t n_points,
                            int geo_feat_dim, float beta, float* feature, float* sdf, float* alpha, void* stream);

/* spacing_to_euclidean_fn of a SpacedSampler (ray_samplers.py:119-120) on per-ray spacing-domain edges
 * bins_s [N, n_edges] -> bins_e [N, n_edges]; PDFSampler's resampled bins go through it (ray_samplers.py:363-366).
 * `kind` / power_* as in b200nerf_spaced_sample. */
int b200nerf_spacing_to_euclidean(b200nerf_ctx* ctx, int kind, float power_lambda, float power_scaling,
                                  const float* nears, const float* fars, const float* bins_s, int64_t n_rays,
                                  int n_edges, float* bins_e, void* stream);

/* Training-mode sampling (SURVEY.md 8f, row f2).  The random numbers are drawn by the caller (torch.rand, as the
 * reference does) so that the operators stay deterministic functions of their inputs:
 *   SpacedSampler with train_stratified (ray_samplers.py:107-115): t_rand [N,1] (single_jitter) or [N,S+1];
 *     outputs per-ray spacing bins [N,S+1] and euclidean edges [N,S+1].
 *   PDFSampler with train_stratified (ray_samplers.py:321-329): u = u_base + rand / (S_new+1), u_base =
 *     linspace(0, 1 - 1/nb, nb) [S_new+1] (device), rand [N,1] or [N,S_new+1]; other arguments as b200nerf_pdf_resample. */
int b200nerf_spaced_sample_stratified(b200nerf_ctx* ctx, int kind, float power_lambda, float power_scaling,
                                      const float* nears, const float* fars, const float* t_rand, int rand_cols,
                                      int64_t n_rays, int n_samples, float* bins_s, float* bins_e, void* stream);
int b200nerf_pdf_resample_stratified(b200nerf_ctx* ctx, const float* weights, const float* bins, const float* u_base,
                                     const float* rand, int rand_cols, int n_rays, int s_old, int s_new,
                                     float histogram_padding, float* new_bins, float* cdf, int32_t* inds, void* stream);

/* ---- backward operators (SURVEY.md 8f, row f2): gradients of the module-level operators with respect to the trained
 * parameters.  The reference gets these from torch autograd (torch mode) or tiny-cuda-nn's backward kernels; here each
 * forward operator has a hand-written counterpart.  Sample bins carry no gradient (PDFSampler detaches them,
 * ray_samplers.py:363-364); the sample MEANS do when the camera poses are optimised (b200nerf_neurad_encoding_mean_bwd,
 * b200nerf_isotropic_gaussian_bwd).  All grad_* outputs are ACCUMULATED into (+=): zero them first (they are the .grad
 * tensors of the parameters); the d* outputs of the two position-gradient operators are written. */

/* Backward of b200nerf_neurad_encoding_fwd for field `field`: scatter-add into the hash-table gradients.
 *   features mode: dfeatures [N*S, L*F] = dL/d features.
 *   density mode : density [N,S] (the forward output) and ddensity [N,S] = dL/d density; folds in the proposal head
 *                  (trunc_exp, Linear(L*F,1,bias=False)); grad_decoder [L*F] receives dL/d density_decoder.weight.
 * grad_static_table [L*T, F] (or NULL); grad_actor_tables_host = HOST array of n_actors device pointers
 * [La*Ta, F] (entries or the array may be NULL); it is copied, stream-ordered, into ONE context-owned device array, so
 * calls that pass it must not run concurrently on different streams of the same context. */
int b200nerf_neurad_encoding_bwd(b200nerf_ctx* ctx, int field, const float* mean, const float* std, const float* times,
                                 const float* flip, int64_t n_rays, int n_samples, const float* dfeatures,
                                 const float* density, const float* ddensity, float* grad_static_table,
                                 float* const* grad_actor_tables_host, float* grad_decoder, void* stream);

/* Gradient of a field's features with respect to the ACTOR TRAJECTORIES (DynamicActors.actor_positions [T,A,3] /
 * actor_rotations_6d [T,A,6], optimize_trajectories model_components/dynamic_actors.py:37): for every sample inside an
 * actor box, the position gradient of the actor-grid lookup chained through the box transform, rotation_6d_to_matrix,
 * the keyframe interpolation and the keyframes' Gram-Schmidt (utils/poses.py:90-150, cameras/camera_utils.py:422-443).
 * The reference does this for the main field only (require_actor_grad, fields/neurad_field.py:50,177); the box-frame
 * directions carry no gradient in torch mode (SHEncoding.pytorch_fwd is no_grad, field_components/encodings.py:797).
 * `rotations_6d` / `positions` are the raw parameters; grad_* are accumulated (+=). */
int b200nerf_neurad_encoding_pose_bwd(b200nerf_ctx* ctx, int field, const float* mean, const float* std, const float* times,
                                      const float* flip, int64_t n_rays, int n_samples, const float* dfeatures,
                                      const float* rotations_6d, const float* positions, float* grad_rotations_6d,
                                      float* grad_positions, void* stream);

/* Gradient of b200nerf_neurad_encoding_fwd (features or density output) with respect to the sample MEANS, for camera
 * pose optimisation (CameraOptimizer.apply_to_raybundle, cameras/camera_optimizers.py:173-182): dmean [N,S,3] is
 * WRITTEN (one row per sample, no accumulation).  Mode selection as b200nerf_neurad_encoding_bwd: dfeatures [N*S, L*F]
 * (features mode, F = 4), or density [N,S] + ddensity [N,S] (density mode, F = 1, through trunc_exp and the density
 * decoder, fields/neurad_field.py:208-213).  Per sample the gradient combines
 *   - the static lookup through ScaledSceneContraction(order=inf) (field_components/spatial_distortions.py:103-114,
 *     132-136): the contracted mean and, outside the unit cube, the std scaling that changes the anti-aliasing level
 *     weights 1 / max(1, 2 res std) (neurad_encoding.py:297-304); at a tie of |x_i| the inf-norm's gradient is split
 *     evenly, as torch's backward does;
 *   - for a sample inside an actor box, the actor lookup chained through the box transform and the training-mode x
 *     flip (neurad_encoding.py:174-219) -- only for field B200NERF_FIELD_MAIN, whose grid the reference builds with
 *     require_actor_grad (fields/neurad_field.py:50).  In the proposal fields the actor branch runs under no_grad and
 *     overwrites the static features, so an actor sample's dmean is exactly 0.
 * Directions carry no gradient (the SH encoding is no_grad in torch mode, encodings.py:797-800).  An empty batch is a
 * no-op. */
int b200nerf_neurad_encoding_mean_bwd(b200nerf_ctx* ctx, int field, const float* mean, const float* std, const float* times,
                                      const float* flip, int64_t n_rays, int n_samples, const float* dfeatures,
                                      const float* density, const float* ddensity, float* dmean, void* stream);

/* Frustums.get_fast_isotropic_gaussian backward (cameras/rays.py:109-124): mean_s = o + d t_s with t_s = start_s +
 * (end_s - start_s) / 2 of the euclidean edges bins_e [N,S+1] (the same t as b200nerf_isotropic_gaussian_fwd; the bins
 * are detached, std does not depend on o or d).  dmean [N,S,3] -> dorigins = sum_s dmean_s and ddirections =
 * sum_s t_s dmean_s, both [N,3], WRITTEN.  An empty batch is a no-op. */
int b200nerf_isotropic_gaussian_bwd(b200nerf_ctx* ctx, const float* bins_e, int64_t n_rays, int n_samples, const float* dmean,
                                    float* dorigins, float* ddirections, void* stream);

/* HashEncoding.forward backward (autograd of encodings.py:425-466 / tcnn's grid backward) for the stand-alone grid operator
 * b200nerf_hashgrid_fwd: x [P,3], dout [P, L*F] -> grad_table [L*T, F] accumulated (+=).  L*F <= 64. */
int b200nerf_hashgrid_bwd(b200nerf_ctx* ctx, const b200nerf_grid_desc* desc, const float* x, const float* dout,
                          int64_t n_points, float* grad_table, void* stream);

/* nerfacc.render_weight_from_alpha backward (call site models/neurad.py:717): alphas, dweights [N,S] -> dalphas. */
int b200nerf_alpha_to_weights_bwd(b200nerf_ctx* ctx, const float* alphas, const float* dweights, int64_t n_rays, int s,
                                  float* dalphas, void* stream);
/* RaySamples.get_weights backward (cameras/rays.py:188-210): deltas, densities, dweights [N,S] -> ddensities. */
int b200nerf_density_to_weights_bwd(b200nerf_ctx* ctx, const float* deltas, const float* densities,
                                    const float* dweights, int64_t n_rays, int s, float* ddensities, void* stream);

/* FeatureRenderer / AccumulationRenderer / render_depth_simple backward (renderers.py:83-85,349; neurad.py:727-734):
 * given dL/d values_out [N,C], dL/d accumulation [N], dL/d depth [N] (each optional) -> dweights [N,S] and
 * dvalues [N,S,C] (each optional). */
int b200nerf_composite_bwd(b200nerf_ctx* ctx, const float* weights, const float* values, int n_channels,
                           const float* starts, const float* ends, const float* dvalues_out,
                           const float* daccumulation, const float* ddepth, int64_t n_rays, int n_samples,
                           float* dweights, float* dvalues, void* stream);

/* NeuRADField heads backward (fields/neurad_field.py:139-149): dfeature [P,G], dsdf [P], dalpha [P],
 * dmlp_feature_in [P,G+16] (each optional) -> dgeo_out [P,G+1]; dbeta [1] (optional) accumulates
 * dL/d(|beta| + 1e-4).  dL/d mlp_feature_out is dfeature itself. */
int b200nerf_field_heads_bwd(b200nerf_ctx* ctx, const float* geo_out, const float* dfeature, const float* dsdf,
                             const float* dalpha, const float* dmlp_feature_in, int64_t n_points, int geo_feat_dim,
                             float beta, float* dgeo_out, float* dbeta, void* stream);

/* MLP backward pieces (field_components/mlp.py:142-178).  For layer l with input X (a hidden pre-activation Z when
 * relu_x != 0, so act = ReLU) and output gradient dY:
 *   b200nerf_linear_wgrad : dweight [out,in] += dY^T act(X), dbias [out] += sum dY            (widths <= 64)
 *   dX = dY W: b200nerf_mlp_dgrad (above; wgmma, ReLU mask fused), or b200nerf_mlp_fwd with the transposed weight and
 *   b200nerf_relu_bwd     : dZ *= (Z > 0) in place. */
int b200nerf_linear_wgrad(b200nerf_ctx* ctx, const float* x, const float* dy, int64_t n_rows, int in_dim, int out_dim,
                          int relu_x, float* dweight, float* dbias, void* stream);
int b200nerf_relu_bwd(b200nerf_ctx* ctx, const float* z, float* dz, int64_t n, void* stream);
/* EXPERIMENTAL twin of b200nerf_linear_wgrad on the wgmma tensor cores (split-K GEMM, output rows = the rows of a
 * 128-row wgmma tile, 48 input rows per MMA chunk, 3xTF32): same arguments and semantics.  The CUDA-core operator stays
 * the default until this one has been timed. */
int b200nerf_linear_wgrad_tc(b200nerf_ctx* ctx, const float* x, const float* dy, int64_t n_rows, int in_dim, int out_dim,
                             int relu_x, float* dweight, float* dbias, void* stream);

/* NeuRAD's per-ray training regularisers (models/neurad.py:262,524,541-545) on the `weights_list` / `ray_samples_list`
 * of get_nff_outputs; spacing-domain edges ("sdist", losses.py:119-125) and weights as [N,S+1] / [N,S].  Per-ray losses
 * out (the reference takes the mean over rays); the optional gradient outputs are d loss_ray / d weights.
 *   distortion loss   (lossfun_distortion, losses.py:160-177): gradient to the final level's weights.
 *   zipnerf interlevel (losses.py:645-705) for ONE proposal level with blur half-width `pulse_width` (0.03 / 0.003 for
 *     levels 0 / 1): the final level (sdist, weights) is detached by the reference, the gradient goes to prop_weights.
 * n_samples <= 64. */
int b200nerf_distortion_loss(b200nerf_ctx* ctx, const float* sdist, const float* weights, int64_t n_rays, int n_samples,
                             float* loss_per_ray, float* dweights, void* stream);
int b200nerf_zipnerf_interlevel_loss(b200nerf_ctx* ctx, const float* sdist, const float* weights, int n_samples,
                                     const float* prop_sdist, const float* prop_weights, int n_prop_samples,
                                     float pulse_width, int64_t n_rays, float* loss_per_ray, float* dprop_weights,
                                     void* stream);

/* NeuRADModel._compute_is_close_to_lidar (models/neurad.py:677-700), training mode: mask [N,S] (uint8) = for lidar rays,
 * (did_return & |directions_norm - sample midpoint| < carving_epsilon) | (~did_return & midpoint < non_return_distance);
 * without did_return (NULL) just the first term; 0 for camera rays.  bins_e [N,S+1] euclidean edges, is_lidar /
 * did_return [N] uint8, directions_norm [N] (the measured lidar distance). */
int b200nerf_lidar_carving_mask(b200nerf_ctx* ctx, const float* bins_e, const uint8_t* is_lidar,
                                const float* directions_norm, const uint8_t* did_return, float carving_epsilon,
                                float non_return_distance, int64_t n_rays, int n_samples, uint8_t* mask, void* stream);

/* Kernel variant used by b200nerf_nff_render_fwd:
 *   2 (default) ray-per-lane mapping (a warp = 32 adjacent rays at one sample index: coherent gathers), MLPs on the
 *     wgmma tensor cores with the 3xTF32 split (fp32-level accuracy, |err| ~1e-6 relative);
 *   1 warp-per-ray mapping, wgmma MLPs;   0 warp-per-ray mapping, CUDA-core fp32 FFMA MLPs. */
int b200nerf_set_mlp_mode(b200nerf_ctx* ctx, int mode);

/* Synchronises with the device and reports (then clears) the device-side failure flag that kernels raise instead
 * of hanging, e.g. when a tensor-core completion barrier times out.  0 = healthy. */
int b200nerf_check_status(b200nerf_ctx* ctx);

/* PDFSampler.generate_ray_samples, eval mode, include_original=False (ray_samplers.py:280-361):
 * weights [N,S], existing spacing bins [N,S+1], quantiles u [S_new+1] (device) -> new spacing bins
 * [N,S_new+1]; optional cdf [N,S+1] and searchsorted indices [N,S_new+1]. */
int b200nerf_pdf_resample(b200nerf_ctx* ctx, const float* weights, const float* bins, const float* u, int n_rays,
                          int s_old, int s_new, float histogram_padding, float* new_bins, float* cdf,
                          int32_t* inds, void* stream);

/* RaySamples.get_weights (cameras/rays.py:188-210): deltas, densities [N,S] -> weights [N,S]. */
int b200nerf_density_to_weights(b200nerf_ctx* ctx, const float* deltas, const float* densities, int n_rays,
                                int s, float* weights, void* stream);

/* nerfacc.render_weight_from_alpha on dense [N,S] (call site neurad.py:717). */
int b200nerf_alpha_to_weights(b200nerf_ctx* ctx, const float* alphas, int n_rays, int s, float* weights,
                              void* stream);

/* ---- generic sampler / renderer operators (BASELINE config 1 and the reference's per-module API) -------- */

/* SpacedSampler.generate_ray_samples in eval mode (model_components/ray_samplers.py:80-132) for the reference's
 * spacing functions: UniformSampler (:135-156), LinearDisparitySampler (:159-180), PowerSampler (:838-852, needs
 * power_lambda / power_scaling), SqrtSampler (:183-204), LogSampler (:207-228).
 * nears [N] (NULL -> 0), fars [N] -> euclidean bin edges bins_e [N, S+1]; the spacing-domain edges
 * linspace(0,1,S+1) are the same for every ray and written to bins_s [S+1] when non-NULL. */
enum { B200NERF_SPACING_UNIFORM = 0, B200NERF_SPACING_LINDISP = 1, B200NERF_SPACING_POWER = 2,
       B200NERF_SPACING_SQRT = 3, B200NERF_SPACING_LOG = 4 };
int b200nerf_spaced_sample(b200nerf_ctx* ctx, int kind, float power_lambda, float power_scaling, const float* nears,
                           const float* fars, int64_t n_rays, int n_samples, float* bins_s, float* bins_e,
                           void* stream);

/* Frustums.get_positions (cameras/rays.py:50-59): origins + directions * (start + end) / 2 -> [N, S, 3]; with
 * `aabb_host` (6 floats, [2,3]) additionally SceneBox.get_normalized_positions (data/scene_box.py:63-79). */
int b200nerf_frustum_positions(b200nerf_ctx* ctx, const float* origins, const float* directions, const float* bins_e,
                               int64_t n_rays, int n_samples, const float* aabb_host, float* positions, void* stream);

/* Head activations of a density + colour field: raw [P, 1+C] -> density [P] = trunc_exp(raw[:,0])
 * (field_components/activations.py:28-35), rgb [P, C] = sigmoid(raw[:,1:]). */
int b200nerf_density_rgb_heads(b200nerf_ctx* ctx, const float* raw, int64_t n_points, int n_channels, float* density,
                               float* rgb, void* stream);

/* Renderers on dense [N,S] samples (model_components/renderers.py):
 *   out_values [N,C]     = sum_s w*v                     FeatureRenderer (:83-85); with value_nan_to_num = 1 and
 *                          + background*(1 - sum_s w)    `background_host` (C floats) RGBRenderer in eval mode
 *                                                        (:103-148, 233-268; NULL = "random"/no blending)
 *   out_accumulation [N] = sum_s w                       AccumulationRenderer (:322-350)
 *   out_depth [N]        DEPTH_EXPECTED: sum w*mid / (sum w + 1e-10), clipped to the GLOBAL [min, max] of mid over
 *                        the whole batch as DepthRenderer("expected") does (:396-416); DEPTH_MEDIAN (:383-394);
 *                        DEPTH_SIMPLE: NeuRAD's un-normalised render_depth_simple (models/neurad.py:727-734)
 * with mid = (starts + ends) / 2, starts / ends [N,S].  Any output (and its inputs) may be NULL. */
enum { B200NERF_DEPTH_NONE = 0, B200NERF_DEPTH_EXPECTED = 1, B200NERF_DEPTH_MEDIAN = 2, B200NERF_DEPTH_SIMPLE = 3 };
int b200nerf_composite(b200nerf_ctx* ctx, const float* weights, const float* values, int n_channels,
                       int value_nan_to_num, const float* background_host, const float* starts, const float* ends,
                       int depth_method, int64_t n_rays, int n_samples, float* out_values, float* out_accumulation,
                       float* out_depth, void* stream);

/* ---- camera rgb decoder (SURVEY 8(f) row f1) ------------------------------------------------------------ */

/* NeuRADModel.rgb_decoder (models/neurad.py:201-216; BasicBlock model_components/cnns.py:19-46), eval mode:
 *   rgb_decoder.0  Conv2d(in_dim -> 32, 1x1) + ReLU        in_conv   weight [32,in_dim,1,1], bias [32]
 *   rgb_decoder.2, .3, .5, .6  BasicBlock(32, 7x7, BN)      block[b][k]: main_branch.{0|3} Conv2d [32,32,7,7] + bias
 *                                                           and main_branch.{1|4} BatchNorm2d weight/bias/running_*
 *   rgb_decoder.4  ConvTranspose2d(32 -> 32, k = s = 3)     up_conv   weight [32,32,3,3], bias [32]
 *   rgb_decoder.7  Conv2d(32 -> 3, 1x1) (+ Sigmoid)         out_conv  weight [3,32,1,1], bias [3]
 * All pointers are DEVICE fp32 tensors in the reference's state_dict layout.  The library folds the BatchNorms into
 * the convolutions and keeps its own re-laid-out copy: call again after the parameters change. */
typedef struct {
  const float* weight;
  const float* bias;
} b200nerf_conv_params;
typedef struct {
  const float* conv_weight;
  const float* conv_bias;
  const float* bn_weight;
  const float* bn_bias;
  const float* bn_running_mean;
  const float* bn_running_var;
} b200nerf_conv_bn_params;
typedef struct {
  int32_t in_dim;     /* nff_out_dim + appearance_dim (48), <= 64 */
  int32_t hidden_dim; /* rgb_hidden_dim, must be 32 */
  int32_t upsample;   /* rgb_upsample_factor, must be 3 */
  float bn_eps;       /* BatchNorm2d.eps (1e-5) */
  b200nerf_conv_params in_conv;
  b200nerf_conv_bn_params block[4][2];
  b200nerf_conv_params up_conv;
  b200nerf_conv_params out_conv;
} b200nerf_rgb_decoder_params;
int b200nerf_set_rgb_decoder(b200nerf_ctx* ctx, const b200nerf_rgb_decoder_params* params);

/* Scratch the decoder needs for `batch` feature images of height x width (intermediate activations: 3 buffers at
 * feature resolution + 3 at image resolution, 128 B per pixel).  The caller allocates it (16-byte aligned). */
int64_t b200nerf_rgb_decode_workspace_bytes(int batch, int height, int width);

/* The camera half of NeuRADModel.decode_features (models/neurad.py:359-366): features [batch, height, width, in_dim]
 * (= the row-major ray order of b200nerf_nff_render_fwd's `features` output, so no permute is needed) ->
 * rgb [batch, 3*height, 3*width, 3].  impl 0: the 7x7 convolutions run as implicit GEMMs on the wgmma tensor cores
 * (bf16 hi/lo split, fp32 accumulate, fp32-level accuracy), operands moved by the TMA engine; impl 2: the same with
 * per-thread 16-byte asynchronous copies instead of TMA; impl 1: the same pipeline on the CUDA cores in fp32 (slow
 * cross-check of the same op). */
int b200nerf_rgb_decode_fwd(b200nerf_ctx* ctx, const float* features, int batch, int height, int width, float* rgb,
                            void* workspace, int64_t workspace_bytes, int impl, void* stream);

/* ---- ray generation ------------------------------------------------------------------------------------- */

/* Cameras.generate_rays for one PERSPECTIVE camera without distortion, top-to-bottom rolling shutter
 * (cameras/cameras.py:633-667, 793-798, 898-969), over the pixel grid rows row0, row0+row_step, ... and
 * columns col0, col0+col_step, ... (pixel centres at +0.5).  NeuRAD renders at [step//2::step] with step =
 * rgb_upsample_factor (neurad.py:641-646), so generating only those pixels removes the reference's 9x waste.
 * `c2w_host` is 12 floats (3x4 row major), `velocity_host` 3 floats (may be NULL: no rolling shutter).
 * Outputs: origins/directions [n_rows*n_cols,3], pixel_area/times [n_rows*n_cols]. */
int b200nerf_raygen_pinhole(b200nerf_ctx* ctx, const float* c2w_host, float fx, float fy, float cx, float cy,
                            int height, int width, int row0, int row_step, int n_rows, int col0, int col_step,
                            int n_cols, float time, const float* velocity_host, float rolling_shutter_time,
                            float time_to_center_pixel, float* origins, float* directions, float* pixel_area,
                            float* times, void* stream);

/* Lidars._generate_rays_from_points, assume_ego_compensated=True (cameras/lidars.py:399-460): points [P,
 * point_stride] = (x,y,z,intensity,dt,...) in the lidar frame -> rays; `distance` (optional) = the range. */
int b200nerf_raygen_lidar_points(b200nerf_ctx* ctx, const float* l2w_host, const float* points, int point_stride,
                                 int64_t n_points, float scan_time, const float* velocity_host, float h_div,
                                 float v_div, float* origins, float* directions, float* pixel_area, float* times,
                                 float* distance, void* stream);

/* Beam x azimuth lidar ray grid with a rolling-shutter sweep (viewer/render_state_machine.py:395-407 for the
 * directions; cameras/lidars.py:421-423, 625-639 for the per-ray time offset `(azimuth/2pi - 0.5) * revolution_time`
 * and the origin shift `velocity * dt`).  Elevations = linspace(elev_min, elev_max, beams), azimuths = i *
 * azimuth_step.  Outputs [beams*n_azimuth, ...] in beam-major order.  BASELINE config 4's input shape (128 x 2048). */
int b200nerf_raygen_lidar_grid(b200nerf_ctx* ctx, const float* l2w_host, float elev_min_rad, float elev_max_rad,
                               int beams, int n_azimuth, double azimuth_step_rad, float scan_time,
                               float revolution_time, const float* velocity_host, float h_div, float v_div,
                               float* origins, float* directions, float* pixel_area, float* times, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200NERF_H_ */
