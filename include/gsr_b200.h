/* gsr_b200.h -- C ABI of the H100-native (sm_90a) differentiable 3D-Gaussian-splatting rasterizer.
 *
 * This is the drop-in boundary for the ONE hot path of buaacyw/GaussianEditor this repo rebuilds:
 * the `diff_gaussian_rasterization._C` extension behind gaussiansplatting/gaussian_renderer.render().
 * Every entry point replaces one binding of the reference's private pybind module
 * (all paths relative to /root/reference/gaussiansplatting/submodules/diff-gaussian-rasterization/):
 *
 *   gsr_forward_preprocess + gsr_forward_render   <- _C.rasterize_gaussians          ext.cpp:16, rasterize_points.cu:35-95,
 *                                                                                     cuda_rasterizer/rasterizer_impl.cu:179-285
 *   gsr_backward                                  <- _C.rasterize_gaussians_backward ext.cpp:17, rasterize_points.cu:97-157,
 *                                                                                     cuda_rasterizer/rasterizer_impl.cu:289-341
 *   gsr_mark_visible                              <- _C.mark_visible                 ext.cpp:18, rasterize_points.cu:159-175
 *   gsr_apply_weights                             <- _C.apply_weights                ext.cpp:19, rasterize_points.cu:177-234
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / C++ types.  Unless a parameter says "host", every pointer is a
 *     DEVICE pointer on the current CUDA device; the caller (PyTorch's caching allocator in the Python
 *     binding, cudaMalloc in a C host) owns all memory.  "Optional" pointers may be NULL; the reference
 *     encodes the same thing as empty tensors (rasterizer_impl.cu:205,241,275).
 *   - every call takes the cudaStream_t to run on (as void*); the reference always ran on the legacy
 *     default stream and blocked on a cudaMemcpy (rasterizer_impl.cu:237) -- here the only host
 *     synchronisation is the caller waiting for `num_rendered` between the two forward halves.
 *   - return value: 0 = ok, <0 = error (see gsr_last_error()).  There is NO CPU fallback: without a usable
 *     sm_90 device every compute entry point fails with GSR_ERR_CUDA.
 *   - all floating-point data is IEEE binary32, exactly as in the reference.
 */
#ifndef GSR_B200_H_
#define GSR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSR_OK 0
#define GSR_ERR_INVALID (-1) /* bad argument combination (mirrors the reference's Python/C++ argument checks) */
#define GSR_ERR_CUDA (-2)    /* CUDA runtime error; message in gsr_last_error() */
#define GSR_ERR_WORKSPACE (-3) /* a workspace is smaller than the matching gsr_*_bytes() query */

#define GSR_ABI_VERSION 2

#if defined(__GNUC__)
#define GSR_API __attribute__((visibility("default")))
#else
#define GSR_API
#endif

/* Per-call camera / configuration bundle: the fields of GaussianRasterizationSettings
 * (diff_gaussian_rasterization/__init__.py:228-240) plus the two SH sizes the glue derives
 * (rasterize_points.cu:73-76). */
typedef struct gsr_settings {
  int32_t image_height;
  int32_t image_width;
  float tanfovx;
  float tanfovy;
  float scale_modifier;
  int32_t sh_degree;   /* D: active degree, 0..3 */
  int32_t sh_coeffs;   /* M: coefficients ALLOCATED per Gaussian in `shs` (0 when colors_precomp is used) */
  int32_t prefiltered; /* kept for API parity; a culled point with prefiltered!=0 is simply skipped */
  int32_t debug;       /* !=0: synchronise and check for CUDA errors after every launch (auxiliary.h:166-173) */
  const float* bg;         /* [3]  */
  const float* viewmatrix; /* [16] transposed world->camera (scene/cameras.py:92)  */
  const float* projmatrix; /* [16] transposed full projection (scene/cameras.py:93-94) */
  const float* campos;     /* [3]  */
} gsr_settings;

/* The Gaussian cloud as the reference's forward takes it (diff_gaussian_rasterization/__init__.py:258-268).
 * Exactly one of {shs, colors_precomp} and exactly one of {(scales, rotations), cov3D_precomp} is non-NULL. */
typedef struct gsr_cloud {
  int32_t P;                   /* number of Gaussians */
  const float* means3D;        /* [P,3] */
  const float* opacities;      /* [P,1] already sigmoid-ed */
  const float* shs;            /* [P,M,3] optional */
  const float* colors_precomp; /* [P,3]   optional */
  const float* scales;         /* [P,3]   optional, already exp-ed */
  const float* rotations;      /* [P,4]   optional, (r,x,y,z), normalised by the caller */
  const float* cov3D_precomp;  /* [P,6]   optional */
} gsr_cloud;

/* Gradient outputs of the backward pass, shapes as rasterize_points.cu:120-128. The kernels write EVERY
 * element (zeros for invisible Gaussians and for SH coefficients above the active degree), so the
 * buffers may be uninitialised on entry. */
typedef struct gsr_grads {
  float* dL_dmeans3D;   /* [P,3] */
  float* dL_dmeans2D;   /* [P,3] (z is always 0; x,y carry the 0.5*W / 0.5*H NDC scaling, backward.cu:460-461) */
  float* dL_dcolors;    /* [P,3] */
  float* dL_dopacity;   /* [P,1] */
  float* dL_dcov3D;     /* [P,6] */
  float* dL_dsh;        /* [P,M,3] (NULL when M == 0) */
  float* dL_dscales;    /* [P,3] */
  float* dL_drotations; /* [P,4] */
} gsr_grads;

GSR_API int gsr_abi_version(void);
GSR_API const char* gsr_last_error(void); /* thread-local, valid until the next failing call on this thread */
/* Threading: every entry point only touches the buffers it is handed and enqueues on the stream it is handed, so calls
 * from several host threads are safe as long as they do not share a workspace. The library-global pieces are the option
 * table (gsr_set_option: set before the threads start), the launch counter (atomic) and the stage profile (mutex). */

/* ---- workspace sizing (the three opaque buffers of rasterize_points.cu:62-69) ------------------------ */
GSR_API size_t gsr_geometry_bytes(int32_t P);
GSR_API size_t gsr_image_bytes(int32_t image_width, int32_t image_height);
GSR_API size_t gsr_binning_bytes(int32_t P, int64_t num_rendered, int32_t image_width, int32_t image_height);
/* scratch for the backward pass (2-D gradient accumulators) */
GSR_API size_t gsr_backward_scratch_bytes(int32_t P);

/* ---- forward, first half: per-Gaussian preprocess + depth order + tile-count scan --------------------
 * Writes `radii` [P] int32 (0 = culled) and fills `geometry`. The total number of (Gaussian, tile)
 * instances is copied asynchronously into *num_rendered_host (PINNED host memory, int32); the caller must
 * synchronise `stream` (or an event recorded after this call) before reading it. */
GSR_API int gsr_forward_preprocess(const gsr_settings* s, const gsr_cloud* c, void* geometry, size_t geometry_bytes,
                           int32_t* radii, int32_t* num_rendered_host, void* stream);

/* ---- forward, second half: instance emission, per-tile ordering, tile ranges, alpha blending ----------
 * out_color [3,H,W], out_depth [1,H,W] (depth = sum view_z*alpha*T, no background, forward.cu:359,377). */
GSR_API int gsr_forward_render(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered, void* geometry,
                       size_t geometry_bytes, void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                       const int32_t* radii, float* out_color, float* out_depth, void* stream);

/* ---- forward, second half, without waiting for num_rendered ------------------------------------------------
 * Same as gsr_forward_render, but launched BEFORE the host knows num_rendered: `capacity` is the caller's guess
 * (e.g. 1.25x the previous frame's value) and sizes the binning workspace and the launches; the real count is read
 * from the scan result on the device and the slots [num_rendered, capacity) are padding that sorts behind every
 * tile. The caller must afterwards read *num_rendered_host (after the stream reaches the copy issued by
 * gsr_forward_preprocess) and, if it exceeds `capacity`, discard the outputs and call gsr_forward_render with the
 * exact count. gsr_backward then takes `capacity` as its num_rendered argument (it only sizes the workspace).
 * This keeps the GPU busy while the host waits for the count (the reference blocks in cudaMemcpy with an idle
 * GPU, rasterizer_impl.cu:237). */
GSR_API int gsr_forward_render_speculative(const gsr_settings* s, const gsr_cloud* c, int32_t capacity, void* geometry,
                       size_t geometry_bytes, void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                       const int32_t* radii, float* out_color, float* out_depth, void* stream);

/* ---- forward, both halves, for a fixed capacity: no host copy, no host wait ---------------------------------------
 * gsr_forward_preprocess + gsr_forward_render_speculative in one call, without the copy of num_rendered to the host:
 * the call only enqueues work on `stream`, so it can be captured in a CUDA graph and the host can run ahead of the
 * GPU. The workspaces are sized for `capacity` (gsr_geometry_bytes(P), gsr_binning_bytes(P, capacity, W, H),
 * gsr_image_bytes(W, H)). A kernel on the stream writes status[0] = num_rendered and status[1] = (num_rendered >
 * capacity) into the caller's DEVICE buffer `status` (int32[2]).
 * When num_rendered > capacity the frame is empty, on every binning path: out_color = background, out_depth = 0, the
 * alpha image (gsr_alpha_image) = 0, and every backward called with `capacity` as its num_rendered returns zero
 * gradients. The caller reads `status` whenever it chooses to synchronise, and re-sizes.
 * P == 0 writes {0, 0} and zero images. Every argument (capacity > 0, status, outputs, workspace sizes) is checked
 * before the first launch. The backward entry points take `capacity` as their num_rendered argument.
 * gsr_forward_static_raw is the fused-activation form (gsr_raw_cloud, as gsr_forward_preprocess_raw). */
GSR_API int gsr_forward_static(const gsr_settings* s, const gsr_cloud* c, int32_t capacity, void* geometry,
                       size_t geometry_bytes, void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                       int32_t* radii, float* out_color, float* out_depth, int32_t* status, void* stream);

/* ---- backward ------------------------------------------------------------------------------------------
 * dL_dout_color [3,H,W]; the three workspaces and `radii` are the ones the forward produced. */
GSR_API int gsr_backward(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered, const void* geometry,
                 size_t geometry_bytes, const void* binning, size_t binning_bytes, const void* image,
                 size_t image_bytes, const int32_t* radii, const float* dL_dout_color, void* scratch,
                 size_t scratch_bytes, const gsr_grads* grads, void* stream);

/* ---- alpha image (north-star output "RGB / depth / alpha"; opt-in, not in the reference's return tuple) ----
 * out_alpha [H*W] = 1 - final_T, where final_T is what the reference keeps as ImageState::accum_alpha
 * (cuda_rasterizer/rasterizer_impl.h:50, written at forward.cu:371-378). Call after gsr_forward_render on the same
 * `image` workspace. gsr_backward_alpha is gsr_backward with the additional upstream gradient dL_dout_alpha [H*W]
 * (NULL = none): d(1 - T_final)/d(alpha_i) = T_final / (1 - alpha_i) enters dL/dalpha_i next to the background term
 * of backward.cu:505-511. */
GSR_API int gsr_alpha_image(const void* image, size_t image_bytes, int32_t image_width, int32_t image_height,
                    float* out_alpha, void* stream);
GSR_API int gsr_backward_alpha(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered, const void* geometry,
                       size_t geometry_bytes, const void* binning, size_t binning_bytes, const void* image,
                       size_t image_bytes, const int32_t* radii, const float* dL_dout_color,
                       const float* dL_dout_alpha, void* scratch, size_t scratch_bytes, const gsr_grads* grads,
                       void* stream);

/* ---- camera gradients (north star: backward over {..., viewmatrix}; opt-in, the reference has none) -------------
 * The reference's autograd returns None for the raster settings (diff_gaussian_rasterization/__init__.py:213-223), so
 * there is nothing to be drop-in for; this entry point extends gsr_backward_alpha with
 *   dL/dviewmatrix [16], dL/dprojmatrix [16], dL/dcampos [3]
 * for the three camera arrays of gsr_settings treated as INDEPENDENT inputs, exactly as the forward reads them (the
 * view matrix through t = view*mean and the rotation W of the EWA Jacobian product, cuda_rasterizer/forward.cu:74-113;
 * the full projection through p_hom, :196-200; the camera centre through the SH view direction, :20-71). The same
 * conventions as the mean gradient apply (clamped t.x / t.y pass no gradient, backward.cu:205-212). A caller that
 * derives projmatrix and campos from the view matrix (scene/cameras.py:92-95) chains the three in its own autograd.
 * Checked against central finite differences of the fp64 CPU oracle (tests/test_parity_gpu.py). */
typedef struct gsr_camera_grads {
  float* dL_dviewmatrix; /* [16] same layout as gsr_settings.viewmatrix; entries the forward never reads stay 0 */
  float* dL_dprojmatrix; /* [16] */
  float* dL_dcampos;     /* [3]  */
  void* scratch;         /* gsr_camera_scratch_bytes(P) bytes of device memory */
  size_t scratch_bytes;
} gsr_camera_grads;
GSR_API size_t gsr_camera_scratch_bytes(int32_t P);
GSR_API int gsr_backward_camera(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered, const void* geometry,
                        size_t geometry_bytes, const void* binning, size_t binning_bytes, const void* image,
                        size_t image_bytes, const int32_t* radii, const float* dL_dout_color,
                        const float* dL_dout_alpha /* may be NULL */, void* scratch, size_t scratch_bytes,
                        const gsr_grads* grads, const gsr_camera_grads* camera, void* stream);

/* ---- depth gradients (north-star output "RGB / depth / alpha"; opt-in, the reference drops dL/ddepth) -----------
 * The forward's depth image is D = sum_i z_i alpha_i T_i with the view depth z_i = (view * mean).z and no background
 * term. gsr_backward_depth is gsr_backward with the additional upstream gradient dL_dout_depth [H*W] (must not be NULL):
 * depth enters the blending backward as a fourth colour channel with colour z_i and background 0, so it reaches
 * dL/dmean2D, dL/dconic and dL/dopacity through dL/dalpha_i, and dL/dz_i = sum_pixels alpha_i T_i dL/dD reaches
 * dL/dmeans3D through z_i (and dL/dviewmatrix row 2 when `camera` is given). One call covers every combination:
 * dL_dout_alpha may be NULL (as gsr_backward_alpha), `camera` may be NULL (as gsr_backward_camera). Pass a zero
 * dL_dout_color for a loss on the depth alone. The blending backward always runs render_bwd variant 15 here.
 * gsr_backward_raw_depth is the same for gsr_backward_raw (fused activations, below).
 * The Gaussian-sharded path has its own depth entry points (gsr_shard_backward_render_depth,
 * gsr_shard_backward_preprocess_depth / _raw and gsr_sparse_backward_preprocess_depth / _raw, below). Its alpha and
 * camera gradients go through gsr_shard_backward_render_alpha and gsr_shard_backward_preprocess_camera /
 * gsr_sparse_backward_preprocess_camera, which take the depth gradient too. */
GSR_API int gsr_backward_depth(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered, const void* geometry,
                       size_t geometry_bytes, const void* binning, size_t binning_bytes, const void* image,
                       size_t image_bytes, const int32_t* radii, const float* dL_dout_color,
                       const float* dL_dout_alpha /* may be NULL */, const float* dL_dout_depth, void* scratch,
                       size_t scratch_bytes, const gsr_grads* grads, const gsr_camera_grads* camera /* may be NULL */,
                       void* stream);

/* ---- deterministic mode (opt-in; bit-reproducible gradients and apply_weights) ---------------------------
 * The default blending backward and apply_weights add per-Gaussian partial sums with float atomics, so their results
 * change in the last bits from call to call. The *_deterministic entry points compute the same quantities without
 * float atomics: each (instance, tile half) -- each instance for apply_weights -- stores its partial sum as a row at
 * the instance's position in the binning's emission order, and one kernel adds every Gaussian's rows in a fixed
 * order. Two calls on the same inputs give the same bits; the values differ from the default path only in the order
 * of the fp32 sums. Forward outputs are the same in both modes.
 * det_scratch: at least gsr_deterministic_scratch_bytes(P, num_rendered, num_channels) bytes (num_channels: the CH
 * of apply_weights, 0 for the backward), device memory, contents irrelevant (nothing of it needs clearing).
 * gsr_backward_deterministic takes the arguments of gsr_backward_depth, with dL_dout_depth allowed to be NULL (no
 * depth gradient), so it covers the plain, alpha, camera and depth combinations; gsr_backward_raw_deterministic is
 * the same for gsr_backward_raw_depth (fused activations, below). cnt of apply_weights is integer and was already
 * exact. The Gaussian-sharded path has its own deterministic entry points (gsr_shard_backward_render_deterministic,
 * gsr_shard_apply_weights_deterministic, below). */
GSR_API size_t gsr_deterministic_scratch_bytes(int32_t P, int64_t num_rendered, int32_t num_channels);
GSR_API int gsr_backward_deterministic(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered,
                               const void* geometry, size_t geometry_bytes, const void* binning,
                               size_t binning_bytes, const void* image, size_t image_bytes, const int32_t* radii,
                               const float* dL_dout_color, const float* dL_dout_alpha /* may be NULL */,
                               const float* dL_dout_depth /* may be NULL */, void* scratch, size_t scratch_bytes,
                               const gsr_grads* grads, const gsr_camera_grads* camera /* may be NULL */,
                               void* det_scratch, size_t det_scratch_bytes, void* stream);

/* ---- markVisible: present[i] = view-space z > 0.2 (auxiliary.h:139-164) ------------------------------- */
GSR_API int gsr_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present, void* stream);

/* ---- apply_weights (semantic tracing, cuda_rasterizer/apply_weights.cu:240-356) ------------------------
 * Second half of a forward whose colours are ignored: for every (pixel, splat) pair the forward would blend,
 * weights[id*CH+ch] += image_weights[ch,pixel] and cnt[id] += 1 once per channel. Call
 * gsr_forward_preprocess first (with colors_precomp = weights, as the reference does,
 * rasterize_points.cu:223). CH = 1..3. */
GSR_API int gsr_apply_weights(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered, void* geometry,
                      size_t geometry_bytes, void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                      const int32_t* radii, const float* image_weights, int32_t num_channels, float* weights,
                      int32_t* cnt, void* stream);
/* gsr_apply_weights in deterministic mode (see gsr_backward_deterministic): bit-identical weights on every call. */
GSR_API int gsr_apply_weights_deterministic(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered,
                                    void* geometry, size_t geometry_bytes, void* binning, size_t binning_bytes,
                                    void* image, size_t image_bytes, const int32_t* radii,
                                    const float* image_weights, int32_t num_channels, float* weights, int32_t* cnt,
                                    void* det_scratch, size_t det_scratch_bytes, void* stream);

/* ---- introspection for parity tests: device pointers into the opaque workspaces ----------------------- */
typedef struct gsr_geometry_view {
  const float* records;          /* [P,12]: x,y,conicA,conicB | conicC,opacity,depth,_ | r,g,b,_  (visible only) */
  const uint32_t* tiles_touched; /* [P] */
  const uint8_t* clamped;        /* [P] bit ch set = SH colour channel ch was clamped at 0 */
  const uint32_t* depth_order;   /* [P] Gaussian indices ascending in (depth bits, index); culled ones last */
} gsr_geometry_view;
typedef struct gsr_binning_view {
  const uint32_t* point_list; /* [R] == the reference's sorted point_list (rasterizer_impl.cu:256-261) */
  const void* tile_keys;      /* [R] sorted tile id of each instance, uint16 or uint32 (tile_key_bytes) */
  int32_t tile_key_bytes;
} gsr_binning_view;
typedef struct gsr_image_view {
  const float* final_T;       /* [H*W] */
  const uint32_t* n_contrib;  /* [H*W] */
  const uint32_t* ranges;     /* [Ntile,2] */
} gsr_image_view;
GSR_API int gsr_view_geometry(const void* geometry, int32_t P, gsr_geometry_view* out);
GSR_API int gsr_view_binning(const void* binning, int32_t P, int64_t num_rendered, int32_t image_width,
                     int32_t image_height, gsr_binning_view* out);
GSR_API int gsr_view_image(const void* image, int32_t image_width, int32_t image_height, gsr_image_view* out);

/* ---- fused activations (SURVEY.md 8(f-3)) -----------------------------------------------------------------------
 * Opt-in variant that takes the scene model's RAW parameters and applies the activations of
 * scene/gaussian_model.py:221-258 inside the preprocess kernels instead of in PyTorch before every render:
 *   opacity = sigmoid(logit), scale = exp(log_scale), rotation = raw / max(|raw|, 1e-12),
 *   SH row  = [features_dc | features_rest]   (read from the two arrays; no torch.cat, no [P,M,3] copy).
 * gsr_forward_preprocess_raw replaces gsr_forward_preprocess; the second forward half is the ordinary
 * gsr_forward_render (pass a gsr_cloud with P and any non-null pointers); gsr_backward_raw replaces gsr_backward and
 * returns gradients w.r.t. the raw parameters (chain rule through the activations included). settings.sh_coeffs is
 * M = 1 + K, the coefficients allocated over both arrays. Results agree with the PyTorch-activated path to rounding
 * (not bit-for-bit: torch's normalize reduces in a different order); the default entry points keep exact parity.
 * The Gaussian-sharded path takes raw shards too: gsr_shard_preprocess_raw, gsr_shard_preprocess_p2p_raw,
 * gsr_sparse_preprocess_raw, gsr_shard_backward_preprocess_raw and gsr_sparse_backward_preprocess_raw (below). */
typedef struct gsr_raw_cloud {
  int32_t P;
  const float* means3D;        /* [P,3] */
  const float* opacity_logits; /* [P,1] */
  const float* features_dc;    /* [P,1,3] */
  const float* features_rest;  /* [P,K,3], K = sh_coeffs - 1 (NULL when K == 0) */
  const float* log_scales;     /* [P,3] */
  const float* raw_rotations;  /* [P,4], 16-byte aligned */
} gsr_raw_cloud;
typedef struct gsr_raw_grads {
  float* dL_dmeans3D;        /* [P,3] */
  float* dL_dmeans2D;        /* [P,3] */
  float* dL_dopacity_logits; /* [P,1] */
  float* dL_dfeatures_dc;    /* [P,1,3] */
  float* dL_dfeatures_rest;  /* [P,K,3] (NULL when K == 0) */
  float* dL_dlog_scales;     /* [P,3] */
  float* dL_draw_rotations;  /* [P,4], 16-byte aligned */
} gsr_raw_grads;
GSR_API int gsr_forward_preprocess_raw(const gsr_settings* s, const gsr_raw_cloud* c, void* geometry,
                               size_t geometry_bytes, int32_t* radii, int32_t* num_rendered_host, void* stream);
/* gsr_forward_static on the raw parameters (see gsr_forward_static) */
GSR_API int gsr_forward_static_raw(const gsr_settings* s, const gsr_raw_cloud* c, int32_t capacity, void* geometry,
                           size_t geometry_bytes, void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                           int32_t* radii, float* out_color, float* out_depth, int32_t* status, void* stream);
GSR_API int gsr_backward_raw(const gsr_settings* s, const gsr_raw_cloud* c, int32_t num_rendered, const void* geometry,
                     size_t geometry_bytes, const void* binning, size_t binning_bytes, const void* image,
                     size_t image_bytes, const int32_t* radii, const float* dL_dout_color, void* scratch,
                     size_t scratch_bytes, const gsr_raw_grads* grads, void* stream);
/* gsr_backward_raw with the depth image's upstream gradient dL_dout_depth [H*W] (see gsr_backward_depth). */
GSR_API int gsr_backward_raw_depth(const gsr_settings* s, const gsr_raw_cloud* c, int32_t num_rendered,
                           const void* geometry, size_t geometry_bytes, const void* binning, size_t binning_bytes,
                           const void* image, size_t image_bytes, const int32_t* radii, const float* dL_dout_color,
                           const float* dL_dout_depth, void* scratch, size_t scratch_bytes, const gsr_raw_grads* grads,
                           void* stream);
/* gsr_backward_raw_depth in deterministic mode (see gsr_backward_deterministic); dL_dout_depth may be NULL. */
GSR_API int gsr_backward_raw_deterministic(const gsr_settings* s, const gsr_raw_cloud* c, int32_t num_rendered,
                                   const void* geometry, size_t geometry_bytes, const void* binning,
                                   size_t binning_bytes, const void* image, size_t image_bytes, const int32_t* radii,
                                   const float* dL_dout_color, const float* dL_dout_depth /* may be NULL */,
                                   void* scratch, size_t scratch_bytes, const gsr_raw_grads* grads, void* det_scratch,
                                   size_t det_scratch_bytes, void* stream);

/* ---- masked backward (opt-in; gradients only for the Gaussians under edit) -----------------------------------
 * grad_mask [P] (one byte per Gaussian, device memory): every per-Gaussian gradient of a Gaussian with grad_mask[i] == 0
 * is written as +0.0 (means3D, means2D, colours or SH, opacity, cov3D, scales, rotations; on the raw entry point every
 * raw-parameter gradient). The rows with grad_mask[i] != 0 are those of the unmasked backward: bit for bit with
 * det_scratch (deterministic mode), to the rounding of the float atomics without it. The blending backward skips the
 * work of unedited Gaussians: their splats only advance the pixel state, each tile's walk stops at its front-most
 * edited instance, and tiles without one are not walked. The preprocess backward treats them as culled.
 * gsr_backward_masked takes the arguments of gsr_backward_deterministic, plus grad_mask and mask_scratch (at least
 * gsr_grad_mask_scratch_bytes(W, H) bytes of device memory, contents irrelevant); det_scratch may be NULL (the default,
 * atomic kernels), dL_dout_alpha and dL_dout_depth may be NULL, camera must be NULL (the camera gradient sums over every
 * Gaussian). gsr_backward_raw_masked is the same for gsr_backward_raw_deterministic (fused activations). A NULL
 * grad_mask or a non-NULL camera returns GSR_ERR_INVALID. The forward is unchanged. */
GSR_API size_t gsr_grad_mask_scratch_bytes(int32_t image_width, int32_t image_height);
GSR_API int gsr_backward_masked(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered, const void* geometry,
                        size_t geometry_bytes, const void* binning, size_t binning_bytes, const void* image,
                        size_t image_bytes, const int32_t* radii, const float* dL_dout_color,
                        const float* dL_dout_alpha /* may be NULL */, const float* dL_dout_depth /* may be NULL */,
                        void* scratch, size_t scratch_bytes, const gsr_grads* grads,
                        const gsr_camera_grads* camera /* must be NULL */, void* det_scratch /* may be NULL */,
                        size_t det_scratch_bytes, const uint8_t* grad_mask, void* mask_scratch,
                        size_t mask_scratch_bytes, void* stream);
GSR_API int gsr_backward_raw_masked(const gsr_settings* s, const gsr_raw_cloud* c, int32_t num_rendered,
                            const void* geometry, size_t geometry_bytes, const void* binning, size_t binning_bytes,
                            const void* image, size_t image_bytes, const int32_t* radii, const float* dL_dout_color,
                            const float* dL_dout_depth /* may be NULL */, void* scratch, size_t scratch_bytes,
                            const gsr_raw_grads* grads, const gsr_camera_grads* camera /* must be NULL */,
                            void* det_scratch /* may be NULL */, size_t det_scratch_bytes, const uint8_t* grad_mask,
                            void* mask_scratch, size_t mask_scratch_bytes, void* stream);

/* ---- mask image in the colour pass (opt-in; forward only) ---------------------------------------------------------
 * The _mask twin of a forward entry point takes its arguments plus mask [P] (one byte per Gaussian, device memory) and
 * out_mask_render [3,H,W] (device memory), and writes, next to its usual outputs, the image of the Gaussians with
 * mask[i] != 0 drawn in white: what the same forward returns as out_color with colors_precomp[i] = (mask[i] != 0) in
 * all three channels, bit for bit, including the background, an overflowing static frame (background) and P == 0
 * (zeros). The blend walk is not repeated: the same pass accumulates one more value per pixel. Every other output is
 * unchanged. gsr_forward_static_raw_mask takes its opacity from the in-kernel sigmoid, so its mask image matches a
 * forward on the activated parameters to that rounding only. The image has no backward. A NULL mask or a NULL
 * out_mask_render returns GSR_ERR_INVALID before any other check or device work. */
GSR_API int gsr_forward_render_mask(const gsr_settings* s, const gsr_cloud* c, int32_t num_rendered, void* geometry,
                            size_t geometry_bytes, void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                            const int32_t* radii, float* out_color, float* out_depth, const uint8_t* mask,
                            float* out_mask_render, void* stream);
GSR_API int gsr_forward_render_speculative_mask(const gsr_settings* s, const gsr_cloud* c, int32_t capacity,
                            void* geometry, size_t geometry_bytes, void* binning, size_t binning_bytes, void* image,
                            size_t image_bytes, const int32_t* radii, float* out_color, float* out_depth,
                            const uint8_t* mask, float* out_mask_render, void* stream);
GSR_API int gsr_forward_static_mask(const gsr_settings* s, const gsr_cloud* c, int32_t capacity, void* geometry,
                            size_t geometry_bytes, void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                            int32_t* radii, float* out_color, float* out_depth, int32_t* status, const uint8_t* mask,
                            float* out_mask_render, void* stream);
GSR_API int gsr_forward_static_raw_mask(const gsr_settings* s, const gsr_raw_cloud* c, int32_t capacity, void* geometry,
                            size_t geometry_bytes, void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                            int32_t* radii, float* out_color, float* out_depth, int32_t* status, const uint8_t* mask,
                            float* out_mask_render, void* stream);

/* ---- masked Adam (one optimizer step over the Gaussians under edit) ------------------------------------------
 * One Adam step (torch.optim.Adam without weight decay, amsgrad or maximize) over n_groups row-aligned fp32 tensors
 * p, g, m, v of shape [P, D] (row-major, D may differ per group), in one launch, restricted to the rows with
 * mask[i] != 0. Of an unedited row nothing is read or written: p, m and v keep their bits whatever g, m and v hold.
 * Edited elements, in fp32:  m += (1 - beta1) * (g - m);  v = v * beta2 + (1 - beta2) * g * g;
 *                            p -= step_size * m / (sqrt(v) / bc2_sqrt + eps)
 * step_dev == NULL: step is the step count after this update (host), and step_size = lr / (1 - beta1^step),
 * bc2_sqrt = (1 - beta2^step)^0.5 are computed on the host in double, as torch computes them for a CPU step.
 * step_dev != NULL (capturable): the call adds 1 to the device float *step_dev first, then the update computes
 * step_size and bc2_sqrt in fp32 from it on the device, as torch's capturable Adam does. No host synchronisation, no
 * atomics: the call can be captured in a CUDA graph, and each replay advances the step once.
 * Groups with P * D == 0 are skipped (their pointers may be NULL; a device step is still advanced).
 * GSR_ERR_INVALID, before any device work: n_groups outside [1, GSR_ADAM_MAX_GROUPS], NULL groups or mask, P < 0,
 * D < 0 or D > GSR_ADAM_MAX_D, a NULL p, g, m or v in a group with P * D > 0, beta1 or beta2 outside [0, 1), eps < 0. */
#define GSR_ADAM_MAX_GROUPS 16
#define GSR_ADAM_MAX_D (1 << 24)
typedef struct gsr_adam_group {
  float* p;
  const float* g;
  float* m;          /* exp_avg */
  float* v;          /* exp_avg_sq */
  int32_t D;         /* floats per row */
  double lr, beta1, beta2, eps;
  double step;       /* used when step_dev == NULL */
  float* step_dev;   /* capturable: device step, incremented by the call */
} gsr_adam_group;
GSR_API int gsr_adam_masked(const gsr_adam_group* groups, int32_t n_groups, int32_t P, const uint8_t* mask,
                            void* stream);

/* ---- anchor loss (GaussianEditor's per-step anchor regularizer, GaussianModel.anchor_loss) -------------------------
 * terms: exactly GSR_ANCHOR_TERMS row-aligned fp32 [P, D] pairs, in GaussianModel.update_anchor's order
 * (_xyz, _features_dc, _features_rest, _scaling, _rotation, _opacity): p the parameter, a its anchor snapshot, g its
 * gradient (backward only). With w_i = schedule[generation[i]] and N_m the number of rows with mask[i] != 0:
 *   L_k = sum over edited rows i, j < D_k of w_i * (p_k[i,j] - a_k[i,j])^2 / (N_m * D_k)
 * accumulated in fp64 and rounded to fp32, and out4 = (L_dc + L_rest, L_xyz + L_rot, L_opacity, L_scale) added in
 * fp32: the reference dict's (color, geo, opacity, scale). A term without elements (N_m == 0 or D == 0) is NaN, as
 * torch's mean of an empty tensor. A generation outside [0, n_schedule) gives the row a NaN weight (never an
 * out-of-bounds read; torch.gather would trap instead). The sums run in a fixed order over a grid that depends on P
 * only, with no float atomics: the result is bit-reproducible.
 * gsr_anchor_loss_forward writes out4 (device [4]) and keeps N_m in the scratch (device, at least
 * gsr_anchor_loss_scratch_bytes(P)) for gsr_anchor_loss_backward, which takes that scratch unchanged and
 * grad_out4 (device [4], the gradients of out4) and writes all six g in one launch: on an edited row
 * g = 2 (p - a) ((grad_out4[group] / (float)(N_m D)) w), the order of torch's mean and mse backward, with -0 written as
 * +0; on every other row +0.0, without reading p or a. Neither call synchronises with the host: both can be captured
 * in a CUDA graph. GSR_ERR_INVALID, before any device work: NULL terms or schedule, P < 0, n_schedule < 1, NULL mask or
 * generation with P > 0, D < 0 or D > GSR_ADAM_MAX_D, a NULL p or a (and g, backward) in a term with P * D > 0, a NULL
 * out4 / grad_out4, a NULL or too small scratch. */
#define GSR_ANCHOR_TERMS 6
typedef struct gsr_anchor_term {
  const float* p;
  const float* a;
  float* g;          /* backward only; may be NULL in the forward */
  int32_t D;         /* floats per row */
} gsr_anchor_term;
GSR_API size_t gsr_anchor_loss_scratch_bytes(int32_t P);
GSR_API int gsr_anchor_loss_forward(const gsr_anchor_term* terms, int32_t P, const uint8_t* mask,
                            const int64_t* generation, const float* schedule, int32_t n_schedule, void* scratch,
                            size_t scratch_bytes, float* out4, void* stream);
GSR_API int gsr_anchor_loss_backward(const gsr_anchor_term* terms, int32_t P, const uint8_t* mask,
                            const int64_t* generation, const float* schedule, int32_t n_schedule, const void* scratch,
                            size_t scratch_bytes, const float* grad_out4, void* stream);

/* ---- Gaussian-sharded multi-GPU path (BASELINE config 4; SURVEY.md 8(e)) ----------------------------------
 * The reference has no multi-GPU rasterizer; these entry points split the single-GPU pipeline at the two places
 * where the Gaussian-index decomposition (preprocess, fused preprocess backward) meets the tile decomposition
 * (binning, blending), so that a host can put one collective in each gap:
 *
 *   rank g owns Gaussians [index_base, index_base + shard.P) of P_total and the tile rows ty % row_stride == row_phase.
 *   forward : gsr_shard_preprocess  -> ALL-GATHER of the 48-byte splat records (gsr_view_exchange gives the array;
 *                                      a record carries its radius and depth key, so it is the whole exchange)
 *             gsr_shard_order       -> radii of all Gaussians, owned-tile counts, depth order, scan, num_rendered
 *                                      (this rank's instances)
 *             gsr_shard_render      -> binning + blending of the owned tiles into zero-initialised full frames
 *                                      -> ALL-REDUCE(sum) of the frames (every pixel has exactly one non-zero
 *                                         contributor, so the sum is a bit-exact concatenation)
 *   backward: gsr_shard_backward_render     -> partial 2-D gradient accumulators [P_total, 12]
 *                                              -> REDUCE-SCATTER(sum) to the index owners
 *             gsr_shard_backward_preprocess -> gradients of this rank's Gaussians
 * All P_total-sized arrays (geometry workspace, radii, accumulators) are indexed by GLOBAL Gaussian index, so
 * the gathered state is exactly the single-GPU state and the images are bit-identical to gsr_forward_render's.
 * Every rank must pass the same P_total and slice_len (= ceil(P_total / world)); slots of a slice beyond
 * shard.P are marked culled.
 * Depth gradient (see gsr_backward_depth): gsr_shard_backward_render_depth also writes dL/dz into float 9 of every
 * accumulator row, which the reduce-scatter (and the sparse return / gather) carries with the other eleven; then
 * gsr_shard_backward_preprocess_depth (or gsr_shard_backward_preprocess_raw with depth = 1) takes it into dL/dmeans3D.
 * Fused activations (see gsr_forward_preprocess_raw): the *_raw entry points take this rank's rows of the raw
 * parameters (gsr_raw_cloud, features_rest 16-byte aligned) and return gradients w.r.t. them (gsr_raw_grads). */
typedef struct gsr_tile_owner {
  int32_t row_stride; /* >= 1 */
  int32_t row_phase;  /* 0 .. row_stride-1 */
} gsr_tile_owner;
typedef struct gsr_exchange_view {
  void* records; /* [P_total] 48-byte splat records; rank g writes [g*slice_len, (g+1)*slice_len) */
} gsr_exchange_view;
GSR_API int gsr_view_exchange(void* geometry, int32_t P_total, gsr_exchange_view* out);
GSR_API int gsr_shard_preprocess(const gsr_settings* s, const gsr_cloud* shard, int32_t P_total, int32_t index_base,
                         int32_t slice_len, void* geometry, size_t geometry_bytes, int32_t* radii_total, void* stream);
/* radii_total [P_total] is (re)written here for ALL Gaussians from the gathered records. */
GSR_API int gsr_shard_order(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total, void* geometry,
                    size_t geometry_bytes, int32_t* radii_total, int32_t* num_rendered_host, void* stream);
GSR_API int gsr_shard_render(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total, int32_t num_rendered,
                     void* geometry, size_t geometry_bytes, void* binning, size_t binning_bytes, void* image,
                     size_t image_bytes, const int32_t* radii_total, float* out_color, float* out_depth, void* stream);
GSR_API int gsr_shard_backward_render(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total,
                              int32_t num_rendered, const void* geometry, size_t geometry_bytes, const void* binning,
                              size_t binning_bytes, const void* image, size_t image_bytes, const float* dL_dout_color,
                              void* acc_total, size_t acc_bytes, void* stream);
/* acc_slice: this rank's [shard.P, 12] rows of the reduced accumulators (gsr_backward_scratch_bytes(shard.P)). */
GSR_API int gsr_shard_backward_preprocess(const gsr_settings* s, const gsr_cloud* shard, int32_t P_total,
                                  int32_t index_base, const void* geometry, size_t geometry_bytes,
                                  const int32_t* radii_total, const void* acc_slice, const gsr_grads* grads,
                                  void* stream);
/* gsr_shard_preprocess on a raw shard (fused activations). */
GSR_API int gsr_shard_preprocess_raw(const gsr_settings* s, const gsr_raw_cloud* shard, int32_t P_total,
                                     int32_t index_base, int32_t slice_len, void* geometry, size_t geometry_bytes,
                                     int32_t* radii_total, void* stream);
/* gsr_shard_backward_render with the depth image's upstream gradient dL_dout_depth [H*W] (must not be NULL; pass a zero
 * dL_dout_color for a loss on the depth alone). det_scratch NULL: float atomics, as gsr_shard_backward_render;
 * otherwise the deterministic form, as gsr_shard_backward_render_deterministic (gsr_deterministic_scratch_bytes(P_total,
 * num_rendered, 0) bytes). */
GSR_API int gsr_shard_backward_render_depth(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total,
                                            int32_t num_rendered, const void* geometry, size_t geometry_bytes,
                                            const void* binning, size_t binning_bytes, const void* image,
                                            size_t image_bytes, const float* dL_dout_color, const float* dL_dout_depth,
                                            void* acc_total, size_t acc_bytes, void* det_scratch /* may be NULL */,
                                            size_t det_scratch_bytes, void* stream);
/* gsr_shard_backward_preprocess with dL/dz (float 9 of the reduced rows) taken into dL/dmeans3D. */
GSR_API int gsr_shard_backward_preprocess_depth(const gsr_settings* s, const gsr_cloud* shard, int32_t P_total,
                                                int32_t index_base, const void* geometry, size_t geometry_bytes,
                                                const int32_t* radii_total, const void* acc_slice,
                                                const gsr_grads* grads, void* stream);
/* gsr_shard_backward_preprocess on a raw shard: gradients w.r.t. the raw parameters; depth != 0 as the DEPTH form. */
GSR_API int gsr_shard_backward_preprocess_raw(const gsr_settings* s, const gsr_raw_cloud* shard, int32_t P_total,
                                              int32_t index_base, const void* geometry, size_t geometry_bytes,
                                              const int32_t* radii_total, const void* acc_slice,
                                              const gsr_raw_grads* grads, int32_t depth, void* stream);
/* Alpha image and camera gradients of a sharded cloud (see gsr_alpha_image and gsr_backward_camera).
 *   gsr_shard_alpha_image: after gsr_shard_render, out_alpha [H*W] = 1 - final_T on the tile rows `owner` owns only
 *       (final_T elsewhere in a shard's image workspace is not written); every other pixel is left untouched, so the
 *       alpha plane travels with the frame (all-reduce of a zero-filled [5,H,W] frame, or gsr_frame_broadcast_planes).
 *   gsr_shard_backward_render_alpha: gsr_shard_backward_render_depth with the alpha image's upstream gradient
 *       dL_dout_alpha [H*W] (must not be NULL). dL_dout_depth may be NULL (no depth gradient) and det_scratch may be
 *       NULL (float atomics), so one entry covers alpha x depth x deterministic.
 *   gsr_shard_backward_preprocess_camera: gsr_shard_backward_preprocess (depth = 0) or its DEPTH form (depth != 0) that
 *       also writes THIS RANK'S PARTIAL camera gradients (its Gaussians only; zeros for an empty shard) into `camera`
 *       (scratch: gsr_camera_scratch_bytes(shard.P)). The host sums the ranks' partials in ascending rank order on every
 *       rank (not with an all-reduce, whose order is not fixed), which gives every rank the same bits; at world 1 the
 *       partial is the single-GPU gsr_backward_camera result. */
GSR_API int gsr_shard_alpha_image(const gsr_tile_owner* owner, const void* image, size_t image_bytes,
                                  int32_t image_width, int32_t image_height, float* out_alpha, void* stream);
GSR_API int gsr_shard_backward_render_alpha(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total,
                                            int32_t num_rendered, const void* geometry, size_t geometry_bytes,
                                            const void* binning, size_t binning_bytes, const void* image,
                                            size_t image_bytes, const float* dL_dout_color, const float* dL_dout_alpha,
                                            const float* dL_dout_depth /* may be NULL */, void* acc_total,
                                            size_t acc_bytes, void* det_scratch /* may be NULL */,
                                            size_t det_scratch_bytes, void* stream);
GSR_API int gsr_shard_backward_preprocess_camera(const gsr_settings* s, const gsr_cloud* shard, int32_t P_total,
                                                 int32_t index_base, const void* geometry, size_t geometry_bytes,
                                                 const int32_t* radii_total, const void* acc_slice,
                                                 const gsr_grads* grads, int32_t depth, const gsr_camera_grads* camera,
                                                 void* stream);
/* Semantic tracing (gsr_apply_weights) of a sharded cloud. After gsr_shard_order (with the same owner and workspaces),
 * bins the owned tile rows and walks them: every hit of splat i (GLOBAL index) adds the pixel's mask value to
 * weights_total[i*weights_stride + ch] (ch < num_channels, float atomics) and num_channels to
 * cnt_total[i*cnt_stride] (int32 atomics). Nothing is zeroed here. num_channels is 1..3, weights_stride >= num_channels,
 * cnt_stride >= 1 (elements); image_weights is the full [num_channels, H, W] mask on every rank. Timed under the
 * "apply_weights" stage. The sequence of one view (the colours are unused: any valid [shard.P, 3] buffer, e.g. means3D,
 * may stand in the colors_precomp slot, as gsr_apply_weights' callers do):
 *   gsr_shard_preprocess -> ALL-GATHER (or gsr_shard_preprocess_p2p -> barrier) -> gsr_shard_order
 *   gsr_shard_apply_weights into ZEROED [P_total, CH] float + [P_total] int32 buffers (strides CH and 1)
 *   -> REDUCE-SCATTER(sum) of both buffers -> add this rank's slices into its weights [shard.P, CH] / cnt [shard.P]
 * The sparse exchange uses the same call on the candidates (see gsr_sparse_apply_weights_gather). */
GSR_API int gsr_shard_apply_weights(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total,
                                    int32_t num_rendered, void* geometry, size_t geometry_bytes, void* binning,
                                    size_t binning_bytes, void* image, size_t image_bytes, const int32_t* radii_total,
                                    const float* image_weights, int32_t num_channels, float* weights_total,
                                    int64_t weights_stride, int32_t* cnt_total, int64_t cnt_stride, void* stream);
/* Deterministic mode of the two sharded stages that add with float atomics (see gsr_backward_deterministic). Each
 * instance of the owned tile rows stores its rows at its slot in this rank's emission order and one kernel adds every
 * Gaussian's rows in a fixed order, so this rank's partial sums are bit-identical from call to call; a host that also
 * adds the ranks' partial rows in a fixed order (ascending rank: the sparse gathers do, a reduce-scatter does not
 * promise it) gets bit-reproducible results for a fixed number of ranks. They are not the single-GPU bits: the sums
 * are grouped per rank. det_scratch: gsr_deterministic_scratch_bytes(P_total, num_rendered, CH) bytes (CH = 0 for the
 * backward), contents irrelevant. All arguments are checked before any device work.
 *   gsr_shard_backward_render_deterministic: the arguments of gsr_shard_backward_render; it writes every one of the
 *       P_total accumulator rows (zeros for a Gaussian without hits on this rank).
 *   gsr_shard_apply_weights_deterministic: the arguments of gsr_shard_apply_weights, but weights_total must be packed,
 *       weights_stride == num_channels (the reduction adds into [P_total, CH]); weights are still accumulated and cnt
 *       keeps its exact int32 atomics. With the sparse exchange, reduce into a separate zeroed [world*seg_cap, CH]
 *       buffer, keep the count in the candidate rows (cnt_total = (int32_t*)(acc + GSR_SPARSE_AW_CNT_SLOT),
 *       cnt_stride = 12) and copy the weights into floats 0..CH-1 of those rows before gsr_sparse_return. */
GSR_API int gsr_shard_backward_render_deterministic(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total,
                                                    int32_t num_rendered, const void* geometry, size_t geometry_bytes,
                                                    const void* binning, size_t binning_bytes, const void* image,
                                                    size_t image_bytes, const float* dL_dout_color, void* acc_total,
                                                    size_t acc_bytes, void* det_scratch, size_t det_scratch_bytes,
                                                    void* stream);
GSR_API int gsr_shard_apply_weights_deterministic(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total,
                                                  int32_t num_rendered, void* geometry, size_t geometry_bytes,
                                                  void* binning, size_t binning_bytes, void* image, size_t image_bytes,
                                                  const int32_t* radii_total, const float* image_weights,
                                                  int32_t num_channels, float* weights_total, int64_t weights_stride,
                                                  int32_t* cnt_total, int64_t cnt_stride, void* det_scratch,
                                                  size_t det_scratch_bytes, void* stream);

/* ---- fused preprocess + all-gather over NVLink peer memory ---------------------------------------------------
 * Instead of gsr_shard_preprocess followed by an all-gather, every rank's preprocess kernel pushes its block of
 * records into the geometry workspace of EVERY rank (TMA bulk stores from shared memory to peer-mapped global
 * memory). The workspaces must come from gsr_peer_alloc and be opened on the other ranks with gsr_peer_open:
 * peer_geometry[r] is rank r's workspace as mapped in THIS process (own entry = the local pointer), all of the same
 * size and therefore the same layout. The caller must run a cross-rank barrier on `stream` (e.g. a 4-byte
 * all-reduce) between this call and gsr_shard_order, and between a rank's last read of a workspace and the next
 * gsr_shard_preprocess_p2p that targets it (any collective of the step does). */
#define GSR_MAX_PEERS 8
#define GSR_PEER_HANDLE_BYTES 64
GSR_API int gsr_peer_alloc(size_t bytes, void** ptr_out, void* handle_out /* [GSR_PEER_HANDLE_BYTES] host */);
GSR_API int gsr_peer_open(const void* handle /* [GSR_PEER_HANDLE_BYTES] host */, void** ptr_out);
GSR_API int gsr_peer_close(void* ptr);
GSR_API int gsr_peer_free(void* ptr);
GSR_API int gsr_shard_preprocess_p2p(const gsr_settings* s, const gsr_cloud* shard, int32_t P_total, int32_t index_base,
                             int32_t slice_len, void* const* peer_geometry /* [world] host array */, int32_t world,
                             int32_t rank, size_t geometry_bytes, int32_t* radii_total, void* stream);
/* gsr_shard_preprocess_p2p on a raw shard (fused activations). */
GSR_API int gsr_shard_preprocess_p2p_raw(const gsr_settings* s, const gsr_raw_cloud* shard, int32_t P_total,
                                         int32_t index_base, int32_t slice_len,
                                         void* const* peer_geometry /* [world] host array */, int32_t world,
                                         int32_t rank, size_t geometry_bytes, int32_t* radii_total, void* stream);

/* ---- sparse exchange for the Gaussian-sharded path -------------------------------------------------------------
 * The dense scheme above moves, sorts and reduces P_total-sized arrays on every rank. Here a splat record travels only
 * to the ranks whose tile rows (ty % world == d) its tile rectangle touches, into slot  rank*seg_cap + j  of that
 * rank's CANDIDATE array, where j is the record's position among this rank's Gaussians bound for d, in index order.
 * The candidate array (world segments of capacity seg_cap; unused slots are holes with the "culled" sort key) is in
 * global-index order, so the existing stable depth sort / scan / binning / blending stages run on it unchanged as a
 * cloud of world*seg_cap Gaussians (gsr_shard_render / gsr_shard_backward_render with P_total = world*seg_cap and the
 * candidate workspace as `geometry`) and produce the single-GPU lists of the owned tiles bit for bit. The backward
 * returns each candidate's 12-float accumulator row to slot  d*seg_cap + j  of the OWNER's `ret` array, where the
 * owner adds the <= world partial rows of each Gaussian in ascending rank order (deterministic).
 *
 *   forward : gsr_sparse_preprocess   preprocess + destination masks + ordered slots + peer stores of the records;
 *                                     writes counts_row[d] = n[rank -> d]
 *             -- host: all-reduce(sum) of the [world, GSR_MAX_PEERS] count matrix (row = source, written by its rank). It is also the barrier that
 *                orders the peer stores before the readers. --
 *             gsr_sparse_order        candidates -> radii / owned-tile counts / depth order / scan; host_out[0] =
 *                                     num_rendered of this rank, host_out[1] = max over the matrix (a value > seg_cap
 *                                     means some segment overflowed on some rank: redo the step with a larger seg_cap)
 *             gsr_shard_render        (existing)   -> gsr_frame_broadcast or an all-reduce of the frames
 *   backward: gsr_shard_backward_render (existing) -> gsr_sparse_return (peer stores) -- barrier --
 *             gsr_sparse_backward_preprocess       gather of the returned rows + fused preprocess backward
 * peer_cand[r] is rank r's candidate workspace (gsr_sparse_candidate_bytes, from gsr_peer_alloc / gsr_peer_open) as
 * mapped in this process; with virtual ranks on one device they are simply different buffers. */
typedef struct gsr_sparse_plan {
  int32_t world, rank;
  int32_t slice_len; /* ceil(P_total / world): Gaussians per rank (the last rank may hold fewer) */
  int32_t seg_cap;   /* capacity of one (source -> destination) segment; the same on every rank */
} gsr_sparse_plan;
typedef struct gsr_sparse_view_t {
  void* records;         /* [world*seg_cap] 48-byte candidate records */
  float* ret;            /* [world*seg_cap, 12] accumulator rows returned by the tile owners */
  size_t geometry_bytes; /* size of the leading part that is laid out like gsr_geometry_bytes(world*seg_cap) */
} gsr_sparse_view_t;
GSR_API size_t gsr_sparse_local_bytes(int32_t slice_len);
GSR_API size_t gsr_sparse_candidate_bytes(int32_t world, int32_t seg_cap);
GSR_API int gsr_sparse_view(void* cand_ws, int32_t world, int32_t seg_cap, gsr_sparse_view_t* out);
GSR_API int gsr_sparse_preprocess(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan, void* local_ws,
                          size_t local_bytes, int32_t* radii_local /* [shard.P] */, void* const* peer_cand /* [world] host */,
                          size_t cand_bytes, int32_t* counts_row /* [GSR_MAX_PEERS] device */, void* stream);
GSR_API int gsr_sparse_order(const gsr_settings* s, const gsr_sparse_plan* plan, void* cand_ws, size_t cand_bytes,
                     const int32_t* counts_matrix /* [world, GSR_MAX_PEERS] device, row = source */,
                     int32_t* radii_cand /* [world*seg_cap] */, int32_t* host_out /* [2] pinned host */, void* stream);
GSR_API int gsr_sparse_return(const gsr_sparse_plan* plan, const void* acc_cand /* [world*seg_cap, 12] */,
                      const int32_t* counts_matrix, void* const* peer_cand, void* stream);
GSR_API int gsr_sparse_backward_preprocess(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan,
                                   const void* local_ws, size_t local_bytes, const int32_t* radii_local,
                                   const void* cand_ws, size_t cand_bytes, void* acc_slice /* [shard.P,12] scratch */,
                                   size_t acc_bytes, const gsr_grads* grads, void* stream);
/* Depth gradient and fused activations with the sparse exchange: gsr_sparse_preprocess_raw replaces
 * gsr_sparse_preprocess for a raw shard; the blending backward is gsr_shard_backward_render_depth on the candidates
 * (the returned rows carry float 9 like the others); gsr_sparse_backward_preprocess_depth (activated) and
 * gsr_sparse_backward_preprocess_raw (raw, depth != 0 for the DEPTH form) replace gsr_sparse_backward_preprocess. */
GSR_API int gsr_sparse_preprocess_raw(const gsr_settings* s, const gsr_raw_cloud* shard, const gsr_sparse_plan* plan,
                                      void* local_ws, size_t local_bytes, int32_t* radii_local,
                                      void* const* peer_cand /* [world] host */, size_t cand_bytes,
                                      int32_t* counts_row, void* stream);
GSR_API int gsr_sparse_backward_preprocess_depth(const gsr_settings* s, const gsr_cloud* shard,
                                                 const gsr_sparse_plan* plan, const void* local_ws, size_t local_bytes,
                                                 const int32_t* radii_local, const void* cand_ws, size_t cand_bytes,
                                                 void* acc_slice, size_t acc_bytes, const gsr_grads* grads,
                                                 void* stream);
GSR_API int gsr_sparse_backward_preprocess_raw(const gsr_settings* s, const gsr_raw_cloud* shard,
                                               const gsr_sparse_plan* plan, const void* local_ws, size_t local_bytes,
                                               const int32_t* radii_local, const void* cand_ws, size_t cand_bytes,
                                               void* acc_slice, size_t acc_bytes, const gsr_raw_grads* grads,
                                               int32_t depth, void* stream);
/* Semantic tracing with the sparse exchange. The candidate rows carry the hits: weights in floats 0..CH-1 and the
 * count as int32 BITS in float GSR_SPARSE_AW_CNT_SLOT (never converted), and gsr_sparse_return copies rows bit for bit.
 *   gsr_sparse_preprocess -- gsr_peer_barrier(with_matrix_row) -- gsr_sparse_order   (as in the forward, overflow redo
 *                                                                                    included)
 *   gsr_shard_apply_weights on the candidates (P_total = world*seg_cap, candidate workspace as `geometry`) into ZEROED
 *       rows acc [world*seg_cap, 12]: weights_total = acc, weights_stride = 12,
 *       cnt_total = (int32_t*)(acc + GSR_SPARSE_AW_CNT_SLOT), cnt_stride = 12
 *   gsr_sparse_return(acc) -- barrier --
 *   gsr_sparse_apply_weights_gather: weights[i, ch] += and cnt[i] += the <= world returned rows of each owned Gaussian i,
 *       in ascending rank order (float adds for the weights, integer adds for the count), in place: weights [n, CH]
 *       and cnt [n] accumulate over views like gsr_apply_weights. local_ws is the one gsr_sparse_preprocess filled. */
#define GSR_SPARSE_AW_CNT_SLOT 11
GSR_API int gsr_sparse_apply_weights_gather(const gsr_sparse_plan* plan, const void* local_ws, size_t local_bytes,
                                            const void* cand_ws, size_t cand_bytes, int32_t n, int32_t num_channels,
                                            float* weights, int32_t* cnt, void* stream);
/* Cross-rank barrier over peer memory (replaces the 4-byte NCCL all-reduces of the dense scheme: ~5 us instead of
 * ~25 us at 8 GPUs). Every rank's peer-visible block starts with GSR_PEER_CTRL_BYTES of control words, zeroed once at
 * creation: flags[rank] = number of the last barrier that rank reached, and the [GSR_MAX_PEERS, GSR_MAX_PEERS] int32
 * count matrix at byte GSR_PEER_CTRL_MATRIX_OFFSET (row s = n[s -> d], written by rank s: gsr_sparse_preprocess takes
 * counts_row = own row of the OWN block). peer_ctrl[r] is rank r's block as mapped here. `epoch` must increase by one per
 * barrier on this block, identically on every rank. with_matrix_row != 0 first copies this rank's row into every
 * peer's matrix, so that after the barrier every rank holds the complete matrix. Work queued on `stream` behind this
 * call starts only after every rank has reached the same barrier (a rank that never arrives costs ~2 s and sets the
 * int32 error word at byte GSR_PEER_CTRL_ERROR_OFFSET of the OWN block to 1 instead of hanging the GPU; the word is
 * sticky -- the host binding copies it out once per step and raises, gaussianeditor_b200/sparse_sharded.py). */
#define GSR_PEER_CTRL_BYTES 512
#define GSR_PEER_CTRL_ERROR_OFFSET 32
#define GSR_PEER_CTRL_MATRIX_OFFSET 64
GSR_API int gsr_peer_barrier(int32_t world, int32_t rank, void* const* peer_ctrl /* [world] host */, uint32_t epoch,
                     int32_t with_matrix_row, void* stream);
/* gsr_peer_barrier with a DEVICE epoch, for a step that is captured in a CUDA graph and replayed (where a host-side
 * epoch argument would be frozen). The epoch is the uint32 counter at byte GSR_PEER_CTRL_EPOCH_OFFSET of the OWN block:
 * the kernel reads it, runs the barrier with counter + 1 and stores counter + 1, so every barrier (and every replay of
 * one) advances it by one; only this rank writes it. status_word (device int32, may be NULL) is stored into slot `rank`
 * of the [GSR_MAX_PEERS] int32 status array at byte GSR_PEER_CTRL_STATUS_OFFSET of EVERY block, own included, before the
 * flag is raised (as the matrix row); it must be read before this rank's next barrier on the block. Timeout and sticky
 * error word as gsr_peer_barrier. A block must only ever see one kind of barrier: host epochs (gsr_peer_barrier) or
 * device epochs (this call). */
#define GSR_PEER_CTRL_EPOCH_OFFSET 320
#define GSR_PEER_CTRL_STATUS_OFFSET 352
GSR_API int gsr_peer_barrier_device(int32_t world, int32_t rank, void* const* peer_ctrl /* [world] host */,
                                    int32_t with_matrix_row, const int32_t* status_word /* may be NULL */, void* stream);
/* Copies the tile rows this rank owns of its [4,H,W] frame (colour + depth) into the frames of all other ranks
 * (128-bit peer stores): with one writer per pixel this replaces the all-reduce of the frames. A cross-rank barrier
 * must follow before the frames are read. */
GSR_API int gsr_frame_broadcast(const gsr_tile_owner* owner, int32_t image_width, int32_t image_height, const float* frame,
                        void* const* peer_frames /* [world] host */, void* stream);
/* gsr_frame_broadcast of a [planes,H,W] frame, 1 <= planes <= GSR_FRAME_MAX_PLANES (the same kernel; gsr_frame_broadcast
 * is the 4-plane call). The sharded alpha output uses 5: colour, depth, then alpha from gsr_shard_alpha_image. */
#define GSR_FRAME_MAX_PLANES 5
GSR_API int gsr_frame_broadcast_planes(const gsr_tile_owner* owner, int32_t image_width, int32_t image_height,
                                       int32_t planes, const float* frame, void* const* peer_frames /* [world] host */,
                                       void* stream);
/* All-gather of one small float row over peer memory: row[0..n) (device, 1 <= n <= GSR_PEER_ROW_FLOATS) is stored bit for
 * bit into slot `rank` of every rank's [GSR_MAX_PEERS][GSR_PEER_ROW_FLOATS] float slots (peer_slots[r] = rank r's slots
 * as mapped here, own entry included). A gsr_peer_barrier must follow before the slots are read, and every rank must
 * read its slots before it enters the next barrier on the same block (then no peer can store into them again before
 * they are read). The sparse exchange gathers the ranks' camera-gradient partials this way. */
#define GSR_PEER_ROW_FLOATS 64
GSR_API int gsr_peer_row_put(int32_t world, int32_t rank, const float* row, int32_t n,
                             void* const* peer_slots /* [world] host */, void* stream);
/* Camera gradients with the sparse exchange: gsr_sparse_backward_preprocess (depth = 0) or its DEPTH form (depth != 0)
 * that also runs the CAM preprocess backward on this rank's shard and writes THIS RANK'S PARTIAL camera gradients (its
 * Gaussians only; zeros for an empty shard) into `camera` (scratch: gsr_camera_scratch_bytes(shard.P)). Summing the
 * ranks' partials in ascending rank order on every rank gives every rank the same bits; at world 1 the partial is the
 * single-GPU gsr_backward_camera result. */
GSR_API int gsr_sparse_backward_preprocess_camera(const gsr_settings* s, const gsr_cloud* shard,
                                                  const gsr_sparse_plan* plan, const void* local_ws, size_t local_bytes,
                                                  const int32_t* radii_local, const void* cand_ws, size_t cand_bytes,
                                                  void* acc_slice, size_t acc_bytes, const gsr_grads* grads,
                                                  int32_t depth, const gsr_camera_grads* camera, void* stream);

/* ---- Gaussian-sharded path for a fixed capacity: no host copy, no host wait -------------------------------------
 * The sharded counterpart of gsr_forward_static: every call only enqueues work, so a sharded step can be captured in
 * a CUDA graph. One rank's forward:
 *   dense : gsr_shard_preprocess(_p2p) -> ALL-GATHER (or barrier) -> gsr_shard_order_static
 *           -> gsr_shard_render_static(capacity, status) -> gsr_shard_alpha_image (optional)
 *           -> ALL-REDUCE(sum) of [planes*H*W + 1] floats whose last float is this rank's status[1] (an exact sum of 0/1)
 *           -> gsr_shard_static_gate(flag_sum = that last float)
 *   sparse: gsr_sparse_preprocess(seg_cap) -> gsr_peer_barrier_device(with_matrix_row) -> gsr_sparse_order_static
 *           -> gsr_shard_render_static(P_total = world*seg_cap, capacity, status, counts_matrix, world, seg_cap)
 *           -> gsr_frame_broadcast(_planes) -> gsr_peer_barrier_device(status_word = status + 1)
 *           -> gsr_shard_static_gate(flags = the control block's status array [world], error_word) on a copy of the frame
 *   gsr_shard_order_static / gsr_sparse_order_static: gsr_shard_order / gsr_sparse_order without the host words.
 *   gsr_shard_render_static: gsr_shard_render with the binning sized for `capacity` instances (gsr_binning_bytes(P_total,
 *       capacity, W, H)); R is read on the device. status (device int32[4]) = {R of this rank, overflow, largest segment
 *       (0 without a matrix), 0}: overflow is R > capacity or, with counts_matrix ([world, GSR_MAX_PEERS], the complete
 *       matrix after the barrier), a segment above seg_cap (world*seg_cap must equal P_total). On overflow the owned
 *       tiles are emptied. Records past seg_cap were dropped by the push and every sparse kernel clamps a segment to
 *       seg_cap, so a truncated step stays memory-safe.
 *   gsr_shard_static_gate: if any of flags[0..num_flags) is non-zero, or *flag_sum != 0 (exactly one of the two is
 *       given), frame [planes,H,W] (planes 4 or 5) = background colour, depth 0, alpha 0, and this rank's tile ranges,
 *       per-tile backward start points and tile counts are zeroed, so every backward returns exact zeros (the
 *       deterministic reduction then reads nothing).
 *       status[1] = that global flag, the same on every rank; status[3] = *error_word (the control block's sticky
 *       barrier error word; NULL: 0). In the sparse exchange it must be queued before this rank's next barrier on the
 *       block: no peer can overwrite the status array before then.
 * The backward entry points take `capacity` as their num_rendered argument (binning, deterministic and accumulator
 * scratch sized by it), as with gsr_forward_static. Every argument is checked before the first launch. */
GSR_API int gsr_shard_order_static(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total, void* geometry,
                                   size_t geometry_bytes, int32_t* radii_total, void* stream);
GSR_API int gsr_sparse_order_static(const gsr_settings* s, const gsr_sparse_plan* plan, void* cand_ws, size_t cand_bytes,
                                    const int32_t* counts_matrix, int32_t* radii_cand, void* stream);
GSR_API int gsr_shard_render_static(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total, int32_t capacity,
                                    void* geometry, size_t geometry_bytes, void* binning, size_t binning_bytes,
                                    void* image, size_t image_bytes, const int32_t* radii_total, float* out_color,
                                    float* out_depth, int32_t* status /* [4] device */,
                                    const int32_t* counts_matrix /* may be NULL */, int32_t world, int32_t seg_cap,
                                    void* stream);
GSR_API int gsr_shard_static_gate(const gsr_settings* s, int32_t P_total, void* geometry, size_t geometry_bytes,
                                  void* image, size_t image_bytes, const int32_t* flags /* [num_flags] or NULL */,
                                  int32_t num_flags, const float* flag_sum /* or NULL */,
                                  const int32_t* error_word /* may be NULL */, float* frame, int32_t planes,
                                  int32_t* status /* [4] device */, void* stream);

/* ---- masked backward on the Gaussian-sharded path (opt-in; the sharded form of gsr_backward_masked) ----------
 * A tile owner's lists hold global indices (dense) or candidate slots (sparse), never the rows of a per-rank mask, so the
 * edit bit travels in the record: the masked preprocess twins below take the same arguments as their unmasked forms
 * plus grad_mask [shard.P] (this rank's rows, one byte each, device memory) and write a nonzero edit word into the
 * record of every visible Gaussian with grad_mask[i] != 0 (0 otherwise). Every exchange already moves whole records
 * (all-gather, p2p push, sparse push), so the bit reaches every tile owner in its own index space at no extra cost;
 * the sparse twins then run the unchanged mask / scan / push kernels. The forward outputs are unchanged.
 *   gsr_shard_backward_render_masked: gsr_shard_backward_render_alpha on records from a masked preprocess, with the
 *     work of unedited splats skipped as in gsr_backward_masked; dL_dout_alpha, dL_dout_depth and det_scratch may be
 *     NULL; mask_scratch holds gsr_grad_mask_scratch_bytes(W, H) bytes (contents irrelevant). Takes no mask: the bits
 *     are in the records. It serves the dense geometry and the sparse candidate workspace alike. Rows of unedited
 *     Gaussians are +0.0.
 *   gsr_{shard,sparse}_backward_preprocess[_raw]_masked: the unmasked forms' arguments (`depth` != 0: the rows carry
 *     dL/dz) plus grad_mask [shard.P]; an unedited Gaussian gets +0.0 in every gradient slot. camera must be NULL.
 * A NULL grad_mask or a non-NULL camera returns GSR_ERR_INVALID before any device work. */
GSR_API int gsr_shard_preprocess_masked(const gsr_settings* s, const gsr_cloud* shard, int32_t P_total, int32_t index_base,
                                        int32_t slice_len, void* geometry, size_t geometry_bytes, int32_t* radii_total,
                                        const uint8_t* grad_mask, void* stream);
GSR_API int gsr_shard_preprocess_raw_masked(const gsr_settings* s, const gsr_raw_cloud* shard, int32_t P_total,
                                            int32_t index_base, int32_t slice_len, void* geometry,
                                            size_t geometry_bytes, int32_t* radii_total, const uint8_t* grad_mask,
                                            void* stream);
GSR_API int gsr_shard_preprocess_p2p_masked(const gsr_settings* s, const gsr_cloud* shard, int32_t P_total,
                                            int32_t index_base, int32_t slice_len, void* const* peer_geometry,
                                            int32_t world, int32_t rank, size_t geometry_bytes, int32_t* radii_total,
                                            const uint8_t* grad_mask, void* stream);
GSR_API int gsr_shard_preprocess_p2p_raw_masked(const gsr_settings* s, const gsr_raw_cloud* shard, int32_t P_total,
                                                int32_t index_base, int32_t slice_len, void* const* peer_geometry,
                                                int32_t world, int32_t rank, size_t geometry_bytes,
                                                int32_t* radii_total, const uint8_t* grad_mask, void* stream);
GSR_API int gsr_sparse_preprocess_masked(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan,
                                         void* local_ws, size_t local_bytes, int32_t* radii_local,
                                         void* const* peer_cand, size_t cand_bytes, int32_t* counts_row,
                                         const uint8_t* grad_mask, void* stream);
GSR_API int gsr_sparse_preprocess_raw_masked(const gsr_settings* s, const gsr_raw_cloud* shard,
                                             const gsr_sparse_plan* plan, void* local_ws, size_t local_bytes,
                                             int32_t* radii_local, void* const* peer_cand, size_t cand_bytes,
                                             int32_t* counts_row, const uint8_t* grad_mask, void* stream);
GSR_API int gsr_shard_backward_render_masked(const gsr_settings* s, const gsr_tile_owner* owner, int32_t P_total,
                                             int32_t R, const void* geometry, size_t geometry_bytes,
                                             const void* binning, size_t binning_bytes, const void* image,
                                             size_t image_bytes, const float* dL_dout_color,
                                             const float* dL_dout_alpha /* may be NULL */,
                                             const float* dL_dout_depth /* may be NULL */, void* acc_total,
                                             size_t acc_bytes, void* det_scratch /* may be NULL */,
                                             size_t det_scratch_bytes, void* mask_scratch, size_t mask_scratch_bytes,
                                             void* stream);
GSR_API int gsr_shard_backward_preprocess_masked(const gsr_settings* s, const gsr_cloud* shard, int32_t P_total,
                                                 int32_t index_base, const void* geometry, size_t geometry_bytes,
                                                 const int32_t* radii_total, const void* acc_slice,
                                                 const gsr_grads* grads, int32_t depth,
                                                 const gsr_camera_grads* camera /* must be NULL */,
                                                 const uint8_t* grad_mask, void* stream);
GSR_API int gsr_shard_backward_preprocess_raw_masked(const gsr_settings* s, const gsr_raw_cloud* shard, int32_t P_total,
                                                     int32_t index_base, const void* geometry, size_t geometry_bytes,
                                                     const int32_t* radii_total, const void* acc_slice,
                                                     const gsr_raw_grads* grads, int32_t depth,
                                                     const uint8_t* grad_mask, void* stream);
GSR_API int gsr_sparse_backward_preprocess_masked(const gsr_settings* s, const gsr_cloud* shard,
                                                  const gsr_sparse_plan* plan, const void* local_ws,
                                                  size_t local_bytes, const int32_t* radii_local, const void* cand_ws,
                                                  size_t cand_bytes, void* acc_slice, size_t acc_bytes,
                                                  const gsr_grads* grads, int32_t depth,
                                                  const gsr_camera_grads* camera /* must be NULL */,
                                                  const uint8_t* grad_mask, void* stream);
GSR_API int gsr_sparse_backward_preprocess_raw_masked(const gsr_settings* s, const gsr_raw_cloud* shard,
                                                      const gsr_sparse_plan* plan, const void* local_ws,
                                                      size_t local_bytes, const int32_t* radii_local,
                                                      const void* cand_ws, size_t cand_bytes, void* acc_slice,
                                                      size_t acc_bytes, const gsr_raw_grads* grads, int32_t depth,
                                                      const uint8_t* grad_mask, void* stream);

/* ---- tuning / instrumentation ---------------------------------------------------------------------------
 * gsr_set_option("render_variant", v) etc.; unknown names return GSR_ERR_INVALID.
 * gsr_launch_count(): number of this library's kernel launches (CUB's included) since process start. */
GSR_API int gsr_set_option(const char* name, int64_t value);
GSR_API int64_t gsr_get_option(const char* name);
GSR_API int64_t gsr_launch_count(void);

/* Per-stage device timing (CUDA events recorded on the launching stream around each stage while the option
 * "profile" is 1). gsr_profile_read synchronises the device, adds up the elapsed times recorded since the last
 * read, writes GSR_NUM_STAGES milliseconds / call counts, and clears the records. */
#define GSR_NUM_STAGES 9
#define GSR_STAGE_NAMES "preprocess_fwd,depth_order_scan,emit_instances,tile_sort,tile_ranges,render_fwd,render_bwd,preprocess_bwd,apply_weights"
GSR_API int gsr_profile_read(double* ms_out, int64_t* calls_out);

/* ---- host-buffer convenience entry points (what a non-PyTorch host binds; used by bench.py's e2e leg) ---
 * One persistent device context; all pointers below are HOST pointers. The cloud is uploaded once with
 * gsr_host_upload_cloud; each gsr_host_step copies the camera + dL/dcolor image in (H2D) and the rendered
 * image + a few gradient checksums out (D2H) inside the call. */
typedef struct gsr_host_ctx gsr_host_ctx;
GSR_API gsr_host_ctx* gsr_host_create(void);
GSR_API void gsr_host_destroy(gsr_host_ctx* ctx);
GSR_API int gsr_host_upload_cloud(gsr_host_ctx* ctx, int32_t P, int32_t M, const float* means3D, const float* opacities,
                          const float* shs, const float* scales, const float* rotations);
/* settings pointers (bg, viewmatrix, projmatrix, campos) are HOST here. dL_dcolor_host may be NULL (forward only).
 * out_color_host [3,H,W] optional, out_radii_host [P] optional, grad_checksum_host[8] optional (sum of each
 * gradient tensor, computed on the device). Returns num_rendered (>=0) or an error (<0). */
GSR_API int64_t gsr_host_step(gsr_host_ctx* ctx, const gsr_settings* s_host, const float* dL_dcolor_host,
                      float* out_color_host, int32_t* out_radii_host, double* grad_checksum_host);

#ifdef __cplusplus
}
#endif
#endif /* GSR_B200_H_ */
