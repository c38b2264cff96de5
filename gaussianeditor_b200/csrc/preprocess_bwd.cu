// Backward of the per-Gaussian preprocess for sm_90a: 2-D gradients -> gradients of means3D, scales,
// rotations (or cov3D), SH coefficients (or colours) and opacity.
//
// Semantics: the reference's two kernels computeCov2DCUDA (cuda_rasterizer/backward.cu:144-274) and
// preprocessCUDA (bwd, :346-396 with computeColorFromSH :20-139 and computeCov3D :278-341), in the order of
// rasterizer_impl.cu:333-340 (the covariance kernel ASSIGNS dL/dmean, the second kernel adds the projection and
// SH view-direction terms).  Fused here into ONE pass over the cloud:
//   * every input byte of a Gaussian is read once (the reference reads mean/radii/cov3D twice and round-trips
//     dL/dcov3D and dL/dmean through HBM between its two kernels); cov3D is recomputed from scale/rotation
//     instead of being stored by the forward (saves 24 B/Gaussian written + read);
//   * the kernel writes EVERY gradient element itself -- zeros for culled Gaussians and for SH coefficients
//     above the active degree -- so the caller allocates outputs uninitialised and the reference's nine
//     zero-fill kernels (rasterize_points.cu:120-128; 300 MB of memset at config 3) disappear;
//   * SH rows (192 B in, 192 B out per Gaussian at degree 3) move through the TMA unit: cp.async.bulk
//     global->shared for visible Gaussians only, cp.async.bulk shared->global for the gradient rows, staged in
//     padded 208-byte shared-memory rows owned by one thread each (conflict-free 128-bit accesses, no
//     block-level synchronisation besides the load mbarrier).
#include <type_traits>

#include "common.cuh"

namespace gsr {

namespace {

constexpr int PB_THREADS = 128;
constexpr int ROW_WORDS = 52;

struct M3 {
  float m[3][3];  // m[column][row]
};
__device__ __forceinline__ M3 mat_mul(const M3& A, const M3& B) {
  M3 R;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int r = 0; r < 3; r++) R.m[c][r] = A.m[0][r] * B.m[c][0] + A.m[1][r] * B.m[c][1] + A.m[2][r] * B.m[c][2];
  return R;
}
__device__ __forceinline__ M3 mat_t(const M3& A) {
  M3 R;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int r = 0; r < 3; r++) R.m[c][r] = A.m[r][c];
  return R;
}

struct PbArgs {
  int P, D, M, W, H;
  float tan_fovx, tan_fovy, h_x, h_y, scale_modifier;
  const float* means3D;
  const float* shs;
  const float* scales;
  const float* rotations;
  const float* cov3D_precomp;
  const float* view;
  const float* proj;
  const float* campos;
  const int32_t* radii;
  const uint8_t* clamped;
  const float* acc;
  float* dL_dmeans3D;
  float* dL_dmeans2D;
  float* dL_dcolors;
  float* dL_dopacity;
  float* dL_dcov3D;
  float* dL_dsh;
  float* dL_dscales;
  float* dL_drotations;
  // RAW variant (fused activations): shs = features_dc [P,1,3], dL_dsh = d features_dc, opacities = logits,
  // scales = log-scales, rotations = unnormalised; gradients are taken w.r.t. those raw parameters
  const float* opacities;
  const float* features_rest;
  float* dL_dfeatures_rest;
  float* cam_partial;  // CAM variant: [nblocks, CAM_STRIDE] block partial sums of the camera gradients
};
// MASK variant (gsr_backward_masked): a separate type, so that every other instantiation keeps its parameter block
struct PbMaskArgs : PbArgs {
  const uint8_t* grad_mask;  // [P] zero: the Gaussian takes the culled branch (all gradients +0)
};
// whether Gaussian idx takes gradients: always without a mask
__device__ __forceinline__ bool edited(const PbArgs&, int) { return true; }
__device__ __forceinline__ bool edited(const PbMaskArgs& a, int idx) { return a.grad_mask[idx] != 0; }

__device__ __forceinline__ M3 quat_to_R(float r, float x, float y, float z) {
  M3 R;
  R.m[0][0] = 1.f - 2.f * (y * y + z * z); R.m[0][1] = 2.f * (x * y - r * z); R.m[0][2] = 2.f * (x * z + r * y);
  R.m[1][0] = 2.f * (x * y + r * z); R.m[1][1] = 1.f - 2.f * (x * x + z * z); R.m[1][2] = 2.f * (y * z - r * x);
  R.m[2][0] = 2.f * (x * z - r * y); R.m[2][1] = 2.f * (y * z + r * x); R.m[2][2] = 1.f - 2.f * (x * x + y * y);
  return R;
}

// Camera gradients (opt-in, gsr_backward_camera; the reference has none: its autograd returns None for the settings,
// diff_gaussian_rasterization/__init__.py:213-223). viewmatrix, projmatrix and campos are treated as INDEPENDENT inputs,
// exactly as the forward reads them; a caller that builds projmatrix / campos from the view matrix chains the three.
// Compact per-thread accumulator layout, CAM_N floats:
//   [4k + j]      dL/dview[k + 4j]   k = 0..2 (row of t = view * mean), j = 0..3 (x, y, z, 1)
//   [12 + 4r + j] dL/dproj[i + 4j]   i = (0, 1, 3)[r] (p_hom.x, .y, .w)
//   [24 + c]      dL/dcampos[c]
constexpr int CAM_N = 27, CAM_STRIDE = 32;

// DEPTH: the accumulators carry dL/dz in slot 9 (acc2.y; the depth image's gradient, render_bwd.cu). z = t.z is the view
// depth the forward blends, not clamped, so dL/dt.z gains it, and with it the mean and, under CAM, view row 2.
template <bool BULK, bool RAW = false, bool CAM = false, bool DEPTH = false>
__global__ void __launch_bounds__(PB_THREADS) preprocess_bwd_kernel(const PbArgs a) {
  constexpr bool MASK = false;
#include "preprocess_bwd_body.inc"
}

// MASK (gsr_backward_masked): an unedited Gaussian (grad_mask[idx] == 0) is treated as culled: it loads no SH row and
// writes zeros. A kernel of its own name, so that every existing instantiation keeps its symbol; no camera forms.
template <bool BULK, bool RAW, bool DEPTH>
__global__ void __launch_bounds__(PB_THREADS) preprocess_bwd_masked_kernel(const PbMaskArgs a) {
  constexpr bool CAM = false, MASK = true;
#include "preprocess_bwd_body.inc"
}

// sums the per-block partials and scatters the compact layout into dL/dviewmatrix[16], dL/dprojmatrix[16], dL/dcampos[3]
__global__ void __launch_bounds__(1024) camera_reduce_kernel(const float* __restrict__ partial, int nblocks, float* __restrict__ dview,
                                                             float* __restrict__ dproj, float* __restrict__ dcampos) {
  __shared__ float s[32][CAM_STRIDE + 1];
  const int c = threadIdx.x & 31, r = threadIdx.x >> 5;
  float v = 0.f;
  for (int b = r; b < nblocks; b += 32) v += partial[(size_t)b * CAM_STRIDE + c];
  s[r][c] = v;
  __syncthreads();
  if (threadIdx.x < 16) { dview[threadIdx.x] = 0.f; dproj[threadIdx.x] = 0.f; }
  __syncthreads();
  if (r == 0 && c < CAM_N) {
    float t = 0.f;
    for (int k = 0; k < 32; k++) t += s[k][c];
    if (c < 12) dview[(c >> 2) + 4 * (c & 3)] = t;
    else if (c < 24) { const int rr = (c - 12) >> 2, j = (c - 12) & 3; dproj[(rr == 2 ? 3 : rr) + 4 * j] = t; }
    else dcampos[c - 24] = t;
  }
}

}  // namespace

size_t camera_scratch_bytes(int P) { return align_up((size_t)((P + PB_THREADS - 1) / PB_THREADS + 1) * CAM_STRIDE * sizeof(float)); }

int launch_preprocess_bwd(const gsr_settings& s, const gsr_cloud& c, const GeometryWS& g, const int32_t* radii,
                          const float* acc, const gsr_grads& gr, cudaStream_t st, const RawBackward* raw,
                          const CameraBackward* cam, bool depth, const uint8_t* grad_mask) {
  PbMaskArgs a;
  a.cam_partial = cam ? cam->scratch : nullptr;
  a.opacities = c.opacities;
  a.features_rest = raw ? raw->features_rest : nullptr;
  a.dL_dfeatures_rest = raw ? raw->dL_dfeatures_rest : nullptr;
  a.P = c.P; a.D = s.sh_degree; a.M = s.sh_coeffs; a.W = s.image_width; a.H = s.image_height;
  a.tan_fovx = s.tanfovx; a.tan_fovy = s.tanfovy;
  a.h_y = a.H / (2.0f * s.tanfovy);
  a.h_x = a.W / (2.0f * s.tanfovx);
  a.scale_modifier = s.scale_modifier;
  a.means3D = c.means3D; a.shs = c.shs; a.scales = c.scales; a.rotations = c.rotations;
  a.cov3D_precomp = c.cov3D_precomp; a.view = s.viewmatrix; a.proj = s.projmatrix; a.campos = s.campos;
  a.radii = radii; a.clamped = g.clamped; a.acc = acc;
  a.dL_dmeans3D = gr.dL_dmeans3D; a.dL_dmeans2D = gr.dL_dmeans2D; a.dL_dcolors = gr.dL_dcolors;
  a.dL_dopacity = gr.dL_dopacity; a.dL_dcov3D = gr.dL_dcov3D; a.dL_dsh = gr.dL_dsh;
  a.dL_dscales = gr.dL_dscales; a.dL_drotations = gr.dL_drotations;
  const int grid = (c.P + PB_THREADS - 1) / PB_THREADS;
  const bool bulk = g_opt.preprocess_variant >= 1 && c.shs != nullptr && gr.dL_dsh != nullptr &&
                    (s.sh_coeffs * 12) % 16 == 0 && s.sh_coeffs * 12 <= 192 &&
                    (reinterpret_cast<uintptr_t>(c.shs) % 16) == 0 && (reinterpret_cast<uintptr_t>(gr.dL_dsh) % 16) == 0;
  if (grad_mask) {  // masked backward: the plain, RAW, DEPTH and RAW + DEPTH forms, BULK where the default takes it
    if (cam) { set_error("camera gradients are not available with a gradient mask"); return GSR_ERR_INVALID; }
    a.grad_mask = grad_mask;
    if (raw) {
      if (depth) preprocess_bwd_masked_kernel<false, true, true><<<grid, PB_THREADS, 0, st>>>(a);
      else preprocess_bwd_masked_kernel<false, true, false><<<grid, PB_THREADS, 0, st>>>(a);
    } else if (bulk) {
      if (depth) preprocess_bwd_masked_kernel<true, false, true><<<grid, PB_THREADS, 0, st>>>(a);
      else preprocess_bwd_masked_kernel<true, false, false><<<grid, PB_THREADS, 0, st>>>(a);
    } else {
      if (depth) preprocess_bwd_masked_kernel<false, false, true><<<grid, PB_THREADS, 0, st>>>(a);
      else preprocess_bwd_masked_kernel<false, false, false><<<grid, PB_THREADS, 0, st>>>(a);
    }
    g_launches++;
    return check_launch("preprocess_bwd (masked)", s.debug != 0, st);
  }
  const PbArgs& pa = a;  // every other form takes the plain parameter block
  if (cam) {  // opt-in camera gradients (never together with the RAW entry point)
    if (raw) { set_error("camera gradients are not available on the fused-activation entry point"); return GSR_ERR_INVALID; }
    if (depth) {
      if (bulk)
        preprocess_bwd_kernel<true, false, true, true><<<grid, PB_THREADS, 0, st>>>(pa);
      else
        preprocess_bwd_kernel<false, false, true, true><<<grid, PB_THREADS, 0, st>>>(pa);
    } else if (bulk) {
      preprocess_bwd_kernel<true, false, true><<<grid, PB_THREADS, 0, st>>>(pa);
    } else {
      preprocess_bwd_kernel<false, false, true><<<grid, PB_THREADS, 0, st>>>(pa);
    }
    camera_reduce_kernel<<<1, 1024, 0, st>>>(cam->scratch, grid, cam->dL_dviewmatrix, cam->dL_dprojmatrix, cam->dL_dcampos);
    g_launches += 2;
    return check_launch("preprocess_bwd (camera)", s.debug != 0, st);
  }
  if (depth) {
    if (raw)
      preprocess_bwd_kernel<false, true, false, true><<<grid, PB_THREADS, 0, st>>>(pa);
    else if (bulk)
      preprocess_bwd_kernel<true, false, false, true><<<grid, PB_THREADS, 0, st>>>(pa);
    else
      preprocess_bwd_kernel<false, false, false, true><<<grid, PB_THREADS, 0, st>>>(pa);
  } else if (raw) {
    preprocess_bwd_kernel<false, true><<<grid, PB_THREADS, 0, st>>>(pa);
  } else if (bulk) {
    preprocess_bwd_kernel<true><<<grid, PB_THREADS, 0, st>>>(pa);
  } else {
    preprocess_bwd_kernel<false><<<grid, PB_THREADS, 0, st>>>(pa);
  }
  g_launches++;
  return check_launch("preprocess_bwd", s.debug != 0, st);
}

}  // namespace gsr
