// ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Thin C-ABI shim (ours) around the reference's OWN, UNMODIFIED CUDA rasterizer
//   /root/reference/gaussiansplatting/submodules/diff-gaussian-rasterization/cuda_rasterizer/
//     {rasterizer_impl,forward,backward,apply_weights}.cu
// which oracle/Makefile compiles from where the sources lie into oracle/_ref/libdgr_ref.so
// (git-ignored, travels to the GPU box).  It plays the role of the reference's torch glue
// (rasterize_points.cu:35-234) without libtorch: the caller owns inputs/outputs (device
// pointers), the three opaque byte buffers (rasterize_points.cu:62-69) live in a grow-only
// cudaMalloc arena per context.  Used to (a) pin our CUDA path and the CPU oracle bit-for-bit
// against the real reference on the GPU, (b) time the reference's CUDA path as the A/B baseline.
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <functional>

#include "cuda_rasterizer/rasterizer.h"
#include "cuda_rasterizer/rasterizer_impl.h"

namespace {
struct Arena {
  char* ptr = nullptr;
  size_t cap = 0;
  char* get(size_t n) {
    if (n > cap) {
      if (ptr) cudaFree(ptr);
      cap = n + n / 4 + 4096;
      if (cudaMalloc(&ptr, cap) != cudaSuccess) { ptr = nullptr; cap = 0; }
    }
    return ptr;
  }
  ~Arena() { if (ptr) cudaFree(ptr); }
};
struct RefCtx {
  Arena geom, binning, img;
};
}  // namespace

#define REF_API extern "C" __attribute__((visibility("default")))

REF_API void* dgr_create() { return new RefCtx(); }
REF_API void dgr_destroy(void* c) { delete (RefCtx*)c; }

// CudaRasterizer::Rasterizer::forward (rasterizer_impl.cu:179-285); returns num_rendered.
REF_API int dgr_forward(void* c, int P, int D, int M, const float* bg, int W, int H, const float* means3D,
                        const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                        float scale_modifier, const float* rotations, const float* cov3D_precomp,
                        const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                        float tan_fovy, int prefiltered, float* out_color, float* out_depth, int* radii) {
  RefCtx* x = (RefCtx*)c;
  std::function<char*(size_t)> g = [x](size_t n) { return x->geom.get(n); };
  std::function<char*(size_t)> b = [x](size_t n) { return x->binning.get(n); };
  std::function<char*(size_t)> i = [x](size_t n) { return x->img.get(n); };
  return CudaRasterizer::Rasterizer::forward(g, b, i, P, D, M, bg, W, H, means3D, shs, colors_precomp, opacities,
                                             scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix,
                                             campos, tan_fovx, tan_fovy, prefiltered != 0, out_color, out_depth, radii,
                                             false);
}

// CudaRasterizer::Rasterizer::backward (rasterizer_impl.cu:289-341). Gradient buffers must be zero-filled by
// the caller exactly as rasterize_points.cu:120-128 does.
REF_API void dgr_backward(void* c, int P, int D, int M, int R, const float* bg, int W, int H, const float* means3D,
                          const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                          const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                          const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy,
                          const int* radii, const float* dL_dpix, float* dL_dmean2D, float* dL_dconic,
                          float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                          float* dL_dscale, float* dL_drot) {
  RefCtx* x = (RefCtx*)c;
  CudaRasterizer::Rasterizer::backward(P, D, M, R, bg, W, H, means3D, shs, colors_precomp, scales, scale_modifier,
                                       rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy,
                                       radii, x->geom.ptr, x->binning.ptr, x->img.ptr, dL_dpix, dL_dmean2D, dL_dconic,
                                       dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot,
                                       false);
}

REF_API void dgr_mark_visible(int P, float* means3D, float* viewmatrix, float* projmatrix, bool* present) {
  CudaRasterizer::Rasterizer::markVisible(P, means3D, viewmatrix, projmatrix, present);
}

// CudaRasterizer::Rasterizer::apply_weights (rasterizer_impl.cu:343-446)
REF_API void dgr_apply_weights(void* c, int P, int D, int M, const float* bg, int W, int H, const float* means3D,
                               const float* shs, float* weights, const float* opacities, const float* scales,
                               float scale_modifier, const float* rotations, const float* cov3D_precomp,
                               const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                               float tan_fovy, int prefiltered, const float* image_weights, int* radii, int* cnt,
                               int num_channels) {
  RefCtx* x = (RefCtx*)c;
  std::function<char*(size_t)> g = [x](size_t n) { return x->geom.get(n); };
  std::function<char*(size_t)> b = [x](size_t n) { return x->binning.get(n); };
  std::function<char*(size_t)> i = [x](size_t n) { return x->img.get(n); };
  CudaRasterizer::Rasterizer::apply_weights(g, b, i, P, D, M, bg, W, H, means3D, shs, weights, opacities, scales,
                                            scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, campos,
                                            tan_fovx, tan_fovy, prefiltered != 0, image_weights, radii, cnt,
                                            num_channels, false);
}

// Decode the opaque buffers with the reference's own fromChunk (rasterizer_impl.cu:135-175) and hand back
// DEVICE pointers to the intermediates, so tests can compare them bit for bit. out[13]:
// depths, clamped, means2D, cov3D, conic_opacity, rgb, point_offsets, tiles_touched,
// point_list_keys, point_list, ranges, n_contrib, accum_alpha
REF_API void dgr_state_ptrs(void* c, int P, int W, int H, int R, void** out) {
  RefCtx* x = (RefCtx*)c;
  char* gp = x->geom.ptr;
  char* bp = x->binning.ptr;
  char* ip = x->img.ptr;
  CudaRasterizer::GeometryState gs = CudaRasterizer::GeometryState::fromChunk(gp, P);
  CudaRasterizer::ImageState is = CudaRasterizer::ImageState::fromChunk(ip, (size_t)W * H);
  out[0] = gs.depths; out[1] = gs.clamped; out[2] = gs.means2D; out[3] = gs.cov3D; out[4] = gs.conic_opacity;
  out[5] = gs.rgb; out[6] = gs.point_offsets; out[7] = gs.tiles_touched;
  if (bp && R > 0) {
    CudaRasterizer::BinningState bs = CudaRasterizer::BinningState::fromChunk(bp, R);
    out[8] = bs.point_list_keys; out[9] = bs.point_list;
  } else {
    out[8] = nullptr; out[9] = nullptr;
  }
  out[10] = is.ranges; out[11] = is.n_contrib; out[12] = is.accum_alpha;
}

REF_API int dgr_last_cuda_error() { return (int)cudaGetLastError(); }

// device->device copy of an intermediate into a caller-owned buffer (after a full device sync)
REF_API int dgr_copy_d2d(void* dst, const void* src, size_t bytes) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToDevice);
  return (int)e;
}
