// Forward per-Gaussian preprocess for sm_90a: near cull, projection, 3-D covariance, EWA 2-D covariance,
// conic, screen radius, tile rectangle, SH -> RGB; writes one 48-byte splat record per visible Gaussian.
//
// Semantics follow the reference kernel preprocessCUDA (cuda_rasterizer/forward.cu:155-256 with its helpers
// computeCov3D :118-152, computeCov2D :74-113, computeColorFromSH :20-71, and auxiliary.h:41-56,139-164).
// The integer outputs (radii, tile counts) are discontinuous functions of the float chain and the conic is
// ill-conditioned for elongated splats, so the projection / covariance chain is pinned with _rn intrinsics to
// the exact FMA contraction nvcc produces for the reference's expression trees (GLM's column-major mat3 product
// order, type_mat3x3.inl:486-518; ndc2Pix in fp64), decoded from the SASS of the unmodified reference build.
// radii, tile counts, means2D, depth, conic and rgb are bit-identical to the reference's CUDA build on the same GPU
// (tests/test_parity_gpu.py).
//
// Hopper-specific structure:
//   * the 192-byte SH row of each Gaussian that survives the near-plane test is fetched by the TMA unit
//     (cp.async.bulk, one 16-byte-aligned row per thread, completion on one CTA mbarrier) into a padded
//     shared-memory row while the thread does the covariance math; culled Gaussians (39 % of config 3)
//     never touch their SH bytes. Rows are padded to 208 B so the 128-bit row reads are bank-conflict free.
//   * outputs are packed AoS (SplatRecord) so the render kernels gather three float4 per splat.
#include "common.cuh"

namespace gsr {

namespace {

constexpr int PRE_THREADS = 128;
constexpr int SH_ROW_WORDS = 52;  // 48 payload + 4 pad words: 208-byte rows

struct M3 {
  float m[3][3];  // m[column][row], GLM convention
};

__device__ __forceinline__ float ndc_to_pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

struct PreArgs {
  int P, D, M, W, H, gx, gy;
  float tan_fovx, tan_fovy, focal_x, focal_y, scale_modifier;
  const float* means3D;
  const float* opacities;
  const float* shs;
  const float* colors_precomp;
  const float* scales;
  const float* rotations;
  const float* cov3D_precomp;
  const float* view;
  const float* proj;
  const float* campos;
  SplatRecord* records;
  uint32_t* tiles_touched;
  uint8_t* clamped;
  uint32_t* depth_keys;
  uint32_t* ident;
  int32_t* radii;
  // RAW kernel variant (fused activations, gsr_b200.h: gsr_raw_cloud): `opacities` are logits, `scales` log-scales,
  // `rotations` unnormalised, `shs` is features_dc [P,1,3] and `features_rest` [P,M-1,3] holds the other coefficients.
  const float* features_rest;
  // Fused all-gather of the Gaussian-sharded path (P2P kernel variant): the CTA's block of records is pushed with one
  // TMA bulk store per destination into the records array of every rank (own copy included) over NVLink peer memory.
  SplatRecord* peer_records[GSR_MAX_PEERS];  // pointers to THIS shard's slice inside each rank's records array
  int npeers;
  // Tile binning without a pass over the instances (tile_binning.cu): every visible Gaussian adds the four corners of
  // its tile rectangle to a 2-D difference array (its 2-D prefix sum is the per-tile instance count -> tile ranges and
  // the radix histograms, its weighted sum is R). Null in the sharded paths (the tile owner does it).
  int32_t* tile_diff;
  int diff_copies;
  int vec_ok;  // means3D and scales are 16-byte aligned: full blocks use 128-bit cooperative loads
};

// SH basis weights of forward.cu:30-61 for the unit view direction (x,y,z), pinned to the operation sequence nvcc emits
// for the reference (decoded from its SASS): every weight is a product of plain multiplications in this association,
// the polynomial factors use the FMA forms noted, and each colour channel is one FMA chain res = fma(w_k, sh_k, res)
// in ascending k starting from C0*sh_0. Signs of k = 1, 3 are folded into the weight (exact).
__device__ __forceinline__ void sh_weights(int deg, float x, float y, float z, float* w) {
  const float C0 = 0.28209479177387814f, C1 = 0.4886025119029199f;
  const float C2_0 = 1.0925484305920792f, C2_1 = -1.0925484305920792f, C2_2 = 0.31539156525252005f,
              C2_3 = -1.0925484305920792f, C2_4 = 0.5462742152960396f;
  const float C3_0 = -0.5900435899266435f, C3_1 = 2.890611442640554f, C3_2 = -0.4570457994644658f,
              C3_3 = 0.3731763325901154f, C3_4 = -0.4570457994644658f, C3_5 = 1.445305721320277f,
              C3_6 = -0.5900435899266435f;
  w[0] = C0;
  if (deg > 0) {
    w[1] = -__fmul_rn(y, C1);
    w[2] = __fmul_rn(z, C1);
    w[3] = -__fmul_rn(x, C1);
    if (deg > 1) {
      const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
      const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
      const float zz2 = __fadd_rn(zz, zz);
      const float xx_yy = __fadd_rn(xx, -yy);
      w[4] = __fmul_rn(xy, C2_0);
      w[5] = __fmul_rn(yz, C2_1);
      w[6] = __fmul_rn(__fadd_rn(__fadd_rn(zz2, -xx), -yy), C2_2);   // (2zz - xx) - yy
      w[7] = __fmul_rn(xz, C2_3);
      w[8] = __fmul_rn(xx_yy, C2_4);
      if (deg > 2) {
        const float p4 = __fadd_rn(__fmaf_rn(zz, 4.0f, -xx), -yy);   // (4zz - xx) - yy
        w[9] = __fmul_rn(__fmul_rn(y, C3_0), __fmaf_rn(xx, 3.0f, -yy));
        w[10] = __fmul_rn(__fmul_rn(xy, C3_1), z);
        w[11] = __fmul_rn(__fmul_rn(y, C3_2), p4);
        w[12] = __fmul_rn(__fmul_rn(z, C3_3), __fmaf_rn(yy, -3.0f, __fmaf_rn(xx, -3.0f, zz2)));
        w[13] = __fmul_rn(__fmul_rn(x, C3_4), p4);
        w[14] = __fmul_rn(xx_yy, __fmul_rn(z, C3_5));
        w[15] = __fmul_rn(__fmul_rn(x, C3_6), __fmaf_rn(yy, -3.0f, xx));
      }
    }
  }
}
template <typename ShFn>
__device__ __forceinline__ float sh_channel(int deg, const float* w, ShFn sh) {
  float res = __fmul_rn(sh(0), w[0]);
  const int nb = (deg + 1) * (deg + 1);
#pragma unroll
  for (int k = 1; k < 16; k++)
    if (k < nb) res = __fmaf_rn(w[k], sh(k), res);
  return __fadd_rn(res, 0.5f);
}

// torch.sigmoid / torch.exp / F.normalize restated for the RAW variant (scene/gaussian_model.py:221-258 applies them in
// PyTorch before every render; here they cost nothing extra in HBM traffic)
__device__ __forceinline__ float sigmoid_act(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// Arguments of the masked forms (the Gaussian-sharded masked backward): a separate type, so that every other kernel
// keeps its parameter block.
struct PreMaskArgs : PreArgs {
  const uint8_t* grad_mask;  // [P] nonzero: the Gaussian is edited; null for the unmasked kernels
};
// the edit word a visible Gaussian's record carries in q1.w (never called without a mask)
__device__ __forceinline__ uint32_t edit_word(const PreArgs&, int) { return 0u; }
__device__ __forceinline__ uint32_t edit_word(const PreMaskArgs& a, int idx) {
  return __ldg(a.grad_mask + idx) != 0 ? GRAD_MASK_EDIT : 0u;
}

template <bool BULK_SH, bool P2P = false, bool RAW = false>
__global__ void __launch_bounds__(PRE_THREADS) preprocess_fwd_kernel(const PreArgs a) {
  constexpr bool MASK = false;
#include "preprocess_fwd_body.inc"
}
// MASK: preprocess_fwd_kernel writing the edit word of grad_mask[idx] into q1.w of each visible record (one byte load
// per Gaussian), so that the records carry the edit bit to every tile owner through whichever exchange moves them (NCCL
// all-gather, the P2P bulk stores of this kernel, the sparse push). A kernel of its own name, so that every existing
// instantiation keeps its symbol.
template <bool BULK_SH, bool P2P, bool RAW>
__global__ void __launch_bounds__(PRE_THREADS) preprocess_fwd_masked_kernel(const PreMaskArgs a) {
  constexpr bool MASK = true;
#include "preprocess_fwd_body.inc"
}
template <bool BULK_SH, bool P2P = false, bool RAW = false>
void launch_form(const PreMaskArgs& a, int grid, cudaStream_t st) {
  if (a.grad_mask != nullptr)
    preprocess_fwd_masked_kernel<BULK_SH, P2P, RAW><<<grid, PRE_THREADS, 0, st>>>(a);
  else
    preprocess_fwd_kernel<BULK_SH, P2P, RAW><<<grid, PRE_THREADS, 0, st>>>(a);
}

__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ view,
                                    uint8_t* __restrict__ present) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P) return;
  float x = means3D[3 * idx], y = means3D[3 * idx + 1], z = means3D[3 * idx + 2];
  float vz = view[2] * x + view[6] * y + view[10] * z + view[14];
  present[idx] = !(vz <= 0.2f);
}

}  // namespace

int launch_preprocess_fwd(const gsr_settings& s, const gsr_cloud& c, const GeometryWS& g, int32_t* radii,
                          cudaStream_t st, SplatRecord* const* peer_records, int npeers, bool raw,
                          const float* features_rest, bool count_tiles, const uint8_t* grad_mask) {
  PreMaskArgs a;
  a.grad_mask = grad_mask;
  a.features_rest = features_rest;
  a.npeers = npeers;
  for (int i = 0; i < GSR_MAX_PEERS; i++) a.peer_records[i] = i < npeers ? peer_records[i] : nullptr;
  a.P = c.P; a.D = s.sh_degree; a.M = s.sh_coeffs; a.W = s.image_width; a.H = s.image_height;
  a.gx = (a.W + TILE - 1) / TILE; a.gy = (a.H + TILE - 1) / TILE;
  a.tan_fovx = s.tanfovx; a.tan_fovy = s.tanfovy;
  a.focal_y = a.H / (2.0f * s.tanfovy);  // rasterizer_impl.cu:190-191
  a.focal_x = a.W / (2.0f * s.tanfovx);
  a.scale_modifier = s.scale_modifier;
  a.means3D = c.means3D; a.opacities = c.opacities; a.shs = c.shs; a.colors_precomp = c.colors_precomp;
  a.scales = c.scales; a.rotations = c.rotations; a.cov3D_precomp = c.cov3D_precomp;
  a.view = s.viewmatrix; a.proj = s.projmatrix; a.campos = s.campos;
  a.records = g.records; a.tiles_touched = g.tiles_touched; a.clamped = g.clamped;
  a.depth_keys = g.depth_keys; a.ident = g.ident; a.radii = radii;
  a.vec_ok = ((reinterpret_cast<uintptr_t>(c.means3D) | reinterpret_cast<uintptr_t>(c.scales)) & 15) == 0;
  a.tile_diff = count_tiles ? g.tile_diff : nullptr;
  a.diff_copies = tile_diff_copies(a.gx, a.gy);
  const int grid = (c.P + PRE_THREADS - 1) / PRE_THREADS;
  // TMA row fetch needs 16-byte aligned rows: M*12 % 16 == 0 and an aligned base pointer.
  const bool bulk = g_opt.preprocess_variant >= 1 && c.colors_precomp == nullptr && c.shs != nullptr &&
                    (s.sh_coeffs * 12) % 16 == 0 && (reinterpret_cast<uintptr_t>(c.shs) % 16) == 0 &&
                    (s.sh_coeffs * 12) <= 192;
  if (raw) {
    if (npeers > 0)
      launch_form<false, true, true>(a, grid, st);
    else
      launch_form<false, false, true>(a, grid, st);
  } else if (npeers > 0) {
    if (bulk)
      launch_form<true, true>(a, grid, st);
    else
      launch_form<false, true>(a, grid, st);
  } else if (bulk)
    launch_form<true>(a, grid, st);
  else
    launch_form<false>(a, grid, st);
  g_launches++;
  return check_launch("preprocess_fwd", s.debug != 0, st);
}

int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present, cudaStream_t st) {
  mark_visible_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, viewmatrix, present);
  g_launches++;
  return check_launch("mark_visible", false, st);
}

}  // namespace gsr
