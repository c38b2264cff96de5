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

template <bool BULK_SH, bool P2P = false, bool RAW = false>
__global__ void __launch_bounds__(PRE_THREADS) preprocess_fwd_kernel(const PreArgs a) {
  // RAW + P2P is fine: the features_rest block arrives in s_rest on `bar`, the records leave from s_rec without it
  static_assert(!(RAW && BULK_SH), "the RAW variant stages its SH block itself");
  __shared__ __align__(16) float sh_rows[BULK_SH ? PRE_THREADS * SH_ROW_WORDS : 4];
  __shared__ __align__(128) float4 s_rec[P2P ? PRE_THREADS * 3 : 1];  // the CTA's records, contiguous like in HBM
  // RAW: the CTA's block of features_rest rows (128 x 12*(M-1) bytes, contiguous and 16-byte aligned in HBM although
  // a single 180-byte row is not), fetched with ONE bulk copy
  __shared__ __align__(128) float s_rest[RAW ? PRE_THREADS * 45 : 1];
  __shared__ uint64_t bar;

  // the CTA's means and scales (128 x 12 B each, contiguous in HBM) arrive through 96 coalesced 128-bit loads per
  // array instead of three stride-3 scalar loads per thread; the word stride 3 is coprime with the 32 banks
  __shared__ __align__(16) float s_mean[PRE_THREADS * 3];
  __shared__ __align__(16) float s_scale[PRE_THREADS * 3];

  const int idx = blockIdx.x * PRE_THREADS + threadIdx.x;
  const bool live = idx < a.P;
  {
    const int first = blockIdx.x * PRE_THREADS;
    const int nhere = min(PRE_THREADS, a.P - first);
    const bool has_scale = a.cov3D_precomp == nullptr;
    if (nhere == PRE_THREADS && a.vec_ok) {
      if (threadIdx.x < 96)
        reinterpret_cast<float4*>(s_mean)[threadIdx.x] = __ldg(reinterpret_cast<const float4*>(a.means3D + (size_t)3 * first) + threadIdx.x);
      if (has_scale && threadIdx.x >= 32)
        reinterpret_cast<float4*>(s_scale)[threadIdx.x - 32] = __ldg(reinterpret_cast<const float4*>(a.scales + (size_t)3 * first) + (threadIdx.x - 32));
    } else {
      for (int i = threadIdx.x; i < 3 * nhere; i += PRE_THREADS) {
        s_mean[i] = a.means3D[(size_t)3 * first + i];
        if (has_scale) s_scale[i] = a.scales[(size_t)3 * first + i];
      }
    }
  }
  // this thread's own rotation / opacity are requested before the barrier too, so that all of the kernel's first-touch
  // loads are in flight together (one exposed memory latency instead of one per dependent stage)
  float4 q_pref = make_float4(0.f, 0.f, 0.f, 0.f);
  float op_pref = 0.f;
  if (live) {
    if (a.rotations != nullptr) q_pref = __ldg(reinterpret_cast<const float4*>(a.rotations) + idx);
    op_pref = a.opacities[idx];
  }
  if (!(BULK_SH || RAW)) __syncthreads();  // the other variants synchronise right below (mbarrier init)

  if (BULK_SH || RAW) {
    if (threadIdx.x == 0) {
      mbar_init(&bar, RAW ? 1 : PRE_THREADS);
      fence_mbar_init();
    }
    __syncthreads();
  }

  // ---- near cull (auxiliary.h:139-164; only the view-space z test is active) ----
  float3 p_orig = make_float3(0.f, 0.f, 0.f);
  float3 p_view = make_float3(0.f, 0.f, 0.f);
  bool vis = false;
  if (live) {
    p_orig = make_float3(s_mean[3 * threadIdx.x], s_mean[3 * threadIdx.x + 1], s_mean[3 * threadIdx.x + 2]);
    const float* m = a.view;  // transformPoint4x3 (auxiliary.h:58-66), contraction pinned like the rest
    p_view.x = __fadd_rn(__fmaf_rn(m[8], p_orig.z, __fmaf_rn(m[0], p_orig.x, __fmul_rn(m[4], p_orig.y))), m[12]);
    p_view.y = __fadd_rn(__fmaf_rn(m[9], p_orig.z, __fmaf_rn(m[1], p_orig.x, __fmul_rn(m[5], p_orig.y))), m[13]);
    p_view.z = __fadd_rn(__fmaf_rn(m[10], p_orig.z, __fmaf_rn(m[2], p_orig.x, __fmul_rn(m[6], p_orig.y))), m[14]);
    vis = !(p_view.z <= 0.2f);
  }
  const bool want_sh = a.colors_precomp == nullptr;
  const int K3 = RAW ? (a.M - 1) * 3 : 0;  // floats per features_rest row
  bool rest_staged = false;
  if (RAW) {
    const int first = blockIdx.x * PRE_THREADS;
    const uint32_t bytes = (uint32_t)(min(PRE_THREADS, a.P - first) * K3 * 4);
    // a partial last block whose byte count is not a multiple of 16 falls back to plain loads
    rest_staged = __syncthreads_or(vis) && a.D > 0 && bytes != 0 && (bytes & 15u) == 0;
    if (rest_staged && threadIdx.x == 0) {
      mbar_arrive_expect_tx(&bar, bytes);
      bulk_g2s(s_rest, a.features_rest + (size_t)first * K3, bytes, &bar);
    }
  }

  // ---- projection (forward.cu:196-200) ----
  float2 p_proj = make_float2(0.f, 0.f);
  if (vis) {
    const float* pm = a.proj;
    float4 p_hom;
    p_hom.x = __fadd_rn(__fmaf_rn(pm[8], p_orig.z, __fmaf_rn(pm[0], p_orig.x, __fmul_rn(pm[4], p_orig.y))), pm[12]);
    p_hom.y = __fadd_rn(__fmaf_rn(pm[9], p_orig.z, __fmaf_rn(pm[1], p_orig.x, __fmul_rn(pm[5], p_orig.y))), pm[13]);
    p_hom.w = __fadd_rn(__fmaf_rn(pm[11], p_orig.z, __fmaf_rn(pm[3], p_orig.x, __fmul_rn(pm[7], p_orig.y))), pm[15]);
    float p_w = __frcp_rn(__fadd_rn(p_hom.w, 0.0000001f));
    p_proj = make_float2(__fmul_rn(p_hom.x, p_w), __fmul_rn(p_hom.y, p_w));
  }
  // The SH row is fetched by the TMA unit NOW, while the thread does the covariance math -- but only for Gaussians
  // whose centre projects onto the screen or its near surroundings (|ndc| <= 1.15): the ~20 % that pass the z test
  // far off-screen would be fetched for nothing (they almost never produce a tile). A Gaussian outside that band that
  // does reach the screen (a huge splat) reads its row with plain loads below: same values, same arithmetic.
  const bool likely = vis && fabsf(p_proj.x) <= 1.15f && fabsf(p_proj.y) <= 1.15f;
  if (BULK_SH) {
    // everybody arrives exactly once on the CTA barrier
    const uint32_t nbytes = (uint32_t)(((a.D + 1) * (a.D + 1) * 12 + 15) & ~15);
    if (likely && want_sh) {
      mbar_arrive_expect_tx(&bar, nbytes);
      bulk_g2s(&sh_rows[threadIdx.x * SH_ROW_WORDS], a.shs + (size_t)idx * a.M * 3, nbytes, &bar);
    } else {
      mbar_arrive(&bar);
    }
  }

  int my_radius_i = 0;
  uint32_t tiles = 0;
  uint32_t depth_key = 0xFFFFFFFFu;
  uint2 rect_min = make_uint2(0, 0), rect_max = make_uint2(0, 0);
  SplatRecord rec;
  bool emit = false;

  if (vis) {

    // ---- 3-D covariance (forward.cu:118-152); the quaternion is used as given ----
    // From here to the conic every operation is pinned with _rn intrinsics to the exact sequence nvcc emits for
    // the reference at sm_90a (decoded from the SASS of the unmodified build, DESIGN.md "Numerics"): every
    // three-term product sum a0*b0 + a1*b1 + a2*b2 is fma(a2,b2, fma(a0,b0, a1*b1)), and the quaternion terms
    // fuse exactly the products noted below. The chain feeds det = a*c - b*b, which cancels catastrophically for
    // elongated splats, so a different (equally valid) contraction changes conics in the 4th digit.
    float cov3D[6];
    if (a.cov3D_precomp != nullptr) {
#pragma unroll
      for (int k = 0; k < 6; k++) cov3D[k] = a.cov3D_precomp[(size_t)idx * 6 + k];
    } else {
      float3 scale = make_float3(s_scale[3 * threadIdx.x], s_scale[3 * threadIdx.x + 1], s_scale[3 * threadIdx.x + 2]);
      float4 q = q_pref;
      if (RAW) {
        scale = make_float3(expf(scale.x), expf(scale.y), expf(scale.z));
        const float n = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);  // F.normalize eps
        q = make_float4(__fdiv_rn(q.x, n), __fdiv_rn(q.y, n), __fdiv_rn(q.z, n), __fdiv_rn(q.w, n));
      }
      const float sx = __fmul_rn(scale.x, a.scale_modifier), sy = __fmul_rn(scale.y, a.scale_modifier),
                  sz = __fmul_rn(scale.z, a.scale_modifier);
      const float r = q.x, x = q.y, y = q.z, z = q.w;
      const float xz = __fmul_rn(x, z), rx = __fmul_rn(r, x), rz = __fmul_rn(r, z);
      const float yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
      const float e02 = __fmaf_rn(r, y, xz);    // x*z + r*y
      const float e20 = __fmaf_rn(-r, y, xz);   // x*z - r*y
      const float e12 = __fmaf_rn(y, z, -rx);   // y*z - r*x
      const float e21 = __fmaf_rn(y, z, rx);    // y*z + r*x
      const float e01 = __fmaf_rn(x, y, -rz);   // x*y - r*z
      const float e10 = __fmaf_rn(x, y, rz);    // x*y + r*z
      const float q00 = __fadd_rn(yy, zz);      // y*y + z*z   (plain add: both squares are shared)
      const float q11 = __fmaf_rn(x, x, zz);    // x*x + z*z
      const float q22 = __fmaf_rn(x, x, yy);    // x*x + y*y
      M3 R;  // glm::mat3(...) lists columns
      R.m[0][0] = __fadd_rn(1.f, -__fadd_rn(q00, q00)); R.m[0][1] = __fadd_rn(e01, e01); R.m[0][2] = __fadd_rn(e02, e02);
      R.m[1][0] = __fadd_rn(e10, e10); R.m[1][1] = __fadd_rn(1.f, -__fadd_rn(q11, q11)); R.m[1][2] = __fadd_rn(e12, e12);
      R.m[2][0] = __fadd_rn(e20, e20); R.m[2][1] = __fadd_rn(e21, e21); R.m[2][2] = __fadd_rn(1.f, -__fadd_rn(q22, q22));
      M3 Mm;  // M = S * R: M[c][r] = s_r * R[c][r] (the zero terms of the GLM product add exact zeros)
#pragma unroll
      for (int c = 0; c < 3; c++) {
        Mm.m[c][0] = __fmul_rn(sx, R.m[c][0]);
        Mm.m[c][1] = __fmul_rn(sy, R.m[c][1]);
        Mm.m[c][2] = __fmul_rn(sz, R.m[c][2]);
      }
      // Sigma = transpose(M) * M: Sigma[c][r] = M[r][0]*M[c][0] + M[r][1]*M[c][1] + M[r][2]*M[c][2]
      auto sig = [&](int c, int r) {
        return __fmaf_rn(Mm.m[r][2], Mm.m[c][2], __fmaf_rn(Mm.m[r][0], Mm.m[c][0], __fmul_rn(Mm.m[r][1], Mm.m[c][1])));
      };
      cov3D[0] = sig(0, 0); cov3D[1] = sig(0, 1); cov3D[2] = sig(0, 2);
      cov3D[3] = sig(1, 1); cov3D[4] = sig(1, 2); cov3D[5] = sig(2, 2);
    }

    // ---- EWA 2-D covariance (forward.cu:74-113) ----
    const float* vm = a.view;
    float3 t = p_view;  // transformPoint4x3(mean, viewmatrix) again in the reference: same value
    const float limx = __fmul_rn(1.3f, a.tan_fovx);
    const float limy = __fmul_rn(1.3f, a.tan_fovy);
    const float txtz = __fdiv_rn(t.x, t.z);
    const float tytz = __fdiv_rn(t.y, t.z);
    t.x = __fmul_rn(fminf(limx, fmaxf(-limx, txtz)), t.z);
    t.y = __fmul_rn(fminf(limy, fmaxf(-limy, tytz)), t.z);
    const float tz2 = __fmul_rn(t.z, t.z);
    const float J00 = __fdiv_rn(a.focal_x, t.z);
    const float J02 = __fdiv_rn(__fmul_rn(-t.x, a.focal_x), tz2);   // -(focal_x * t.x) / (t.z * t.z)
    const float J11 = __fdiv_rn(a.focal_y, t.z);
    const float J12 = __fdiv_rn(__fmul_rn(-t.y, a.focal_y), tz2);
    // T = W * J with J's zero entries: T[0][r] = W[0][r]*J00 + W[2][r]*J02, T[1][r] = W[1][r]*J11 + W[2][r]*J12,
    // W[0] = (v0,v4,v8), W[1] = (v1,v5,v9), W[2] = (v2,v6,v10)
    const float T00 = __fmaf_rn(vm[2], J02, __fmul_rn(vm[0], J00));
    const float T01 = __fmaf_rn(vm[6], J02, __fmul_rn(vm[4], J00));
    const float T02 = __fmaf_rn(vm[10], J02, __fmul_rn(vm[8], J00));
    const float T10 = __fmaf_rn(vm[2], J12, __fmul_rn(vm[1], J11));
    const float T11 = __fmaf_rn(vm[6], J12, __fmul_rn(vm[5], J11));
    const float T12 = __fmaf_rn(vm[10], J12, __fmul_rn(vm[9], J11));
    const float V00 = cov3D[0], V01 = cov3D[1], V02 = cov3D[2], V11 = cov3D[3], V12 = cov3D[4], V22 = cov3D[5];
    // A = transpose(T) * transpose(Vrk): A[c][r] = T[r][0]*V[c][0] + T[r][1]*V[c][1] + T[r][2]*V[c][2]
    const float A00 = __fmaf_rn(T02, V02, __fmaf_rn(T00, V00, __fmul_rn(T01, V01)));
    const float A01 = __fmaf_rn(T12, V02, __fmaf_rn(T10, V00, __fmul_rn(T11, V01)));
    const float A10 = __fmaf_rn(T02, V12, __fmaf_rn(T00, V01, __fmul_rn(T01, V11)));
    const float A11 = __fmaf_rn(T12, V12, __fmaf_rn(T10, V01, __fmul_rn(T11, V11)));
    const float A20 = __fmaf_rn(T02, V22, __fmaf_rn(T00, V02, __fmul_rn(T01, V12)));
    const float A21 = __fmaf_rn(T12, V22, __fmaf_rn(T10, V02, __fmul_rn(T11, V12)));
    // cov = A * T: cov[c][r] = A[0][r]*T[c][0] + A[1][r]*T[c][1] + A[2][r]*T[c][2]; +0.3 low-pass on the diagonal
    const float3 cov2 = make_float3(
        __fadd_rn(__fmaf_rn(T02, A20, __fmaf_rn(T00, A00, __fmul_rn(T01, A10))), 0.3f),
        __fmaf_rn(T02, A21, __fmaf_rn(T00, A01, __fmul_rn(T01, A11))),
        __fadd_rn(__fmaf_rn(T12, A21, __fmaf_rn(T10, A01, __fmul_rn(T11, A11))), 0.3f));

    // ---- conic, radius, tile rectangle (forward.cu:218-237, auxiliary.h:46-56) ----
    float det = __fmaf_rn(cov2.x, cov2.z, -__fmul_rn(cov2.y, cov2.y));
    if (det != 0.0f) {
      float det_inv = __frcp_rn(det);
      float3 conic = make_float3(__fmul_rn(cov2.z, det_inv), __fmul_rn(cov2.y, -det_inv), __fmul_rn(cov2.x, det_inv));
      float mid = __fmul_rn(__fadd_rn(cov2.x, cov2.z), 0.5f);
      float disc = sqrtf(fmaxf(0.1f, __fmaf_rn(mid, mid, -det)));
      float lambda1 = __fadd_rn(mid, disc);
      float lambda2 = __fadd_rn(mid, -disc);
      float my_radius = ceilf(__fmul_rn(3.f, sqrtf(fmaxf(lambda1, lambda2))));
      float2 point_image = make_float2(ndc_to_pix(p_proj.x, a.W), ndc_to_pix(p_proj.y, a.H));
      const int max_radius = (int)my_radius;
      rect_min.x = (unsigned)min(a.gx, max((int)0, (int)((point_image.x - max_radius) / TILE)));
      rect_min.y = (unsigned)min(a.gy, max((int)0, (int)((point_image.y - max_radius) / TILE)));
      rect_max.x = (unsigned)min(a.gx, max((int)0, (int)((point_image.x + max_radius + TILE - 1) / TILE)));
      rect_max.y = (unsigned)min(a.gy, max((int)0, (int)((point_image.y + max_radius + TILE - 1) / TILE)));
      tiles = (rect_max.y - rect_min.y) * (rect_max.x - rect_min.x);
      if (tiles != 0) {
        emit = true;
        my_radius_i = max_radius;
        depth_key = __float_as_uint(p_view.z);
        rec.q0 = make_float4(point_image.x, point_image.y, conic.x, conic.y);
        rec.q1 = make_float4(conic.z, RAW ? sigmoid_act(op_pref) : op_pref, p_view.z, 0.f);
      }
    }
  }

  // ---- colour (forward.cu:20-71) ----
  uint8_t clamp_bits = 0;
  if (BULK_SH) mbar_wait(&bar, 0);  // all rows of this CTA have landed (every thread waits: no divergent exit before)
  if (RAW && rest_staged) mbar_wait(&bar, 0);
  if (emit) {
    float3 rgb;
    if (!want_sh) {
      rgb = make_float3(a.colors_precomp[3 * idx], a.colors_precomp[3 * idx + 1], a.colors_precomp[3 * idx + 2]);
    } else {
      float3 dir = make_float3(__fadd_rn(p_orig.x, -a.campos[0]), __fadd_rn(p_orig.y, -a.campos[1]),
                               __fadd_rn(p_orig.z, -a.campos[2]));
      const float len = __fsqrt_rn(__fmaf_rn(dir.z, dir.z, __fmaf_rn(dir.x, dir.x, __fmul_rn(dir.y, dir.y))));
      dir.x = __fdiv_rn(dir.x, len);
      dir.y = __fdiv_rn(dir.y, len);
      dir.z = __fdiv_rn(dir.z, len);
      float w[16];
      sh_weights(a.D, dir.x, dir.y, dir.z, w);
      float res[3];
      if (BULK_SH && likely) {
        const float* row = &sh_rows[threadIdx.x * SH_ROW_WORDS];
        // pull the row into registers with 128-bit shared loads (row stride 208 B: conflict-free)
        float v[48];
        const int nvec = ((a.D + 1) * (a.D + 1) * 3 + 3) >> 2;
#pragma unroll
        for (int k = 0; k < 12; k++) {
          if (k < nvec) {
            float4 q = *reinterpret_cast<const float4*>(row + 4 * k);
            v[4 * k] = q.x; v[4 * k + 1] = q.y; v[4 * k + 2] = q.z; v[4 * k + 3] = q.w;
          } else {
            v[4 * k] = v[4 * k + 1] = v[4 * k + 2] = v[4 * k + 3] = 0.f;
          }
        }
#pragma unroll
        for (int ch = 0; ch < 3; ch++) res[ch] = sh_channel(a.D, w, [&](int k) { return v[3 * k + ch]; });
      } else if (RAW) {
        const float* dc = a.shs + (size_t)idx * 3;
        const float* rest_g = a.features_rest + (size_t)idx * K3;
        const float* rest_s = s_rest + threadIdx.x * K3;
#pragma unroll
        for (int ch = 0; ch < 3; ch++)
          res[ch] = sh_channel(a.D, w, [&](int k) {
            return k == 0 ? dc[ch] : (rest_staged ? rest_s[3 * (k - 1) + ch] : rest_g[3 * (k - 1) + ch]);
          });
      } else {
        const float* sh = a.shs + (size_t)idx * a.M * 3;
#pragma unroll
        for (int ch = 0; ch < 3; ch++) res[ch] = sh_channel(a.D, w, [&](int k) { return sh[3 * k + ch]; });
      }
      clamp_bits = (res[0] < 0 ? 1 : 0) | (res[1] < 0 ? 2 : 0) | (res[2] < 0 ? 4 : 0);
      rgb = make_float3(fmaxf(res[0], 0.0f), fmaxf(res[1], 0.0f), fmaxf(res[2], 0.0f));
    }
    // q2.w carries the radius and q1.z the view depth (= the depth-sort key bits): a record is self-contained, which
    // is what lets the Gaussian-sharded path exchange the records alone (binning.cu: retouch_kernel)
    rec.q2 = make_float4(rgb.x, rgb.y, rgb.z, __int_as_float(my_radius_i));
    float4* dst = P2P ? &s_rec[threadIdx.x * 3] : reinterpret_cast<float4*>(a.records + idx);
    dst[0] = rec.q0;
    dst[1] = rec.q1;
    dst[2] = rec.q2;
  } else if (live) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);  // radius 0 = culled
    if (P2P) {
      s_rec[threadIdx.x * 3] = z; s_rec[threadIdx.x * 3 + 1] = z; s_rec[threadIdx.x * 3 + 2] = z;
    } else {
      reinterpret_cast<float4*>(a.records + idx)[2] = z;
    }
  }
  if (P2P) {
    // compute -> collective in one kernel: the block of records goes straight from shared memory to every rank's
    // records array (TMA bulk stores over NVLink peer mappings; one elected thread per destination)
    fence_proxy_async_smem();
    __syncthreads();
    const int first = blockIdx.x * PRE_THREADS;
    const uint32_t bytes = (uint32_t)(min(PRE_THREADS, a.P - first) * (int)sizeof(SplatRecord));
    if ((int)threadIdx.x < a.npeers) {
      bulk_s2g(a.peer_records[threadIdx.x] + first, s_rec, bytes);
      bulk_commit();
      bulk_wait_read0();  // shared memory must stay intact until the TMA unit has read it
    }
  }
  if (a.tile_diff != nullptr) {
    if (emit) add_tile_rect(a.tile_diff, a.gx, a.gy, a.diff_copies, (uint32_t)idx, rect_min.x, rect_min.y, rect_max.x, rect_max.y);
  }
  if (live) {
    a.radii[idx] = my_radius_i;
    a.tiles_touched[idx] = tiles;
    a.clamped[idx] = clamp_bits;
    a.depth_keys[idx] = depth_key;
    a.ident[idx] = (uint32_t)idx;
  }
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
                          const float* features_rest, bool count_tiles) {
  PreArgs a;
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
      preprocess_fwd_kernel<false, true, true><<<grid, PRE_THREADS, 0, st>>>(a);
    else
      preprocess_fwd_kernel<false, false, true><<<grid, PRE_THREADS, 0, st>>>(a);
  } else if (npeers > 0) {
    if (bulk)
      preprocess_fwd_kernel<true, true><<<grid, PRE_THREADS, 0, st>>>(a);
    else
      preprocess_fwd_kernel<false, true><<<grid, PRE_THREADS, 0, st>>>(a);
  } else if (bulk)
    preprocess_fwd_kernel<true><<<grid, PRE_THREADS, 0, st>>>(a);
  else
    preprocess_fwd_kernel<false><<<grid, PRE_THREADS, 0, st>>>(a);
  g_launches++;
  return check_launch("preprocess_fwd", s.debug != 0, st);
}

int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present, cudaStream_t st) {
  mark_visible_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, viewmatrix, present);
  g_launches++;
  return check_launch("mark_visible", false, st);
}

}  // namespace gsr
