// ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// CPU restatement of the differentiable 3D-Gaussian-splatting rasterizer that
// GaussianEditor installs (gaussiansplatting/submodules/diff-gaussian-rasterization,
// "DGR/" below; all path:line citations are relative to /root/reference/).
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
// legs may load this file's shared object; the product path (gaussianeditor_b200/)
// never does.
//
// PARITY PINNING: the reference ships no tests, golden vectors or CPU path for this
// code (SURVEY.md section 4), so this restatement is pinned two ways instead:
//   (1) against the reference's own CUDA sources compiled unmodified into
//       oracle/_ref/libdgr_ref.so and run on the GPU box (tests/test_parity_gpu.py:
//       test_oracle_matches_reference_cuda and the *_matches_reference_cuda tests),
//   (2) against closed-form known-answer cases and fp64 finite differences
//       (tests/test_oracle_kat.py), and against the reference's independent PyTorch
//       helpers eval_sh / build_scaling_rotation re-stated in the tests.
//
// Every function is templated on the arithmetic type: F=float follows the reference
// operation by operation (expression order as written in the CUDA source; no FMA
// contraction -- build with -ffp-contract=off), F=double is the gradient ground truth.
//
// Build: see oracle/Makefile (g++ -O2 -fopenmp -ffp-contract=off -shared -fPIC).

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

constexpr int BLOCK_X = 16;  // DGR/cuda_rasterizer/config.h:16-17
constexpr int BLOCK_Y = 16;

// DGR/cuda_rasterizer/auxiliary.h:22-39
const float SH_C0 = 0.28209479177387814f;
const float SH_C1 = 0.4886025119029199f;
const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                        -1.0925484305920792f, 0.5462742152960396f};
const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                        0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                        -0.5900435899266435f};

template <typename F> struct V3 { F x, y, z; };

// Column-major 3x3 in GLM's convention: m[c][r].
template <typename F> struct M3 {
  F m[3][3];
};

// GLM mat3*mat3, DGR/third_party/glm/glm/detail/type_mat3x3.inl:486-518:
// Result[c][r] = A[0][r]*B[c][0] + A[1][r]*B[c][1] + A[2][r]*B[c][2]
template <typename F> M3<F> mul(const M3<F>& A, const M3<F>& B) {
  M3<F> R;
  for (int c = 0; c < 3; c++)
    for (int r = 0; r < 3; r++)
      R.m[c][r] = A.m[0][r] * B.m[c][0] + A.m[1][r] * B.m[c][1] + A.m[2][r] * B.m[c][2];
  return R;
}
template <typename F> M3<F> transpose(const M3<F>& A) {
  M3<F> R;
  for (int c = 0; c < 3; c++)
    for (int r = 0; r < 3; r++) R.m[c][r] = A.m[r][c];
  return R;
}

// auxiliary.h:41-44 -- NOTE the literals are double, so the reference evaluates ndc2Pix in
// fp64 and rounds once on return; both variants here do the same.
template <typename F> F ndc2Pix(F v, int S) { return (F)((((double)v + 1.0) * S - 1.0) * 0.5); }

// float -> int as the GPU converts (cvt.rzi.s32.f32): truncation toward zero, saturating at INT_MIN / INT_MAX, NaN -> 0.
// A plain (int) cast of an out-of-range or NaN value is undefined in C++ and gives INT_MIN on x86; the reference's CUDA
// build sees a saturated radius (a splat over the whole grid) where such a cast would see a negative one.
template <typename F> int to_int_rz(F v) {
  if (std::isnan(v)) return 0;
  if (v >= (F)2147483648.0) return INT32_MAX;
  if (v <= (F)-2147483648.0) return INT32_MIN;
  return (int)v;
}

// auxiliary.h:46-56 (float -> int conversions truncate toward zero and saturate, to_int_rz)
template <typename F>
void getRect(F px, F py, int max_radius, int gx, int gy, uint32_t* rmin, uint32_t* rmax) {
  rmin[0] = (uint32_t)std::min(gx, std::max(0, to_int_rz<F>((px - max_radius) / BLOCK_X)));
  rmin[1] = (uint32_t)std::min(gy, std::max(0, to_int_rz<F>((py - max_radius) / BLOCK_Y)));
  rmax[0] = (uint32_t)std::min(gx, std::max(0, to_int_rz<F>((px + max_radius + BLOCK_X - 1) / BLOCK_X)));
  rmax[1] = (uint32_t)std::min(gy, std::max(0, to_int_rz<F>((py + max_radius + BLOCK_Y - 1) / BLOCK_Y)));
}

// auxiliary.h:58-77
template <typename F> V3<F> transformPoint4x3(V3<F> p, const float* m) {
  return {(F)m[0] * p.x + (F)m[4] * p.y + (F)m[8] * p.z + (F)m[12],
          (F)m[1] * p.x + (F)m[5] * p.y + (F)m[9] * p.z + (F)m[13],
          (F)m[2] * p.x + (F)m[6] * p.y + (F)m[10] * p.z + (F)m[14]};
}
template <typename F> void transformPoint4x4(V3<F> p, const float* m, F out[4]) {
  out[0] = (F)m[0] * p.x + (F)m[4] * p.y + (F)m[8] * p.z + (F)m[12];
  out[1] = (F)m[1] * p.x + (F)m[5] * p.y + (F)m[9] * p.z + (F)m[13];
  out[2] = (F)m[2] * p.x + (F)m[6] * p.y + (F)m[10] * p.z + (F)m[14];
  out[3] = (F)m[3] * p.x + (F)m[7] * p.y + (F)m[11] * p.z + (F)m[15];
}

// forward.cu:118-152 computeCov3D (quaternion NOT normalised, :127)
template <typename F>
void computeCov3D(const float* scale, F mod, const float* rot, F* cov3D) {
  M3<F> S = {};
  S.m[0][0] = mod * (F)scale[0];
  S.m[1][1] = mod * (F)scale[1];
  S.m[2][2] = mod * (F)scale[2];
  F r = rot[0], x = rot[1], y = rot[2], z = rot[3];
  // glm::mat3(a,b,c, d,e,f, g,h,i) lists COLUMNS: m[0]=(a,b,c) ...
  M3<F> R;
  R.m[0][0] = (F)1 - (F)2 * (y * y + z * z); R.m[0][1] = (F)2 * (x * y - r * z); R.m[0][2] = (F)2 * (x * z + r * y);
  R.m[1][0] = (F)2 * (x * y + r * z); R.m[1][1] = (F)1 - (F)2 * (x * x + z * z); R.m[1][2] = (F)2 * (y * z - r * x);
  R.m[2][0] = (F)2 * (x * z - r * y); R.m[2][1] = (F)2 * (y * z + r * x); R.m[2][2] = (F)1 - (F)2 * (x * x + y * y);
  M3<F> M = mul(S, R);
  M3<F> Sigma = mul(transpose(M), M);
  cov3D[0] = Sigma.m[0][0]; cov3D[1] = Sigma.m[0][1]; cov3D[2] = Sigma.m[0][2];
  cov3D[3] = Sigma.m[1][1]; cov3D[4] = Sigma.m[1][2]; cov3D[5] = Sigma.m[2][2];
}

// Shared by forward.cu:74-113 (computeCov2D) and backward.cu:166-199 (its recomputation)
template <typename F> struct Cov2DCtx {
  V3<F> t;  // clamped view-space mean
  F txtz, tytz, limx, limy;
  M3<F> J, W, T, Vrk, cov;
};
template <typename F>
void cov2D_setup(V3<F> mean, F focal_x, F focal_y, F tan_fovx, F tan_fovy, const F* cov3D,
                 const float* view, Cov2DCtx<F>& c) {
  c.t = transformPoint4x3(mean, view);
  c.limx = (F)1.3f * tan_fovx;
  c.limy = (F)1.3f * tan_fovy;
  c.txtz = c.t.x / c.t.z;
  c.tytz = c.t.y / c.t.z;
  c.t.x = std::fmin(c.limx, std::fmax(-c.limx, c.txtz)) * c.t.z;
  c.t.y = std::fmin(c.limy, std::fmax(-c.limy, c.tytz)) * c.t.z;
  M3<F>& J = c.J;
  J.m[0][0] = focal_x / c.t.z; J.m[0][1] = 0; J.m[0][2] = -(focal_x * c.t.x) / (c.t.z * c.t.z);
  J.m[1][0] = 0; J.m[1][1] = focal_y / c.t.z; J.m[1][2] = -(focal_y * c.t.y) / (c.t.z * c.t.z);
  J.m[2][0] = 0; J.m[2][1] = 0; J.m[2][2] = 0;
  M3<F>& W = c.W;
  W.m[0][0] = view[0]; W.m[0][1] = view[4]; W.m[0][2] = view[8];
  W.m[1][0] = view[1]; W.m[1][1] = view[5]; W.m[1][2] = view[9];
  W.m[2][0] = view[2]; W.m[2][1] = view[6]; W.m[2][2] = view[10];
  c.T = mul(W, J);
  M3<F>& V = c.Vrk;
  V.m[0][0] = cov3D[0]; V.m[0][1] = cov3D[1]; V.m[0][2] = cov3D[2];
  V.m[1][0] = cov3D[1]; V.m[1][1] = cov3D[3]; V.m[1][2] = cov3D[4];
  V.m[2][0] = cov3D[2]; V.m[2][1] = cov3D[4]; V.m[2][2] = cov3D[5];
  c.cov = mul(mul(transpose(c.T), transpose(V)), c.T);
  c.cov.m[0][0] += (F)0.3f;
  c.cov.m[1][1] += (F)0.3f;
}

// SH basis for the direction (x,y,z); forward.cu:30-61 and backward.cu:47-97
template <typename F> void sh_basis(int deg, F x, F y, F z, F* b) {
  b[0] = SH_C0;
  if (deg > 0) {
    b[1] = -(F)SH_C1 * y; b[2] = (F)SH_C1 * z; b[3] = -(F)SH_C1 * x;
    if (deg > 1) {
      F xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
      b[4] = (F)SH_C2[0] * xy; b[5] = (F)SH_C2[1] * yz; b[6] = (F)SH_C2[2] * ((F)2 * zz - xx - yy);
      b[7] = (F)SH_C2[3] * xz; b[8] = (F)SH_C2[4] * (xx - yy);
      if (deg > 2) {
        b[9] = (F)SH_C3[0] * y * ((F)3 * xx - yy);
        b[10] = (F)SH_C3[1] * xy * z;
        b[11] = (F)SH_C3[2] * y * ((F)4 * zz - xx - yy);
        b[12] = (F)SH_C3[3] * z * ((F)2 * zz - (F)3 * xx - (F)3 * yy);
        b[13] = (F)SH_C3[4] * x * ((F)4 * zz - xx - yy);
        b[14] = (F)SH_C3[5] * z * (xx - yy);
        b[15] = (F)SH_C3[6] * x * (xx - (F)3 * yy);
      }
    }
  }
}

struct Params {
  int P, D, M, W, H;
  float tan_fovx, tan_fovy, scale_modifier;
  const float* bg;
  const float* means3D;
  const float* shs;            // [P,M,3] or null
  const float* colors_precomp; // [P,3] or null
  const float* opacities;
  const float* scales;         // or null
  const float* rotations;      // or null
  const float* cov3D_precomp;  // or null
  const float* viewmatrix;
  const float* projmatrix;
  const float* campos;
};

template <typename F> struct Geom {
  std::vector<F> depths, means2D, cov3D, conic_opacity, rgb;
  std::vector<uint8_t> clamped;
  std::vector<int32_t> radii;
  std::vector<uint32_t> tiles_touched, point_offsets;
};

// forward.cu:155-256 preprocessCUDA
template <typename F> void preprocess(const Params& p, Geom<F>& g) {
  const int P = p.P;
  g.depths.assign(P, 0); g.means2D.assign(2 * (size_t)P, 0); g.cov3D.assign(6 * (size_t)P, 0);
  g.conic_opacity.assign(4 * (size_t)P, 0); g.rgb.assign(3 * (size_t)P, 0);
  g.clamped.assign(3 * (size_t)P, 0); g.radii.assign(P, 0); g.tiles_touched.assign(P, 0);
  const F focal_y = (F)p.H / ((F)2.0f * (F)p.tan_fovy);  // rasterizer_impl.cu:190-191
  const F focal_x = (F)p.W / ((F)2.0f * (F)p.tan_fovx);
  const int gx = (p.W + BLOCK_X - 1) / BLOCK_X, gy = (p.H + BLOCK_Y - 1) / BLOCK_Y;
#pragma omp parallel for schedule(static)
  for (int idx = 0; idx < P; idx++) {
    V3<F> po = {(F)p.means3D[3 * idx], (F)p.means3D[3 * idx + 1], (F)p.means3D[3 * idx + 2]};
    V3<F> p_view = transformPoint4x3(po, p.viewmatrix);
    if (p_view.z <= (F)0.2f) continue;  // auxiliary.h:154
    F ph[4];
    transformPoint4x4(po, p.projmatrix, ph);
    F p_w = (F)1.0f / (ph[3] + (F)0.0000001f);
    F projx = ph[0] * p_w, projy = ph[1] * p_w;
    F cov3D_local[6];
    const F* cov3D;
    if (p.cov3D_precomp) {
      for (int k = 0; k < 6; k++) cov3D_local[k] = p.cov3D_precomp[6 * (size_t)idx + k];
    } else {
      computeCov3D<F>(p.scales + 3 * (size_t)idx, (F)p.scale_modifier, p.rotations + 4 * (size_t)idx, cov3D_local);
    }
    for (int k = 0; k < 6; k++) g.cov3D[6 * (size_t)idx + k] = cov3D_local[k];
    cov3D = cov3D_local;
    Cov2DCtx<F> c;
    cov2D_setup<F>(po, focal_x, focal_y, (F)p.tan_fovx, (F)p.tan_fovy, cov3D, p.viewmatrix, c);
    F cx = c.cov.m[0][0], cy = c.cov.m[0][1], cz = c.cov.m[1][1];
    F det = cx * cz - cy * cy;
    if (det == (F)0) continue;
    F det_inv = (F)1 / det;
    F conic[3] = {cz * det_inv, -cy * det_inv, cx * det_inv};
    F mid = (F)0.5f * (cx + cz);
    F lambda1 = mid + std::sqrt(std::fmax((F)0.1f, mid * mid - det));
    F lambda2 = mid - std::sqrt(std::fmax((F)0.1f, mid * mid - det));
    F my_radius = std::ceil((F)3 * std::sqrt(std::fmax(lambda1, lambda2)));
    F pix = ndc2Pix<F>(projx, p.W);
    F piy = ndc2Pix<F>(projy, p.H);
    uint32_t rmin[2], rmax[2];
    getRect<F>(pix, piy, to_int_rz<F>(my_radius), gx, gy, rmin, rmax);
    if ((rmax[0] - rmin[0]) * (rmax[1] - rmin[1]) == 0) continue;
    if (!p.colors_precomp) {
      // forward.cu:20-71 computeColorFromSH
      F dx = po.x - (F)p.campos[0], dy = po.y - (F)p.campos[1], dz = po.z - (F)p.campos[2];
      F len = std::sqrt(dx * dx + dy * dy + dz * dz);
      dx = dx / len; dy = dy / len; dz = dz / len;
      F b[16];
      sh_basis<F>(p.D, dx, dy, dz, b);
      const float* sh = p.shs + (size_t)idx * p.M * 3;
      int nb = (p.D + 1) * (p.D + 1);
      for (int ch = 0; ch < 3; ch++) {
        F res = 0;
        // summation order as in the source: running sum over k
        for (int k = 0; k < nb; k++) res = (k == 0) ? b[0] * (F)sh[ch] : res + b[k] * (F)sh[3 * k + ch];
        res += (F)0.5f;
        g.clamped[3 * (size_t)idx + ch] = res < 0;
        g.rgb[3 * (size_t)idx + ch] = std::fmax(res, (F)0);
      }
    }
    g.depths[idx] = p_view.z;
    g.radii[idx] = to_int_rz<F>(my_radius);
    g.means2D[2 * (size_t)idx] = pix; g.means2D[2 * (size_t)idx + 1] = piy;
    g.conic_opacity[4 * (size_t)idx + 0] = conic[0]; g.conic_opacity[4 * (size_t)idx + 1] = conic[1];
    g.conic_opacity[4 * (size_t)idx + 2] = conic[2]; g.conic_opacity[4 * (size_t)idx + 3] = p.opacities[idx];
    g.tiles_touched[idx] = (rmax[1] - rmin[1]) * (rmax[0] - rmin[0]);
  }
}

// rasterizer_impl.cu:36-49
uint32_t getHigherMsb(uint32_t n) {
  uint32_t msb = sizeof(n) * 4, step = msb;
  while (step > 1) {
    step /= 2;
    if (n >> msb) msb += step; else msb -= step;
  }
  if (n >> msb) msb++;
  return msb;
}

struct Binning {
  std::vector<uint64_t> keys;       // sorted
  std::vector<uint32_t> point_list; // sorted
  std::vector<uint32_t> ranges;     // [Ntile,2]
  int64_t R = 0;
};

// rasterizer_impl.cu:227-270: scan, duplicateWithKeys (:67-100), stable radix sort on the low
// 32+bit bits (:253-261), identifyTileRanges (:105-125)
template <typename F> void bin(const Params& p, Geom<F>& g, Binning& b) {
  const int P = p.P;
  const int gx = (p.W + BLOCK_X - 1) / BLOCK_X, gy = (p.H + BLOCK_Y - 1) / BLOCK_Y;
  g.point_offsets.assign(P, 0);
  uint32_t run = 0;
  for (int i = 0; i < P; i++) { run += g.tiles_touched[i]; g.point_offsets[i] = run; }
  b.R = P ? g.point_offsets[P - 1] : 0;
  std::vector<uint64_t> keys_unsorted(b.R);
  std::vector<uint32_t> vals_unsorted(b.R);
#pragma omp parallel for schedule(dynamic, 1024)
  for (int idx = 0; idx < P; idx++) {
    if (g.radii[idx] > 0) {
      uint32_t off = idx == 0 ? 0 : g.point_offsets[idx - 1];
      uint32_t rmin[2], rmax[2];
      getRect<F>(g.means2D[2 * (size_t)idx], g.means2D[2 * (size_t)idx + 1], g.radii[idx], gx, gy, rmin, rmax);
      float depth_f = (float)g.depths[idx];  // keys always carry the fp32 depth bits
      uint32_t dbits;
      std::memcpy(&dbits, &depth_f, 4);
      for (uint32_t y = rmin[1]; y < rmax[1]; y++)
        for (uint32_t x = rmin[0]; x < rmax[0]; x++) {
          uint64_t key = (uint64_t)(y * gx + x);
          key <<= 32;
          key |= dbits;
          keys_unsorted[off] = key;
          vals_unsorted[off] = idx;
          off++;
        }
    }
  }
  int bit = getHigherMsb((uint32_t)(gx * gy));
  uint64_t mask = (32 + bit >= 64) ? ~0ull : ((1ull << (32 + bit)) - 1);
  std::vector<uint32_t> order(b.R);
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t c) {
    return (keys_unsorted[a] & mask) < (keys_unsorted[c] & mask);
  });
  b.keys.resize(b.R);
  b.point_list.resize(b.R);
  for (int64_t i = 0; i < b.R; i++) { b.keys[i] = keys_unsorted[order[i]]; b.point_list[i] = vals_unsorted[order[i]]; }
  b.ranges.assign(2 * (size_t)gx * gy, 0);
  for (int64_t idx = 0; idx < b.R; idx++) {
    uint32_t cur = (uint32_t)(b.keys[idx] >> 32);
    if (idx == 0) b.ranges[2 * cur] = 0;
    else {
      uint32_t prev = (uint32_t)(b.keys[idx - 1] >> 32);
      if (cur != prev) { b.ranges[2 * prev + 1] = (uint32_t)idx; b.ranges[2 * cur] = (uint32_t)idx; }
    }
    if (idx == b.R - 1) b.ranges[2 * cur + 1] = (uint32_t)b.R;
  }
}

template <typename F> struct Image {
  std::vector<F> out_color, out_depth, final_T;
  std::vector<uint32_t> n_contrib;
};

// Counters for workload descriptors (pairs evaluated / hits), not part of the reference.
struct Stats { int64_t pairs = 0, hits = 0; };

// forward.cu:261-379 renderCUDA. A pixel's walk is independent of its neighbours; the
// block-level early exit (:312-314) only stops work nobody needs.
template <typename F>
void render_forward(const Params& p, const Geom<F>& g, const Binning& b, Image<F>& im, Stats* st) {
  const int W = p.W, H = p.H;
  const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
  im.out_color.assign(3 * (size_t)W * H, 0); im.out_depth.assign((size_t)W * H, 0);
  im.final_T.assign((size_t)W * H, 0); im.n_contrib.assign((size_t)W * H, 0);
  const F* feat_own = g.rgb.data();
  int64_t pairs = 0, hits = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : pairs, hits)
  for (int tile = 0; tile < gx * gy; tile++) {
    int ty = tile / gx, tx = tile % gx;
    uint32_t r0 = b.ranges[2 * tile], r1 = b.ranges[2 * tile + 1];
    for (int py = ty * BLOCK_Y; py < std::min((ty + 1) * BLOCK_Y, H); py++)
      for (int px = tx * BLOCK_X; px < std::min((tx + 1) * BLOCK_X, W); px++) {
        F T = 1, C[3] = {0, 0, 0}, Dp = 0;
        uint32_t contributor = 0, last = 0;
        F pixx = (F)px, pixy = (F)py;
        for (uint32_t k = r0; k < r1; k++) {
          contributor++;
          uint32_t id = b.point_list[k];
          F dx = g.means2D[2 * (size_t)id] - pixx, dy = g.means2D[2 * (size_t)id + 1] - pixy;
          const F* co = &g.conic_opacity[4 * (size_t)id];
          F power = (F)-0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
          pairs++;
          if (power > 0) continue;
          F alpha = std::fmin((F)0.99f, co[3] * std::exp(power));
          if (alpha < (F)(1.0f / 255.0f)) continue;
          F test_T = T * (1 - alpha);
          if (test_T < (F)0.0001f) break;  // done = true
          hits++;
          for (int ch = 0; ch < 3; ch++) {
            F f = p.colors_precomp ? (F)p.colors_precomp[3 * (size_t)id + ch] : feat_own[3 * (size_t)id + ch];
            C[ch] += f * alpha * T;
          }
          Dp += g.depths[id] * alpha * T;
          T = test_T;
          last = contributor;
        }
        size_t pix_id = (size_t)W * py + px;
        im.final_T[pix_id] = T;
        im.n_contrib[pix_id] = last;
        for (int ch = 0; ch < 3; ch++) im.out_color[(size_t)ch * H * W + pix_id] = C[ch] + T * (F)p.bg[ch];
        im.out_depth[pix_id] = Dp;
      }
  }
  if (st) { st->pairs = pairs; st->hits = hits; }
}

template <typename F> struct Grads {
  std::vector<F> dmean2D, dconic, dopacity, dcolor, dmean3D, dcov3D, dsh, dscale, drot;
};

// backward.cu:399-557 renderCUDA (bwd). Per-Gaussian sums are accumulated per tile and
// merged under a critical section (the reference uses float atomics; order differs).
template <typename F>
void render_backward(const Params& p, const Geom<F>& g, const Binning& b, const Image<F>& im,
                     const float* dL_dpix, Grads<F>& gr) {
  const int W = p.W, H = p.H, P = p.P;
  const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
  gr.dmean2D.assign(3 * (size_t)P, 0); gr.dconic.assign(4 * (size_t)P, 0);
  gr.dopacity.assign(P, 0); gr.dcolor.assign(3 * (size_t)P, 0);
  const F ddelx_dx = (F)0.5 * W, ddely_dy = (F)0.5 * H;
  const F* feat_own = g.rgb.data();
#pragma omp parallel
  {
    std::vector<F> acc;  // [n,9] per tile
#pragma omp for schedule(dynamic, 1)
    for (int tile = 0; tile < gx * gy; tile++) {
      int ty = tile / gx, tx = tile % gx;
      uint32_t r0 = b.ranges[2 * tile], r1 = b.ranges[2 * tile + 1];
      uint32_t n = r1 - r0;
      if (n == 0) continue;
      acc.assign(9 * (size_t)n, 0);
      for (int py = ty * BLOCK_Y; py < std::min((ty + 1) * BLOCK_Y, H); py++)
        for (int px = tx * BLOCK_X; px < std::min((tx + 1) * BLOCK_X, W); px++) {
          size_t pix_id = (size_t)W * py + px;
          const F T_final = im.final_T[pix_id];
          F T = T_final;
          uint32_t contributor = n;
          const uint32_t last_contributor = im.n_contrib[pix_id];
          F accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, last_alpha = 0, dpx[3];
          for (int ch = 0; ch < 3; ch++) dpx[ch] = dL_dpix[(size_t)ch * H * W + pix_id];
          F pixx = (F)px, pixy = (F)py;
          for (uint32_t j = 0; j < n; j++) {
            uint32_t k = r1 - 1 - j;
            contributor--;
            if (contributor >= last_contributor) continue;
            uint32_t id = b.point_list[k];
            F dx = g.means2D[2 * (size_t)id] - pixx, dy = g.means2D[2 * (size_t)id + 1] - pixy;
            const F* co = &g.conic_opacity[4 * (size_t)id];
            F power = (F)-0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
            if (power > 0) continue;
            F G = std::exp(power);
            F alpha = std::fmin((F)0.99f, co[3] * G);
            if (alpha < (F)(1.0f / 255.0f)) continue;
            T = T / ((F)1 - alpha);
            F dchannel_dcolor = alpha * T;
            F dL_dalpha = 0;
            F* a = &acc[9 * (size_t)(k - r0)];
            for (int ch = 0; ch < 3; ch++) {
              F c = p.colors_precomp ? (F)p.colors_precomp[3 * (size_t)id + ch] : feat_own[3 * (size_t)id + ch];
              accum_rec[ch] = last_alpha * last_color[ch] + ((F)1 - last_alpha) * accum_rec[ch];
              last_color[ch] = c;
              dL_dalpha += (c - accum_rec[ch]) * dpx[ch];
              a[ch] += dchannel_dcolor * dpx[ch];
            }
            dL_dalpha *= T;
            last_alpha = alpha;
            F bg_dot = 0;
            for (int ch = 0; ch < 3; ch++) bg_dot += (F)p.bg[ch] * dpx[ch];
            dL_dalpha += (-T_final / ((F)1 - alpha)) * bg_dot;
            F dL_dG = co[3] * dL_dalpha;
            F gdx = G * dx, gdy = G * dy;
            F dG_ddelx = -gdx * co[0] - gdy * co[1];
            F dG_ddely = -gdy * co[2] - gdx * co[1];
            a[3] += dL_dG * dG_ddelx * ddelx_dx;
            a[4] += dL_dG * dG_ddely * ddely_dy;
            a[5] += (F)-0.5f * gdx * dx * dL_dG;
            a[6] += (F)-0.5f * gdx * dy * dL_dG;
            a[7] += (F)-0.5f * gdy * dy * dL_dG;
            a[8] += G * dL_dalpha;
          }
        }
#pragma omp critical
      {
        for (uint32_t k = 0; k < n; k++) {
          uint32_t id = b.point_list[r0 + k];
          const F* a = &acc[9 * (size_t)k];
          gr.dcolor[3 * (size_t)id] += a[0]; gr.dcolor[3 * (size_t)id + 1] += a[1]; gr.dcolor[3 * (size_t)id + 2] += a[2];
          gr.dmean2D[3 * (size_t)id] += a[3]; gr.dmean2D[3 * (size_t)id + 1] += a[4];
          gr.dconic[4 * (size_t)id] += a[5]; gr.dconic[4 * (size_t)id + 1] += a[6]; gr.dconic[4 * (size_t)id + 3] += a[7];
          gr.dopacity[id] += a[8];
        }
      }
    }
  }
}

// backward.cu:144-274 computeCov2DCUDA, then :346-396 preprocessCUDA (bwd) with
// :20-139 (SH backward) and :278-341 (cov3D backward); order per rasterizer_impl.cu:320-340.
template <typename F>
void preprocess_backward(const Params& p, const Geom<F>& g, Grads<F>& gr) {
  const int P = p.P, M = p.M;
  gr.dmean3D.assign(3 * (size_t)P, 0); gr.dcov3D.assign(6 * (size_t)P, 0);
  gr.dsh.assign(3 * (size_t)P * std::max(M, 0), 0); gr.dscale.assign(3 * (size_t)P, 0); gr.drot.assign(4 * (size_t)P, 0);
  const F h_y = (F)p.H / ((F)2.0f * (F)p.tan_fovy);
  const F h_x = (F)p.W / ((F)2.0f * (F)p.tan_fovx);
  const float* view = p.viewmatrix;
  const float* proj = p.projmatrix;
#pragma omp parallel for schedule(static)
  for (int idx = 0; idx < P; idx++) {
    if (!(g.radii[idx] > 0)) continue;
    V3<F> mean = {(F)p.means3D[3 * idx], (F)p.means3D[3 * idx + 1], (F)p.means3D[3 * idx + 2]};
    // ---- computeCov2DCUDA ----
    {
      const F* cov3D = &g.cov3D[6 * (size_t)idx];
      F dcx = gr.dconic[4 * (size_t)idx], dcy = gr.dconic[4 * (size_t)idx + 1], dcz = gr.dconic[4 * (size_t)idx + 3];
      Cov2DCtx<F> c;
      cov2D_setup<F>(mean, h_x, h_y, (F)p.tan_fovx, (F)p.tan_fovy, cov3D, view, c);
      const F x_grad_mul = (c.txtz < -c.limx || c.txtz > c.limx) ? 0 : 1;
      const F y_grad_mul = (c.tytz < -c.limy || c.tytz > c.limy) ? 0 : 1;
      const M3<F>& T = c.T; const M3<F>& Vrk = c.Vrk; const M3<F>& Wm = c.W;
      F a = c.cov.m[0][0], b = c.cov.m[0][1], cc = c.cov.m[1][1];
      F denom = a * cc - b * b;
      F dL_da = 0, dL_db = 0, dL_dc = 0;
      F denom2inv = (F)1 / ((denom * denom) + (F)0.0000001f);
      F* dcov = &gr.dcov3D[6 * (size_t)idx];
      if (denom2inv != 0) {
        dL_da = denom2inv * (-cc * cc * dcx + 2 * b * cc * dcy + (denom - a * cc) * dcz);
        dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * cc) * dcx);
        dL_db = denom2inv * 2 * (b * cc * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
        dcov[0] = (T.m[0][0] * T.m[0][0] * dL_da + T.m[0][0] * T.m[1][0] * dL_db + T.m[1][0] * T.m[1][0] * dL_dc);
        dcov[3] = (T.m[0][1] * T.m[0][1] * dL_da + T.m[0][1] * T.m[1][1] * dL_db + T.m[1][1] * T.m[1][1] * dL_dc);
        dcov[5] = (T.m[0][2] * T.m[0][2] * dL_da + T.m[0][2] * T.m[1][2] * dL_db + T.m[1][2] * T.m[1][2] * dL_dc);
        dcov[1] = 2 * T.m[0][0] * T.m[0][1] * dL_da + (T.m[0][0] * T.m[1][1] + T.m[0][1] * T.m[1][0]) * dL_db + 2 * T.m[1][0] * T.m[1][1] * dL_dc;
        dcov[2] = 2 * T.m[0][0] * T.m[0][2] * dL_da + (T.m[0][0] * T.m[1][2] + T.m[0][2] * T.m[1][0]) * dL_db + 2 * T.m[1][0] * T.m[1][2] * dL_dc;
        dcov[4] = 2 * T.m[0][2] * T.m[0][1] * dL_da + (T.m[0][1] * T.m[1][2] + T.m[0][2] * T.m[1][1]) * dL_db + 2 * T.m[1][1] * T.m[1][2] * dL_dc;
      } else {
        for (int i = 0; i < 6; i++) dcov[i] = 0;
      }
      F dL_dT00 = 2 * (T.m[0][0] * Vrk.m[0][0] + T.m[0][1] * Vrk.m[0][1] + T.m[0][2] * Vrk.m[0][2]) * dL_da +
                  (T.m[1][0] * Vrk.m[0][0] + T.m[1][1] * Vrk.m[0][1] + T.m[1][2] * Vrk.m[0][2]) * dL_db;
      F dL_dT01 = 2 * (T.m[0][0] * Vrk.m[1][0] + T.m[0][1] * Vrk.m[1][1] + T.m[0][2] * Vrk.m[1][2]) * dL_da +
                  (T.m[1][0] * Vrk.m[1][0] + T.m[1][1] * Vrk.m[1][1] + T.m[1][2] * Vrk.m[1][2]) * dL_db;
      F dL_dT02 = 2 * (T.m[0][0] * Vrk.m[2][0] + T.m[0][1] * Vrk.m[2][1] + T.m[0][2] * Vrk.m[2][2]) * dL_da +
                  (T.m[1][0] * Vrk.m[2][0] + T.m[1][1] * Vrk.m[2][1] + T.m[1][2] * Vrk.m[2][2]) * dL_db;
      F dL_dT10 = 2 * (T.m[1][0] * Vrk.m[0][0] + T.m[1][1] * Vrk.m[0][1] + T.m[1][2] * Vrk.m[0][2]) * dL_dc +
                  (T.m[0][0] * Vrk.m[0][0] + T.m[0][1] * Vrk.m[0][1] + T.m[0][2] * Vrk.m[0][2]) * dL_db;
      F dL_dT11 = 2 * (T.m[1][0] * Vrk.m[1][0] + T.m[1][1] * Vrk.m[1][1] + T.m[1][2] * Vrk.m[1][2]) * dL_dc +
                  (T.m[0][0] * Vrk.m[1][0] + T.m[0][1] * Vrk.m[1][1] + T.m[0][2] * Vrk.m[1][2]) * dL_db;
      F dL_dT12 = 2 * (T.m[1][0] * Vrk.m[2][0] + T.m[1][1] * Vrk.m[2][1] + T.m[1][2] * Vrk.m[2][2]) * dL_dc +
                  (T.m[0][0] * Vrk.m[2][0] + T.m[0][1] * Vrk.m[2][1] + T.m[0][2] * Vrk.m[2][2]) * dL_db;
      F dL_dJ00 = Wm.m[0][0] * dL_dT00 + Wm.m[0][1] * dL_dT01 + Wm.m[0][2] * dL_dT02;
      F dL_dJ02 = Wm.m[2][0] * dL_dT00 + Wm.m[2][1] * dL_dT01 + Wm.m[2][2] * dL_dT02;
      F dL_dJ11 = Wm.m[1][0] * dL_dT10 + Wm.m[1][1] * dL_dT11 + Wm.m[1][2] * dL_dT12;
      F dL_dJ12 = Wm.m[2][0] * dL_dT10 + Wm.m[2][1] * dL_dT11 + Wm.m[2][2] * dL_dT12;
      F tz = (F)1 / c.t.z, tz2 = tz * tz, tz3 = tz2 * tz;
      F dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
      F dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
      F dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * c.t.x) * tz3 * dL_dJ02 + (2 * h_y * c.t.y) * tz3 * dL_dJ12;
      // transformVec4x3Transpose, auxiliary.h:89-97 -- ASSIGNED (backward.cu:273)
      gr.dmean3D[3 * (size_t)idx + 0] = (F)view[0] * dL_dtx + (F)view[1] * dL_dty + (F)view[2] * dL_dtz;
      gr.dmean3D[3 * (size_t)idx + 1] = (F)view[4] * dL_dtx + (F)view[5] * dL_dty + (F)view[6] * dL_dtz;
      gr.dmean3D[3 * (size_t)idx + 2] = (F)view[8] * dL_dtx + (F)view[9] * dL_dty + (F)view[10] * dL_dtz;
    }
    // ---- preprocessCUDA (bwd) ----
    F mh[4];
    transformPoint4x4(mean, proj, mh);
    F m_w = (F)1 / (mh[3] + (F)0.0000001f);
    F mul1 = ((F)proj[0] * mean.x + (F)proj[4] * mean.y + (F)proj[8] * mean.z + (F)proj[12]) * m_w * m_w;
    F mul2 = ((F)proj[1] * mean.x + (F)proj[5] * mean.y + (F)proj[9] * mean.z + (F)proj[13]) * m_w * m_w;
    F g2x = gr.dmean2D[3 * (size_t)idx], g2y = gr.dmean2D[3 * (size_t)idx + 1];
    gr.dmean3D[3 * (size_t)idx + 0] += ((F)proj[0] * m_w - (F)proj[3] * mul1) * g2x + ((F)proj[1] * m_w - (F)proj[3] * mul2) * g2y;
    gr.dmean3D[3 * (size_t)idx + 1] += ((F)proj[4] * m_w - (F)proj[7] * mul1) * g2x + ((F)proj[5] * m_w - (F)proj[7] * mul2) * g2y;
    gr.dmean3D[3 * (size_t)idx + 2] += ((F)proj[8] * m_w - (F)proj[11] * mul1) * g2x + ((F)proj[9] * m_w - (F)proj[11] * mul2) * g2y;
    if (p.shs) {
      // backward.cu:20-139
      F ox = mean.x - (F)p.campos[0], oy = mean.y - (F)p.campos[1], oz = mean.z - (F)p.campos[2];
      F len = std::sqrt(ox * ox + oy * oy + oz * oz);
      F x = ox / len, y = oy / len, z = oz / len;
      const float* shp = p.shs + (size_t)idx * M * 3;
      auto SH = [&](int k, int ch) { return (F)shp[3 * k + ch]; };
      F dRGB[3];
      for (int ch = 0; ch < 3; ch++) dRGB[ch] = gr.dcolor[3 * (size_t)idx + ch] * (g.clamped[3 * (size_t)idx + ch] ? 0 : 1);
      F bs[16];
      sh_basis<F>(p.D, x, y, z, bs);
      int nb = (p.D + 1) * (p.D + 1);
      F* dsh = &gr.dsh[(size_t)idx * M * 3];
      for (int k = 0; k < nb; k++)
        for (int ch = 0; ch < 3; ch++) dsh[3 * k + ch] = bs[k] * dRGB[ch];
      F ddir[3] = {0, 0, 0};
      for (int ch = 0; ch < 3; ch++) {
        F dx_ = 0, dy_ = 0, dz_ = 0;
        if (p.D > 0) {
          dx_ = -(F)SH_C1 * SH(3, ch); dy_ = -(F)SH_C1 * SH(1, ch); dz_ = (F)SH_C1 * SH(2, ch);
          if (p.D > 1) {
            F xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            dx_ += (F)SH_C2[0] * y * SH(4, ch) + (F)SH_C2[2] * (F)2 * -x * SH(6, ch) + (F)SH_C2[3] * z * SH(7, ch) + (F)SH_C2[4] * (F)2 * x * SH(8, ch);
            dy_ += (F)SH_C2[0] * x * SH(4, ch) + (F)SH_C2[1] * z * SH(5, ch) + (F)SH_C2[2] * (F)2 * -y * SH(6, ch) + (F)SH_C2[4] * (F)2 * -y * SH(8, ch);
            dz_ += (F)SH_C2[1] * y * SH(5, ch) + (F)SH_C2[2] * (F)2 * (F)2 * z * SH(6, ch) + (F)SH_C2[3] * x * SH(7, ch);
            if (p.D > 2) {
              dx_ += ((F)SH_C3[0] * SH(9, ch) * (F)3 * (F)2 * xy + (F)SH_C3[1] * SH(10, ch) * yz + (F)SH_C3[2] * SH(11, ch) * (F)-2 * xy +
                      (F)SH_C3[3] * SH(12, ch) * (F)-3 * (F)2 * xz + (F)SH_C3[4] * SH(13, ch) * ((F)-3 * xx + (F)4 * zz - yy) +
                      (F)SH_C3[5] * SH(14, ch) * (F)2 * xz + (F)SH_C3[6] * SH(15, ch) * (F)3 * (xx - yy));
              dy_ += ((F)SH_C3[0] * SH(9, ch) * (F)3 * (xx - yy) + (F)SH_C3[1] * SH(10, ch) * xz + (F)SH_C3[2] * SH(11, ch) * ((F)-3 * yy + (F)4 * zz - xx) +
                      (F)SH_C3[3] * SH(12, ch) * (F)-3 * (F)2 * yz + (F)SH_C3[4] * SH(13, ch) * (F)-2 * xy + (F)SH_C3[5] * SH(14, ch) * (F)-2 * yz +
                      (F)SH_C3[6] * SH(15, ch) * (F)-3 * (F)2 * xy);
              dz_ += ((F)SH_C3[1] * SH(10, ch) * xy + (F)SH_C3[2] * SH(11, ch) * (F)4 * (F)2 * yz + (F)SH_C3[3] * SH(12, ch) * (F)3 * ((F)2 * zz - xx - yy) +
                      (F)SH_C3[4] * SH(13, ch) * (F)4 * (F)2 * xz + (F)SH_C3[5] * SH(14, ch) * (xx - yy));
            }
          }
        }
        ddir[0] += dx_ * dRGB[ch]; ddir[1] += dy_ * dRGB[ch]; ddir[2] += dz_ * dRGB[ch];
      }
      // dnormvdv, auxiliary.h:107-117
      F sum2 = ox * ox + oy * oy + oz * oz;
      F invsum32 = (F)1 / std::sqrt(sum2 * sum2 * sum2);
      gr.dmean3D[3 * (size_t)idx + 0] += ((+sum2 - ox * ox) * ddir[0] - oy * ox * ddir[1] - oz * ox * ddir[2]) * invsum32;
      gr.dmean3D[3 * (size_t)idx + 1] += (-ox * oy * ddir[0] + (sum2 - oy * oy) * ddir[1] - oz * oy * ddir[2]) * invsum32;
      gr.dmean3D[3 * (size_t)idx + 2] += (-ox * oz * ddir[0] - oy * oz * ddir[1] + (sum2 - oz * oz) * ddir[2]) * invsum32;
    }
    if (p.scales) {
      // backward.cu:278-341 computeCov3D (bwd)
      const float* rot = p.rotations + 4 * (size_t)idx;
      F r = rot[0], x = rot[1], y = rot[2], z = rot[3];
      M3<F> R;
      R.m[0][0] = (F)1 - (F)2 * (y * y + z * z); R.m[0][1] = (F)2 * (x * y - r * z); R.m[0][2] = (F)2 * (x * z + r * y);
      R.m[1][0] = (F)2 * (x * y + r * z); R.m[1][1] = (F)1 - (F)2 * (x * x + z * z); R.m[1][2] = (F)2 * (y * z - r * x);
      R.m[2][0] = (F)2 * (x * z - r * y); R.m[2][1] = (F)2 * (y * z + r * x); R.m[2][2] = (F)1 - (F)2 * (x * x + y * y);
      F s[3] = {(F)p.scale_modifier * (F)p.scales[3 * (size_t)idx], (F)p.scale_modifier * (F)p.scales[3 * (size_t)idx + 1],
                (F)p.scale_modifier * (F)p.scales[3 * (size_t)idx + 2]};
      M3<F> S = {};
      S.m[0][0] = s[0]; S.m[1][1] = s[1]; S.m[2][2] = s[2];
      M3<F> Mm = mul(S, R);
      const F* d = &gr.dcov3D[6 * (size_t)idx];
      M3<F> dSig;
      dSig.m[0][0] = d[0]; dSig.m[0][1] = (F)0.5f * d[1]; dSig.m[0][2] = (F)0.5f * d[2];
      dSig.m[1][0] = (F)0.5f * d[1]; dSig.m[1][1] = d[3]; dSig.m[1][2] = (F)0.5f * d[4];
      dSig.m[2][0] = (F)0.5f * d[2]; dSig.m[2][1] = (F)0.5f * d[4]; dSig.m[2][2] = d[5];
      M3<F> twoM;
      for (int c = 0; c < 3; c++) for (int rr = 0; rr < 3; rr++) twoM.m[c][rr] = Mm.m[c][rr] * (F)2.0f;  // scalar*mat = m[c]*scalar
      M3<F> dL_dM = mul(twoM, dSig);
      M3<F> Rt = transpose(R), dMt = transpose(dL_dM);
      for (int j = 0; j < 3; j++)
        gr.dscale[3 * (size_t)idx + j] = Rt.m[j][0] * dMt.m[j][0] + Rt.m[j][1] * dMt.m[j][1] + Rt.m[j][2] * dMt.m[j][2];
      for (int j = 0; j < 3; j++) for (int k = 0; k < 3; k++) dMt.m[j][k] *= s[j];
      F* dq = &gr.drot[4 * (size_t)idx];
      dq[0] = 2 * z * (dMt.m[0][1] - dMt.m[1][0]) + 2 * y * (dMt.m[2][0] - dMt.m[0][2]) + 2 * x * (dMt.m[1][2] - dMt.m[2][1]);
      dq[1] = 2 * y * (dMt.m[1][0] + dMt.m[0][1]) + 2 * z * (dMt.m[2][0] + dMt.m[0][2]) + 2 * r * (dMt.m[1][2] - dMt.m[2][1]) - 4 * x * (dMt.m[2][2] + dMt.m[1][1]);
      dq[2] = 2 * x * (dMt.m[1][0] + dMt.m[0][1]) + 2 * r * (dMt.m[2][0] - dMt.m[0][2]) + 2 * z * (dMt.m[1][2] + dMt.m[2][1]) - 4 * y * (dMt.m[2][2] + dMt.m[0][0]);
      dq[3] = 2 * r * (dMt.m[0][1] - dMt.m[1][0]) + 2 * x * (dMt.m[2][0] + dMt.m[0][2]) + 2 * y * (dMt.m[1][2] + dMt.m[2][1]) - 4 * z * (dMt.m[1][1] + dMt.m[0][0]);
    }
  }
}

template <typename F> struct Ctx {
  Params p;
  Geom<F> g;
  Binning b;
  Image<F> im;
  Grads<F> gr;
  Stats st;
  // owned copies of the inputs so backward can run after the caller's arrays are gone
  std::vector<float> bg, means3D, shs, colors, opac, scales, rots, cov3Dp, view, proj, campos;
};

template <typename F> void copy_out(void* dst, const std::vector<F>& v) {
  if (dst && !v.empty()) std::memcpy(dst, v.data(), v.size() * sizeof(F));
}

template <typename F>
void* forward_impl(int P, int D, int M, int W, int H, const float* bg, const float* means3D, const float* shs,
                   const float* colors_precomp, const float* opacities, const float* scales, float scale_modifier,
                   const float* rotations, const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                   const float* campos, float tan_fovx, float tan_fovy, bool render) {
  auto* c = new Ctx<F>();
  auto own = [](std::vector<float>& v, const float* src, size_t n) -> const float* {
    if (!src || n == 0) return nullptr;
    v.assign(src, src + n);
    return v.data();
  };
  Params& p = c->p;
  p.P = P; p.D = D; p.M = M; p.W = W; p.H = H;
  p.tan_fovx = tan_fovx; p.tan_fovy = tan_fovy; p.scale_modifier = scale_modifier;
  p.bg = own(c->bg, bg, 3);
  p.means3D = own(c->means3D, means3D, 3 * (size_t)P);
  p.shs = own(c->shs, shs, 3 * (size_t)P * M);
  p.colors_precomp = own(c->colors, colors_precomp, 3 * (size_t)P);
  p.opacities = own(c->opac, opacities, P);
  p.scales = own(c->scales, scales, 3 * (size_t)P);
  p.rotations = own(c->rots, rotations, 4 * (size_t)P);
  p.cov3D_precomp = own(c->cov3Dp, cov3D_precomp, 6 * (size_t)P);
  p.viewmatrix = own(c->view, viewmatrix, 16);
  p.projmatrix = own(c->proj, projmatrix, 16);
  p.campos = own(c->campos, campos, 3);
  if (P > 0) {
    preprocess<F>(p, c->g);
    bin<F>(p, c->g, c->b);
    if (render) render_forward<F>(p, c->g, c->b, c->im, &c->st);
  } else {
    c->b.ranges.assign(2 * (size_t)((W + 15) / 16) * ((H + 15) / 16), 0);
    if (render) {
      c->im.out_color.assign(3 * (size_t)W * H, 0); c->im.out_depth.assign((size_t)W * H, 0);
      c->im.final_T.assign((size_t)W * H, 0); c->im.n_contrib.assign((size_t)W * H, 0);
    }
  }
  return c;
}

}  // namespace

#define ORACLE_API extern "C" __attribute__((visibility("default")))

// ---- C entry points (ctypes) -------------------------------------------------------------
// `f32` != 0 selects the float variant, else double. All *output* pointers are typed
// accordingly (float* or double*); integer outputs are fixed-width.

ORACLE_API void* oracle_forward(int f32, int P, int D, int M, int W, int H, const float* bg, const float* means3D,
                                const float* shs, const float* colors_precomp, const float* opacities,
                                const float* scales, float scale_modifier, const float* rotations,
                                const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                                const float* campos, float tan_fovx, float tan_fovy, int render) {
  if (f32)
    return forward_impl<float>(P, D, M, W, H, bg, means3D, shs, colors_precomp, opacities, scales, scale_modifier,
                               rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, render);
  return forward_impl<double>(P, D, M, W, H, bg, means3D, shs, colors_precomp, opacities, scales, scale_modifier,
                              rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, render);
}

ORACLE_API int64_t oracle_num_rendered(int f32, void* h) {
  return f32 ? ((Ctx<float>*)h)->b.R : ((Ctx<double>*)h)->b.R;
}

ORACLE_API void oracle_stats(int f32, void* h, int64_t* pairs, int64_t* hits) {
  const Stats& s = f32 ? ((Ctx<float>*)h)->st : ((Ctx<double>*)h)->st;
  *pairs = s.pairs; *hits = s.hits;
}

template <typename F>
static void get_forward(Ctx<F>* c, void* out_color, void* out_depth, int32_t* radii, void* final_T, uint32_t* n_contrib,
                        void* depths, void* means2D, void* conic_opacity, void* rgb, void* cov3D, uint8_t* clamped,
                        uint32_t* tiles_touched, uint32_t* point_offsets, uint64_t* keys, uint32_t* point_list,
                        uint32_t* ranges) {
  copy_out<F>(out_color, c->im.out_color); copy_out<F>(out_depth, c->im.out_depth);
  copy_out<F>(final_T, c->im.final_T);
  if (n_contrib && !c->im.n_contrib.empty()) std::memcpy(n_contrib, c->im.n_contrib.data(), 4 * c->im.n_contrib.size());
  if (radii && !c->g.radii.empty()) std::memcpy(radii, c->g.radii.data(), 4 * c->g.radii.size());
  copy_out<F>(depths, c->g.depths); copy_out<F>(means2D, c->g.means2D); copy_out<F>(conic_opacity, c->g.conic_opacity);
  copy_out<F>(rgb, c->g.rgb); copy_out<F>(cov3D, c->g.cov3D);
  if (clamped && !c->g.clamped.empty()) std::memcpy(clamped, c->g.clamped.data(), c->g.clamped.size());
  if (tiles_touched && !c->g.tiles_touched.empty()) std::memcpy(tiles_touched, c->g.tiles_touched.data(), 4 * c->g.tiles_touched.size());
  if (point_offsets && !c->g.point_offsets.empty()) std::memcpy(point_offsets, c->g.point_offsets.data(), 4 * c->g.point_offsets.size());
  if (keys && !c->b.keys.empty()) std::memcpy(keys, c->b.keys.data(), 8 * c->b.keys.size());
  if (point_list && !c->b.point_list.empty()) std::memcpy(point_list, c->b.point_list.data(), 4 * c->b.point_list.size());
  if (ranges && !c->b.ranges.empty()) std::memcpy(ranges, c->b.ranges.data(), 4 * c->b.ranges.size());
}

ORACLE_API void oracle_get_forward(int f32, void* h, void* out_color, void* out_depth, int32_t* radii, void* final_T,
                                   uint32_t* n_contrib, void* depths, void* means2D, void* conic_opacity, void* rgb,
                                   void* cov3D, uint8_t* clamped, uint32_t* tiles_touched, uint32_t* point_offsets,
                                   uint64_t* keys, uint32_t* point_list, uint32_t* ranges) {
  if (f32) get_forward<float>((Ctx<float>*)h, out_color, out_depth, radii, final_T, n_contrib, depths, means2D,
                              conic_opacity, rgb, cov3D, clamped, tiles_touched, point_offsets, keys, point_list, ranges);
  else get_forward<double>((Ctx<double>*)h, out_color, out_depth, radii, final_T, n_contrib, depths, means2D,
                           conic_opacity, rgb, cov3D, clamped, tiles_touched, point_offsets, keys, point_list, ranges);
}

template <typename F>
static void backward_impl(Ctx<F>* c, const float* dL_dpix, void* dmean2D, void* dconic, void* dopacity, void* dcolor,
                          void* dmean3D, void* dcov3D, void* dsh, void* dscale, void* drot) {
  const int P = c->p.P;
  Grads<F>& gr = c->gr;
  if (P > 0) {
    render_backward<F>(c->p, c->g, c->b, c->im, dL_dpix, gr);
    preprocess_backward<F>(c->p, c->g, gr);
  }
  copy_out<F>(dmean2D, gr.dmean2D); copy_out<F>(dconic, gr.dconic); copy_out<F>(dopacity, gr.dopacity);
  copy_out<F>(dcolor, gr.dcolor); copy_out<F>(dmean3D, gr.dmean3D); copy_out<F>(dcov3D, gr.dcov3D);
  copy_out<F>(dsh, gr.dsh); copy_out<F>(dscale, gr.dscale); copy_out<F>(drot, gr.drot);
}

// DGR/rasterize_points.cu:120-128 shapes: dmean2D[P,3] dconic[P,2,2] dopacity[P,1] dcolor[P,3] dmean3D[P,3]
// dcov3D[P,6] dsh[P,M,3] dscale[P,3] drot[P,4]; caller zero-fills (entries of invisible Gaussians stay 0).
ORACLE_API void oracle_backward(int f32, void* h, const float* dL_dpix, void* dmean2D, void* dconic, void* dopacity,
                                void* dcolor, void* dmean3D, void* dcov3D, void* dsh, void* dscale, void* drot) {
  if (f32) backward_impl<float>((Ctx<float>*)h, dL_dpix, dmean2D, dconic, dopacity, dcolor, dmean3D, dcov3D, dsh, dscale, drot);
  else backward_impl<double>((Ctx<double>*)h, dL_dpix, dmean2D, dconic, dopacity, dcolor, dmean3D, dcov3D, dsh, dscale, drot);
}

ORACLE_API void oracle_free(int f32, void* h) {
  if (f32) delete (Ctx<float>*)h; else delete (Ctx<double>*)h;
}

// rasterizer_impl.cu:53-63,128-133 checkFrustum / markVisible
ORACLE_API void oracle_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present) {
  for (int i = 0; i < P; i++) {
    V3<float> po = {means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]};
    present[i] = transformPoint4x3(po, viewmatrix).z > 0.2f;
  }
}

// apply_weights.cu:240-356 renderCUDA_apply_weights on top of the forward preprocess+binning of handle `h`
// (which must have been created with colors_precomp != null, sh == null: rasterize_points.cu:223).
// weights [P,CH] float (accumulated), cnt [P] int32 (advances CH per hit: :331-334), image_weights [CH,H,W].
ORACLE_API void oracle_apply_weights(void* h, float* weights, int32_t* cnt, const float* image_weights, int CH) {
  Ctx<float>* c = (Ctx<float>*)h;
  const Params& p = c->p;
  const int W = p.W, H = p.H;
  const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
  const Geom<float>& g = c->g;
  const Binning& b = c->b;
  for (int tile = 0; tile < gx * gy; tile++) {
    int ty = tile / gx, tx = tile % gx;
    uint32_t r0 = b.ranges[2 * tile], r1 = b.ranges[2 * tile + 1];
    for (int py = ty * BLOCK_Y; py < std::min((ty + 1) * BLOCK_Y, H); py++)
      for (int px = tx * BLOCK_X; px < std::min((tx + 1) * BLOCK_X, W); px++) {
        float T = 1.0f, C[3] = {0, 0, 0};
        size_t pix_id = (size_t)W * py + px;
        for (int ch = 0; ch < CH; ch++) C[ch] = image_weights[(size_t)ch * H * W + pix_id];
        for (uint32_t k = r0; k < r1; k++) {
          uint32_t id = b.point_list[k];
          float dx = g.means2D[2 * (size_t)id] - (float)px, dy = g.means2D[2 * (size_t)id + 1] - (float)py;
          const float* co = &g.conic_opacity[4 * (size_t)id];
          float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
          if (power > 0.0f) continue;
          float alpha = std::fmin(0.99f, co[3] * std::exp(power));
          if (alpha < 1.0f / 255.0f) continue;
          float test_T = T * (1 - alpha);
          if (test_T < 0.0001f) break;
          for (int ch = 0; ch < CH; ch++) { weights[(size_t)id * CH + ch] += C[ch]; cnt[id] += 1; }
          T = test_T;
        }
      }
  }
}

ORACLE_API int oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
