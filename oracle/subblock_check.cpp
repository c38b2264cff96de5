// ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Host build of the render kernels' sub-block culling predicate (gaussianeditor_b200/csrc/common.cuh:
// splat_subblock_mask, compiled here from the same header) checked against the reference's per-pixel hit test
//   power = splat_power(x - px, y - py, A, B, C);  hit = power <= 0 && min(0.99, o * expf(power)) >= 1/255
// (forward.cu:335-345). A (pixel, splat) pair that the predicate rejects but the hit test blends is a MISS: the
// kernels that use the predicate would drop a contribution the reference makes. Built by oracle/Makefile with
// -ffp-contract=off, so the header's host arithmetic rounds like its device intrinsics.
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "../gaussianeditor_b200/csrc/common.cuh"

namespace {

struct Counts {
  int64_t blocks = 0, rejected = 0, rejected_pixels = 0, misses = 0, hits = 0;
};

inline bool reference_hit(float x, float y, float A, float B, float C, float o, float px, float py) {
  const float power = gsr::splat_power(x - px, y - py, A, B, C);
  if (power > 0.0f) return false;
  return !(fminf(0.99f, gsr::mul_rn(o, expf(power))) < 1.0f / 255.0f);
}

// all 8 sub-blocks of tile (tx, ty) against every pixel in them (pixels at or beyond W x H are outside the frame)
template <int TERM_ULPS>
void check_tile(const float4 q0, const float4 q1, int tx, int ty, int W, int H, Counts& c) {
  const float X0 = (float)(tx * gsr::TILE), Y0 = (float)(ty * gsr::TILE);
  const uint32_t mask = gsr::splat_subblock_mask<8, TERM_ULPS>(q0, q1, X0, Y0, 0);
  for (int k = 0; k < 8; k++) {
    const bool keep = (mask >> k) & 1u;
    c.blocks++;
    c.rejected += !keep;
    for (int ly = 0; ly < 4; ly++)
      for (int lx = 0; lx < 8; lx++) {
        const int px = tx * gsr::TILE + 8 * (k & 1) + lx, py = ty * gsr::TILE + 4 * (k >> 1) + ly;
        if (px >= W || py >= H) continue;
        const bool hit = reference_hit(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, (float)px, (float)py);
        c.hits += hit;
        if (!keep) {
          c.rejected_pixels++;
          c.misses += hit;
        }
      }
  }
}

void check_tile_any(int term_ulps, const float4 q0, const float4 q1, int tx, int ty, int W, int H, Counts& c) {
  if (term_ulps == 0)
    check_tile<0>(q0, q1, tx, ty, W, H, c);
  else
    check_tile<16>(q0, q1, tx, ty, W, H, c);
}

// counter-based generator: splat i draws the same numbers whatever the thread count
struct Rng {
  uint64_t s;
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uni() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

void add(Counts& a, const Counts& b) {
  a.blocks += b.blocks; a.rejected += b.rejected; a.rejected_pixels += b.rejected_pixels;
  a.misses += b.misses; a.hits += b.hits;
}

void store(const Counts& c, int64_t* out) {
  out[0] = c.blocks; out[1] = c.rejected; out[2] = c.rejected_pixels; out[3] = c.misses; out[4] = c.hits;
}

}  // namespace

extern "C" {

// Seeded sweep of needle-like splats. Splat i: 2-D covariance with long-axis variance log-uniform in
// [10, 10^4.5] px^2, short axis at the 0.3 px^2 dilation floor, angle uniform (both signs of B); opacity: a third
// within 5 % above 1/255 (the first of those exactly fp32(1/255)), a third in [0.95, 1] (the 0.99 clamp), a third
// uniform in (1/255, 1]. Tiles: `tip_tiles` around the ends of the alpha = 1/255 contour along the long axis (where the
// terms of `power` are largest and cancel), and `random_tiles` anywhere in the splat's 3-sigma square.
// Counts (out[5]): sub-blocks tested, sub-blocks rejected, pixels in rejected sub-blocks, misses, reference hits.
__attribute__((visibility("default"))) void subblock_sweep(uint64_t seed, int nsplat, int tip_tiles, int random_tiles,
                                                           int term_ulps, int64_t* out) {
  Counts total;
#pragma omp parallel
  {
    Counts c;
#pragma omp for schedule(dynamic, 256)
    for (int i = 0; i < nsplat; i++) {
      Rng r{seed * 0x100000001B3ull + (uint64_t)i};
      const double lam1 = pow(10.0, 1.0 + 3.5 * r.uni()), lam2 = 0.3;
      const double th = M_PI * r.uni(), cs = cos(th), sn = sin(th);
      const double a = lam1 * cs * cs + lam2 * sn * sn, b = (lam1 - lam2) * cs * sn, cc = lam1 * sn * sn + lam2 * cs * cs;
      const double det = a * cc - b * b;
      const float A = (float)(cc / det), B = (float)(-b / det), C = (float)(a / det);
      const int kind = i % 3;
      float o;
      if (kind == 0)
        o = (i % 300 == 0) ? 1.0f / 255.0f : (float)((1.0 + 0.05 * r.uni()) / 255.0);
      else if (kind == 1)
        o = (float)(0.95 + 0.05 * r.uni());
      else
        o = (float)(1.0 / 255.0 + (1.0 - 1.0 / 255.0) * r.uni());
      const float x = (float)(4096.0 + 4096.0 * r.uni()), y = (float)(4096.0 + 4096.0 * r.uni());
      const float4 q0 = make_float4(x, y, A, B), q1 = make_float4(C, o, 0.f, 0.f);
      const double thr = 2.0 * log(fmax(255.0 * o, 1.0)), L = sqrt(thr * lam1), w = sqrt(thr * lam2) + 2.0;
      for (int t = 0; t < tip_tiles; t++) {  // a point near one end of the contour, +-30 % along, +-w across
        const double s = (r.uni() < 0.5 ? -1.0 : 1.0) * L * (0.7 + 0.6 * r.uni()), n = w * (2.0 * r.uni() - 1.0);
        const double px = x + s * cs - n * sn, py = y + s * sn + n * cs;
        check_tile_any(term_ulps, q0, q1, (int)floor(px / gsr::TILE), (int)floor(py / gsr::TILE), 1 << 30, 1 << 30, c);
      }
      const double rad = ceil(3.0 * sqrt(lam1));
      for (int t = 0; t < random_tiles; t++) {
        const double px = x + rad * (2.0 * r.uni() - 1.0), py = y + rad * (2.0 * r.uni() - 1.0);
        check_tile_any(term_ulps, q0, q1, (int)floor(px / gsr::TILE), (int)floor(py / gsr::TILE), 1 << 30, 1 << 30, c);
      }
    }
#pragma omp critical
    add(total, c);
  }
  store(total, out);
}

// The same check over a projected scene: every tile of every visible splat's tile rectangle (the reference's getRect,
// auxiliary.h:46-56, from means2D and radii), pixels inside the W x H frame. means2D [P,2], conic_opacity [P,4].
__attribute__((visibility("default"))) void subblock_scene(int P, const float* means2D, const float* conic_opacity,
                                                           const int* radii, int W, int H, int term_ulps,
                                                           int64_t* out) {
  const int gx = (W + gsr::TILE - 1) / gsr::TILE, gy = (H + gsr::TILE - 1) / gsr::TILE;
  Counts total;
#pragma omp parallel
  {
    Counts c;
#pragma omp for schedule(dynamic, 16)
    for (int i = 0; i < P; i++) {
      if (radii[i] <= 0) continue;
      const float x = means2D[2 * i], y = means2D[2 * i + 1];
      const float4 q0 = make_float4(x, y, conic_opacity[4 * i], conic_opacity[4 * i + 1]);
      const float4 q1 = make_float4(conic_opacity[4 * i + 2], conic_opacity[4 * i + 3], 0.f, 0.f);
      uint2 rmin, rmax;  // the kernels' own rectangle (saturating conversions: a radius of INT_MAX covers the grid)
      gsr::tile_rect(x, y, radii[i], gx, gy, rmin, rmax);
      for (int ty = (int)rmin.y; ty < (int)rmax.y; ty++)
        for (int tx = (int)rmin.x; tx < (int)rmax.x; tx++) check_tile_any(term_ulps, q0, q1, tx, ty, W, H, c);
    }
#pragma omp critical
    add(total, c);
  }
  store(total, out);
}

}  // extern "C"
