// Backward of the alpha blending for sm_90a: per-pixel dL/dcolor -> per-Gaussian 2-D gradients
// (dL/dcolor, dL/dmean2D, dL/dconic, dL/dopacity), accumulated into the 48-byte-per-Gaussian scratch `acc`.
//
// Semantics: renderCUDA (bwd) of the reference (cuda_rasterizer/backward.cu:399-557): walk each tile's list
// back to front, skip list positions behind the pixel's last contributor, recompute G = exp(power) and alpha
// with the forward's arithmetic (same skip decisions), T <- T/(1-alpha), and accumulate nine partial sums per
// (pixel, splat) hit.
//
// The reference issues nine global float atomics PER HIT (~10^9 REDG at config 3) and walks every tile list
// from its very end.  Here:
//   * the walk starts at tile_last = max n_contrib of the tile (written by the forward): on a saturated scene
//     three quarters of every list lie behind the last contributor of all 256 pixels and are never loaded;
//   * warp variants (1/2/3 branchy, 4..9 branch-light, 10/11 skip by sub-block mask, 12..14 register caps; 14 =
//     one warp per half tile, 96 registers -> 5 CTAs/SM, updates of sub-blocks without a hit skipped warp-uniformly:
//     0.627 ms at config 3 on an H100 80GB HBM3; the A/B of all of them is in DESIGN.md section 3): a
//     warp owns a whole tile, half or a quarter of it, each lane owns one pixel of each of its
//     8x4 sub-blocks; the nine partial sums are first accumulated over the lane's own pixels in registers,
//     then summed across the warp with a transposing butterfly (16 shuffles for 9 values instead of 45), and
//     only then added to global memory: 9 atomics per (tile, splat) instead of 9 per (pixel, splat);
//   * DEFAULT 15 = variant 14 with that warp reduction deferred: the moments of 4 splats are summed at once through
//     shared memory (flush_moments), 0.553 instead of 0.646 ms at config 3 on an H100 80GB HBM3 at a 400 W power limit;
//   * the same opacity-aware sub-block culling as the forward (render_fwd.cu) removes splats whose
//     alpha>=1/255 ellipse misses the sub-block before any pixel looks at them.
// Variant 0: the reference's CTA-per-tile structure with a plain warp-shuffle reduction before the atomics.
//
// Gradients are sums of floats in a different order than the reference's atomics (which are themselves
// non-deterministic), so parity is to tolerance (tests: rel L2 <= 1e-4), not bit-exact.
#include <type_traits>

#include "common.cuh"

namespace gsr {

namespace {

struct BwdArgs {
  const uint2* ranges;
  const uint32_t* point_list;
  const SplatRecord* records;
  const uint32_t* tile_last;
  int W, H, gx, gy;
  const float* bg;
  const float* final_T;
  const uint32_t* n_contrib;
  const float* dL_dpix;
  const float* dL_dalpha_img;  // optional [H*W]: gradient of the alpha image 1 - final_T (gsr_backward_alpha)
  float* acc;  // [P, ACC_STRIDE]
  int own_stride, own_phase;  // tile-row ownership (1, 0 = all tiles)
};
// Arguments of the depth instantiation: a separate type, so that the parameter block of every other kernel keeps its
// size and layout (and those kernels their code).
struct BwdDepthArgs : BwdArgs {
  const float* dL_ddepth;  // [H*W] gradient of the depth image (gsr_backward_depth)
};
// Arguments of the deterministic instantiations (DET): the finished rows go to rows[2*slot + part] with a flag instead
// of atomics into acc (common.cuh: DetWS); again a separate type, so the other kernels keep their parameter block.
template <class Base> struct BwdDetArgs : Base {
  const uint32_t* excl;  // [P] exclusive prefix of the tile counts in depth order
  float* rows;           // [2R, ACC_STRIDE]
  uint8_t* flags;        // [2R]
};
// Arguments of the masked instantiations (MASK, gsr_backward_masked): which Gaussians take gradients, and where each
// tile's walk may stop (grad_mask_first_kernel).
template <class Base> struct BwdMaskArgs : Base {
  const uint8_t* grad_mask;  // [P] nonzero: the Gaussian is edited (unused by render_bwd_recmask_kernel)
  const uint32_t* first;     // [Ntile] 1-based position of the front-most edited instance, GRAD_MASK_NONE if none
};
template <bool DEPTH, bool DET = false>
using BwdArgsT = std::conditional_t<DET, BwdDetArgs<std::conditional_t<DEPTH, BwdDepthArgs, BwdArgs>>,
                                    std::conditional_t<DEPTH, BwdDepthArgs, BwdArgs>>;

// One (pixel, splat) hit. `ar` tracks the reference's accum_rec (backward.cu:515) dotted with dL_dpixel, updated
// eagerly; `bgT` = T_final * (bg . dL_dpixel).
//
// The nine sums of backward.cu:523-554 are accumulated as moments of w = dL_dG * G over the pixels,
//   g[3..7] = sum w*{dx, dy, dx*dx, dx*dy, dy*dy},  g[8] = sum w,  g[0..2] = sum alpha*T*dL_dpixel,
// and turned into the reference's quantities once per (tile, splat) by finish_sums() -- the per-splat factors
// (conic, opacity, 0.5*W, 0.5*H) are constant over the pixels, so this is the same sum with the common factor
// pulled out (8 instead of 17 operations per hit).
//
// The depth image D = sum z*alpha*T (no background term) is a fourth channel with colour z, so with a depth upstream
// dD = dL/dD the DEPTH kernels add z*dD to that dot product and keep a tenth moment g[9] = sum alpha*T*dD = dL/dz.
struct PixState {
  float T, ar, d0, d1, d2, bgT;   // ar = accum_rec . dL_dpixel (scalar; see hit_update)
  float dD;                       // DEPTH only: dL/dD of the pixel
};

// What multiplies dT_final/dalpha_i = -T_final/(1-alpha_i) in dL/dalpha_i: the background term of the colour
// (backward.cu:505-511: bg . dL_dpixel) and, when the caller asked for the alpha image A = 1 - T_final, -dL/dA.
__device__ __forceinline__ float bg_term(const BwdArgs& a, size_t pix_id, float bg0, float bg1, float bg2, const PixState& p) {
  float t = bg0 * p.d0 + bg1 * p.d1 + bg2 * p.d2;
  if (a.dL_dalpha_img != nullptr) t -= a.dL_dalpha_img[pix_id];
  return t;
}

template <bool DEPTH = false>
__device__ __forceinline__ void hit_update(PixState& p, float* g, float dx, float dy, float G, float alpha, float o,
                                           float c0, float c1, float c2, float z = 0.f) {
  const float oma = 1.f - alpha;
  float rcp;  // 1-alpha is in [0.01, 1]: the bare MUFU.RCP (<= 1 ulp here) needs no range fix-up
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rcp) : "f"(oma));
  rcp = alpha > 0.f ? rcp : 1.0f;          // (alpha, G) = (0, 0) encodes "no hit" in the branch-light variants: exact no-op
  p.T = p.T * rcp;                         // T / (1 - alpha)
  const float dchannel_dcolor = alpha * p.T;
  // backward.cu:515-519 keeps the blended colour behind the splat per channel (accum_rec) and forms
  // sum_ch (c_ch - accum_rec_ch) * dL_dpixel_ch. Only that dot product is ever used, and the recurrence
  // accum_rec' = alpha*c + (1-alpha)*accum_rec is linear, so the scalar ar = accum_rec . dL_dpixel obeys
  // ar' = ar + alpha*(c.dL_dpixel - ar): one state variable and 5 operations instead of three and 9.
  float s = fmaf(c2, p.d2, fmaf(c1, p.d1, c0 * p.d0));
  if constexpr (DEPTH) s = fmaf(z, p.dD, s);  // the depth channel: colour z, upstream dL/dD
  float dL_dalpha = s - p.ar;
  g[0] = fmaf(dchannel_dcolor, p.d0, g[0]);
  g[1] = fmaf(dchannel_dcolor, p.d1, g[1]);
  g[2] = fmaf(dchannel_dcolor, p.d2, g[2]);
  if constexpr (DEPTH) g[9] = fmaf(dchannel_dcolor, p.dD, g[9]);
  p.ar = fmaf(alpha, dL_dalpha, p.ar);
  dL_dalpha = fmaf(dL_dalpha, p.T, -p.bgT * rcp);
  const float w = (o * dL_dalpha) * G;  // dL_dG * G
  const float wdx = w * dx, wdy = w * dy;
  g[3] += wdx;
  g[4] += wdy;
  g[5] = fmaf(wdx, dx, g[5]);
  g[6] = fmaf(wdx, dy, g[6]);
  g[7] = fmaf(wdy, dy, g[7]);
  g[8] += w;
}

// MASK: the pixel-state part of hit_update alone, for a splat of a Gaussian that takes no gradient. The operations are
// hit_update's own (rcp with its alpha > 0 select, T * rcp, the dot product s, ar + alpha*(s - ar)), so every later
// edited splat sees the bits it would see in the unmasked walk.
template <bool DEPTH = false>
__device__ __forceinline__ void state_update(PixState& p, float alpha, float c0, float c1, float c2, float z = 0.f) {
  const float oma = 1.f - alpha;
  float rcp;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rcp) : "f"(oma));
  rcp = alpha > 0.f ? rcp : 1.0f;
  p.T = p.T * rcp;
  float s = fmaf(c2, p.d2, fmaf(c1, p.d1, c0 * p.d0));
  if constexpr (DEPTH) s = fmaf(z, p.dD, s);
  const float dL_dalpha = s - p.ar;
  p.ar = fmaf(alpha, dL_dalpha, p.ar);
}

// Warp totals of the moments -> the reference's nine gradient contributions (acc layout: 0..2 dcolor, 3..4 dmean2D,
// 5..7 dconic a,b,c, 8 dopacity). After warp_sum9 lane 4*j holds the total of moment j (j = 0..7) and every lane holds
// sw = sum w. Output j is a two-term combination  ka*tot + kb*other  with `other` = the partner moment of the
// (w*dx, w*dy) pair (lanes 12..15 <-> 16..19, one shuffle) and lane-constant selectors -- no divergent code:
//   j<3: tot | j=3: -(A*s_x + B*s_y)*0.5W | j=4: -(C*s_y + B*s_x)*0.5H | j=5..7: -0.5*tot | opacity: sw / o
struct LaneRole {
  bool is_x, is_y, writer, opac;  // moment-3 group, moment-4 group, lane that issues the atomic, opacity lane
  float kconst;                   // 1 for the colour groups, -0.5 for the conic groups
  int slot;
};
__device__ __forceinline__ LaneRole lane_role(int lane) {
  LaneRole r;
  r.slot = lane >> 2;
  r.is_x = r.slot == 3;
  r.is_y = r.slot == 4;
  r.writer = (lane & 3) == 0;
  r.opac = lane == 1;
  r.kconst = r.slot < 3 ? 1.0f : -0.5f;
  return r;
}
__device__ __forceinline__ void finish_and_add(float* dst, float tot, float sw, const LaneRole& role, float A, float B,
                                               float C, float o, float ddelx_dx, float ddely_dy) {
  const float other = __shfl_xor_sync(0xffffffffu, tot, 28);  // s_x <-> s_y between lanes 12..15 and 16..19
  const float nBx = -B * ddelx_dx, nBy = -B * ddely_dy;
  const float ka = role.is_x ? -A * ddelx_dx : (role.is_y ? -C * ddely_dy : role.kconst);
  const float kb = role.is_x ? nBx : (role.is_y ? nBy : 0.0f);
  // only the two mean moments take the other axis: kb = 0 elsewhere, and 0 * other would turn a NaN moment of the conic
  // (a splat whose overflowed 2-D covariance gives a NaN conic) into a NaN colour gradient the reference does not have
  const float v = (role.is_x || role.is_y) ? fmaf(kb, other, ka * tot) : ka * tot;
  if (role.writer) atomicAdd(dst + role.slot, v);
  if (role.opac) atomicAdd(dst + 8, __fdividef(sw, o));  // dL/dopacity = sum G*dL_dalpha = (sum w) / o
}

// Sum nine per-lane values over the warp. g[0..7] go through a transposing butterfly: after it, lane 4*j (and
// its three neighbours) holds the warp total of g[j]; g[8] takes a plain butterfly. Returns this lane's total of
// value (lane>>2), and the total of g[8] in `g8`.
__device__ __forceinline__ float warp_sum9(const float* g, int lane, float& g8) {
  const unsigned F = 0xffffffffu;
  float a[4], b[2], c;
  {
    const bool up = lane & 16;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float keep = up ? g[4 + i] : g[i];
      const float send = up ? g[i] : g[4 + i];
      a[i] = keep + __shfl_xor_sync(F, send, 16);
    }
  }
  {
    const bool up = lane & 8;
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const float keep = up ? a[2 + i] : a[i];
      const float send = up ? a[i] : a[2 + i];
      b[i] = keep + __shfl_xor_sync(F, send, 8);
    }
  }
  {
    const bool up = lane & 4;
    const float keep = up ? b[1] : b[0];
    const float send = up ? b[0] : b[1];
    c = keep + __shfl_xor_sync(F, send, 4);
  }
  c += __shfl_xor_sync(F, c, 2);
  c += __shfl_xor_sync(F, c, 1);
  float t = g[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(F, t, o);
  g8 = t;
  return c;
}

// ------------------------------------------------------------------------------------------------------
// Variant 1: NSB sub-blocks per warp (8 = one warp per tile, 4 = two warps per tile)
// ------------------------------------------------------------------------------------------------------
constexpr int BW_WARPS = 4;

template <int NSB>
__global__ void __launch_bounds__(BW_WARPS * 32) render_bwd_warp_kernel(const BwdArgs a, const int ntiles) {
  __shared__ float4 s_stage[BW_WARPS][3][32];
  __shared__ uint32_t s_id[BW_WARPS][32];
  constexpr int PARTS = 8 / NSB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * BW_WARPS + warp;
  const int part = gw % PARTS;
  if (gw / PARTS >= ntiles) return;
  const int tile = owned_tile(gw / PARTS, a.gx, a.own_stride, a.own_phase);  // ntiles counts the OWNED tiles
  float4(*stg)[32] = s_stage[warp];
  uint32_t* sid = s_id[warp];

  const int tx = tile % a.gx, ty = tile / a.gx;
  const int lx = lane & 7, ly = lane >> 3;
  const float X0 = (float)(tx * TILE), Y0 = (float)(ty * TILE);
  const float fx = X0 + (float)lx, fy = Y0 + (float)ly;
  const uint2 range = a.ranges[tile];
  if (a.tile_last[tile] == 0) return;
  const size_t HW = (size_t)a.H * a.W;
  const float bg0 = a.bg[0], bg1 = a.bg[1], bg2 = a.bg[2];
  const float ddelx_dx = 0.5f * a.W, ddely_dy = 0.5f * a.H;
  const LaneRole role = lane_role(lane);

  PixState ps[NSB];
  uint32_t nc[NSB], sblast[NSB];
  uint32_t my_last = 0;
#pragma unroll
  for (int k = 0; k < NSB; k++) {
    const int kg = part * NSB + k;
    const int px = tx * TILE + 8 * (kg & 1) + lx, py = ty * TILE + 4 * (kg >> 1) + ly;
    PixState p;
    p.T = 0.f; p.ar = 0.f; p.d0 = p.d1 = p.d2 = 0.f; p.bgT = 0.f;
    nc[k] = 0;
    if (px < a.W && py < a.H) {
      const size_t pix_id = (size_t)a.W * py + px;
      const float Tf = a.final_T[pix_id];
      p.T = Tf;
      p.d0 = a.dL_dpix[pix_id];
      p.d1 = a.dL_dpix[HW + pix_id];
      p.d2 = a.dL_dpix[2 * HW + pix_id];
      p.bgT = Tf * bg_term(a, pix_id, bg0, bg1, bg2, p);
      nc[k] = a.n_contrib[pix_id];
    }
    ps[k] = p;
    sblast[k] = __reduce_max_sync(0xffffffffu, nc[k]);
    my_last = max(my_last, sblast[k]);
  }

  for (int hi = (int)my_last; hi > 0; hi -= 32) {
    // ---- stage positions hi, hi-1, ... (1-based), cull, compact (descending order is preserved) ----
    const int pos = hi - lane;
    uint32_t mask = 0, id = 0;
    float4 q0, q1, q2;
    if (pos >= 1) {
      id = a.point_list[range.x + pos - 1];
      const float4* r = reinterpret_cast<const float4*>(a.records + id);
      q0 = __ldg(r);
      q1 = __ldg(r + 1);
      q2 = __ldg(r + 2);
      mask = splat_subblock_mask<NSB>(q0, q1, X0, Y0, part);
    }
    const uint32_t keep = __ballot_sync(0xffffffffu, mask != 0);
    const int cnt = __popc(keep);
    if (mask != 0) {
      const int slot = __popc(keep & ((1u << lane) - 1u));
      q1.w = __uint_as_float(mask);
      q2.w = __uint_as_float((uint32_t)pos);
      stg[0][slot] = q0;
      stg[1][slot] = q1;
      stg[2][slot] = q2;
      sid[slot] = id;
    }
    __syncwarp();
    const uint32_t lo = (uint32_t)max(hi - 31, 1);
    uint32_t act = 0;  // sub-blocks that can still have a contributor at these positions
#pragma unroll
    for (int k = 0; k < NSB; k++)
      if (sblast[k] >= lo) act |= 1u << k;

    for (int j = 0; j < cnt; j++) {
      const float4 s1 = stg[1][j];
      const uint32_t m = __float_as_uint(s1.w) & act;
      if (m == 0) continue;
      const float4 s0 = stg[0][j];
      const float4 s2 = stg[2][j];
      const uint32_t spos = __float_as_uint(s2.w);
      float dxv[2], dxA[2], dxB[2], dyv[NSB / 2], t0[NSB / 2];
#pragma unroll
      for (int c = 0; c < 2; c++) {
        dxv[c] = s0.x - (fx + 8.0f * c);
        dxA[c] = __fmul_rn(dxv[c], s0.z);
        dxB[c] = __fmul_rn(dxv[c], s0.w);
      }
#pragma unroll
      for (int r = 0; r < NSB / 2; r++) {
        dyv[r] = s0.y - (fy + 4.0f * (float)(part * (NSB / 2) + r));
        t0[r] = __fmul_rn(__fmul_rn(dyv[r], s1.x), dyv[r]);
      }
      float g[9];
#pragma unroll
      for (int i = 0; i < 9; i++) g[i] = 0.f;
      bool any = false;
#pragma unroll
      for (int k = 0; k < NSB; k++) {
        if (!((m >> k) & 1u)) continue;  // warp-uniform
        const int c = k & 1, r = k >> 1;  // NSB is even, so the column parity of sub-block part*NSB+k is k&1
        const float dx = dxv[c], dy = dyv[r];
        const float s = __fmaf_rn(dx, dxA[c], t0[r]);
        const float power = __fmaf_rn(s, -0.5f, -__fmul_rn(dxB[c], dy));
        if (power > 0.0f || spos > nc[k]) continue;
        const float G = expf(power);
        const float alpha = fminf(0.99f, __fmul_rn(s1.y, G));
        if (alpha < 1.0f / 255.0f) continue;
        any = true;
        hit_update(ps[k], g, dx, dy, G, alpha, s1.y, s2.x, s2.y, s2.z);
      }
      if (__any_sync(0xffffffffu, any)) {
        float m8;
        const float tot = warp_sum9(g, lane, m8);
        finish_and_add(a.acc + (size_t)sid[j] * ACC_STRIDE, tot, m8, role, s0.z, s0.w, s1.x, s1.y, ddelx_dx, ddely_dy);
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------------
// Variant 4/5: same mapping as variant 2 (NSB sub-blocks per warp) with a branch-light inner body.
// The profile of variant 2 is latency-bound (33 % of the stall samples are fixed-latency dependency waits, 11 % branch
// resolution, 16 warps/SM): here the NSB evaluations of a splat are issued as independent straight-line chains
// (instruction-level parallelism NSB), hit / no-hit is folded into (alpha, G) = (0, 0) so the gradient arithmetic
// needs no per-pixel branch, and G uses ex2.approx -- the skip decision alpha < 1/255 still equals the forward's
// (which uses libdevice expf) because evaluations within 1e-5 of the threshold are re-done with expf.
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ------------------------------------------------------------------------------------------------------
// Variant 15: variant 14 with the per-splat warp reduction deferred and batched through shared memory.
// Every staged splat with a hit costs variant 14 a warp_sum9 + finish_and_add (~90 instructions: 15 SHFL, the FSEL of
// the transposing butterfly, two REDG behind divergent writer branches) in its critical path. Here each lane instead
// stores its nine moments as one column of a per-warp buffer  part[slot][moment][lane]  (9 STS.32), and every
// BATCH_NB splats the warp sums the 9*BATCH_NB rows at once: lane l owns the row (slot l>>3, moment l&7) and sums its
// 32 entries with 8 LDS.128 + 31 FADD; the BATCH_NB moment-8 rows (sum w) are split over the 8 lanes of a slot
// (1 LDS.128 + 3 FADD each) and completed with a 3-level butterfly. The row owners then issue the nine atomics of a
// slot (moments 0..7 from 8 lanes, opacity from the first of them) into one 48-byte acc row: 2 REDG per batch.
// A slot records the stage index j of its splat (5 bits of the warp-uniform register jpack, behind a leading 1 that
// also counts the slots), so the batch is also flushed before the stage is refilled.
// Banks (4-byte words, 32 banks). A row is 32 words plus 4 of padding (BATCH_ROW = 36), so row r starts on bank 4r mod 32:
//   * column write of moment i by lane l: word (slot*9 + i)*36 + l -> bank (4*(slot*9 + i) + l) mod 32, a different
//     bank for each of the 32 lanes: conflict-free;
//   * row read: an LDS.128 is served per quarter warp (8 lanes, 128 bytes). At step k lane l reads chunk k of row
//     slot*9 + (l&7) = banks 4*(slot*9 + (l&7) + k) mod 32 .. +3; the 8 lanes of a quarter warp share the slot and have
//     distinct l&7, so distinct bank quads. The padding is what lets every lane read its chunks at the same immediate
//     offsets (no per-load address arithmetic);
//   * moment-8 read: the 8 lanes of a quarter warp are the 8 lanes of one slot and read chunks 0..7 of its row.
// Static SASS (nvcc 12.9, sm_90a): the per-splat loop is 388 instructions against 362 for variant 14, but 110 of them
// are the flush, run once per 4 splats, and 42 the rare expf re-check. A splat with hits in all four sub-blocks costs
// 236 + 110/4 = 264 instead of ~320: 14 for the write (9 STS) and 28 for its share of the flush, against ~90 for the
// warp reduction. 96 registers, 0 spills, 27392 B of shared memory per CTA (5 CTAs/SM).
// Gradients differ from variant 14 only in the order of the fp32 sums.
// ------------------------------------------------------------------------------------------------------
// DEPTH (the depth-gradient instantiation): part[slot][10][BATCH_ROW]; the moment-9 rows (sum alpha*T*dL/dD) are summed
// like the moment-8 rows, split over the 8 lanes of a slot, and go to acc slot 9 in the same REDG as the opacity.
// Rows start on bank 4*(slot*10 + i) mod 32, so the column writes and row reads stay conflict-free by the argument above.
constexpr int BATCH_NB = 4;    // slots per flush (8 slots, 43 KB per CTA, measured no faster)
constexpr int BATCH_ROW = 36;  // floats per row: 32 lanes + 4 of padding; 4 * 9 * 36 * 4 B = 5 KB per warp
template <bool DEPTH> constexpr int batch_moments() { return DEPTH ? 10 : 9; }

// Sums the nslot filled slots (warp-uniform; all lanes call it) and adds them to acc. The slots refer to the stage:
// call it before the stage is refilled.
// DET: sid[j] holds the instance's emission slot instead of the Gaussian index; the finished row of stage entry j is
// stored, not added, at rows[2*sid[j] + part] and its flag is set; the reduction kernel (deterministic.cu) adds the rows
// of each Gaussian.
template <bool DEPTH = false, bool DET = false>
__device__ __forceinline__ void flush_moments(const float4* part4, uint32_t jpack, int nslot, const float4 (*stg)[32],
                                              const uint32_t* sid, float* acc, int lane, float ddelx_dx,
                                              float ddely_dy, float* rows = nullptr, uint8_t* flags = nullptr,
                                              int part = 0) {
  constexpr int NM = batch_moments<DEPTH>();
  const unsigned F = 0xffffffffu;
  const int s = lane >> 3, m = lane & 7;  // this lane's slot and moment row
  const float4* row = part4 + (s * NM + m) * (BATCH_ROW / 4);
  float4 t = row[0];
#pragma unroll
  for (int k = 1; k < 8; k++) {
    const float4 v = row[k];
    t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
  }
  const float tot = (t.x + t.y) + (t.z + t.w);
  const float4 v8 = part4[(s * NM + 8) * (BATCH_ROW / 4) + m];  // chunk m of the slot's moment-8 row
  float sw = (v8.x + v8.y) + (v8.z + v8.w);
  sw += __shfl_xor_sync(F, sw, 1);
  sw += __shfl_xor_sync(F, sw, 2);
  sw += __shfl_xor_sync(F, sw, 4);
  float sz = 0.f;  // DEPTH: the slot's sum alpha*T*dL/dD = dL/dz
  if constexpr (DEPTH) {
    const float4 v9 = part4[(s * NM + 9) * (BATCH_ROW / 4) + m];
    sz = (v9.x + v9.y) + (v9.z + v9.w);
    sz += __shfl_xor_sync(F, sz, 1);
    sz += __shfl_xor_sync(F, sz, 2);
    sz += __shfl_xor_sync(F, sz, 4);
  }
  const float other = __shfl_xor_sync(F, tot, 7);  // s_x <-> s_y between moments 3 and 4
  if (s < nslot) {
    const int j = (jpack >> (5 * (nslot - 1 - s))) & 31u;
    const float4 s0 = stg[0][j];  // x, y, A, B
    const float4 s1 = stg[1][j];  // C, o
    size_t row = 0;
    if constexpr (DET) row = (size_t)2 * sid[j] + (size_t)part;
    float* dst = DET ? rows + row * ACC_STRIDE : acc + (size_t)sid[j] * ACC_STRIDE;
    // as finish_and_add: m<3 tot | 3: -(A*s_x + B*s_y)*0.5W | 4: -(C*s_y + B*s_x)*0.5H | 5..7: -0.5*tot | opacity sw / o
    const bool is_x = m == 3, is_y = m == 4;
    const float nAx = -s0.z * ddelx_dx, nCy = -s1.x * ddely_dy, nBx = -s0.w * ddelx_dx, nBy = -s0.w * ddely_dy;
    const float ka = is_x ? nAx : (is_y ? nCy : (m < 3 ? 1.0f : -0.5f));
    const float kb = is_x ? nBx : (is_y ? nBy : 0.0f);
    // kb * other only on the two mean moments (see finish_and_add: a NaN conic moment must not reach the colour rows)
    const float v = (is_x || is_y) ? fmaf(kb, other, ka * tot) : ka * tot;
    if constexpr (DET) dst[m] = v;
    else atomicAdd(dst + m, v);
    if constexpr (DEPTH) {
      if (m < 2) {  // lane m = 0: opacity into slot 8, lane m = 1: dL/dz into slot 9
        float rcp;
        asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rcp) : "f"(s1.y));
        if constexpr (DET) dst[8 + m] = m == 0 ? sw * rcp : sz;
        else atomicAdd(dst + 8 + m, m == 0 ? sw * rcp : sz);
      }
    } else if (m == 0) {
      float rcp;  // o >= 1/255 for every staged splat (splat_subblock_mask): __fdividef(sw, o) without its denormal guard
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rcp) : "f"(s1.y));
      if constexpr (DET) dst[8] = sw * rcp;
      else atomicAdd(dst + 8, sw * rcp);
    }
    if constexpr (DET) {
      if (m == 0) flags[row] = 1;
    }
  }
}

// BATCHED (variant 15): the per-splat reduction is deferred and batched through shared memory (flush_moments)
// DEPTH: variant 15 with the depth channel (a.dL_ddepth, tenth moment -> acc slot 9)
// DET: variant 15 (or its DEPTH form) in deterministic mode. Mapping, staging, evaluation, skip decisions and the
// batched sum are unchanged; the staging lane computes the instance's emission slot and keeps it in sid in place of the
// Gaussian index, and the flush stores the finished row at that slot instead of adding it to acc.
// MASK: variant 15 (any of its DEPTH / DET forms) for gsr_backward_masked. The staging lane loads grad_mask of the
// instance's Gaussian and carries it in bit 31 of the staged sub-block mask (q1.w; `act` clears it again). A splat of an
// unedited Gaussian is evaluated as usual, but its hits only advance the pixel state (state_update): no column, no batch
// slot, no flush, no row or flag. The walk stops at the tile's front-most edited position (a.first), and a warp or tile
// without an edited instance in its range returns at once.
// MASKREC (with MASK): the edit bit is the record's edit word q1.w (preprocess_fwd_masked_kernel) instead of grad_mask[id],
// taken by the staging lane from the q1 it has already loaded, before q1.w becomes the sub-block mask.
template <int NSB, int MINB, bool SKIP = false, bool MASKSKIP = false, bool BATCHED = false, bool DEPTH = false,
          bool DET = false>
__global__ void __launch_bounds__(BW_WARPS * 32, MINB) render_bwd_flat_kernel(const BwdArgsT<DEPTH, DET> a, const int ntiles) {
  constexpr bool MASK = false, MASKREC = false;
#include "render_bwd_flat_body.inc"
}
// MASK form of variant 15 (gsr_backward_masked), with DEPTH / DET as render_bwd_flat_kernel. A kernel of its own name
// (not a further template parameter of render_bwd_flat_kernel), so that every existing kernel keeps its symbol.
template <int MINB, bool DEPTH, bool DET>
__global__ void __launch_bounds__(BW_WARPS * 32, MINB) render_bwd_masked_kernel(const BwdMaskArgs<BwdArgsT<DEPTH, DET>> a,
                                                                                const int ntiles) {
  constexpr int NSB = 4;
  constexpr bool SKIP = true, MASKSKIP = false, BATCHED = true, MASK = true, MASKREC = false;
#include "render_bwd_flat_body.inc"
}
// MASKREC form of render_bwd_masked_kernel for a tile owner of the Gaussian-sharded path (gsr_shard_backward_render_masked):
// a list entry is a global index (dense) or a candidate slot (sparse), so no per-rank mask can be indexed by it; the
// record carries the bit instead. a.grad_mask is unused.
template <int MINB, bool DEPTH, bool DET>
__global__ void __launch_bounds__(BW_WARPS * 32, MINB) render_bwd_recmask_kernel(const BwdMaskArgs<BwdArgsT<DEPTH, DET>> a,
                                                                                 const int ntiles) {
  constexpr int NSB = 4;
  constexpr bool SKIP = true, MASKSKIP = false, BATCHED = true, MASK = true, MASKREC = true;
#include "render_bwd_flat_body.inc"
}

// ------------------------------------------------------------------------------------------------------
// Variant 0: CTA per tile, one pixel per thread, butterfly reduction of the nine sums per splat
// ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TILE_PIX) render_bwd_cta_kernel(const BwdArgs a) {
  __shared__ float4 s_q0[TILE_PIX], s_q1[TILE_PIX], s_q2[TILE_PIX];
  __shared__ uint32_t s_ids[TILE_PIX];
  const int tile = blockIdx.y * a.gx + blockIdx.x;
  const int tid = threadIdx.y * TILE + threadIdx.x;
  const int lane = tid & 31;
  const uint2 pix = make_uint2(blockIdx.x * TILE + threadIdx.x, blockIdx.y * TILE + threadIdx.y);
  const bool inside = pix.x < (unsigned)a.W && pix.y < (unsigned)a.H;
  const size_t pix_id = (size_t)a.W * pix.y + pix.x;
  const float2 pixf = make_float2((float)pix.x, (float)pix.y);
  const uint2 range = a.ranges[tile];
  const int tl = (int)a.tile_last[tile];  // block-uniform
  const size_t HW = (size_t)a.H * a.W;

  PixState p;
  p.T = 0.f; p.ar = 0.f; p.d0 = p.d1 = p.d2 = 0.f; p.bgT = 0.f;
  uint32_t nc = 0;
  if (inside) {
    const float Tf = a.final_T[pix_id];
    p.T = Tf;
    p.d0 = a.dL_dpix[pix_id]; p.d1 = a.dL_dpix[HW + pix_id]; p.d2 = a.dL_dpix[2 * HW + pix_id];
    p.bgT = Tf * bg_term(a, pix_id, a.bg[0], a.bg[1], a.bg[2], p);
    nc = a.n_contrib[pix_id];
  }
  const float ddelx_dx = 0.5f * a.W, ddely_dy = 0.5f * a.H;
  const LaneRole role = lane_role(lane);

  for (int hi = tl; hi > 0; hi -= TILE_PIX) {
    __syncthreads();
    const int pos = hi - tid;
    if (pos >= 1) {
      const uint32_t id = a.point_list[range.x + pos - 1];
      const float4* r = reinterpret_cast<const float4*>(a.records + id);
      s_q0[tid] = __ldg(r); s_q1[tid] = __ldg(r + 1); s_q2[tid] = __ldg(r + 2);
      s_ids[tid] = id;
    }
    __syncthreads();
    const int n = min(TILE_PIX, hi);
    for (int j = 0; j < n; j++) {
      const uint32_t spos = (uint32_t)(hi - j);
      const float4 q0 = s_q0[j], q1 = s_q1[j];
      const float dx = q0.x - pixf.x, dy = q0.y - pixf.y;
      const float power = splat_power(dx, dy, q0.z, q0.w, q1.x);
      float g[9];
#pragma unroll
      for (int i = 0; i < 9; i++) g[i] = 0.f;
      bool hit = false;
      if (!(power > 0.0f) && spos <= nc) {
        const float G = expf(power);
        const float alpha = fminf(0.99f, __fmul_rn(q1.y, G));
        if (!(alpha < 1.0f / 255.0f)) {
          hit = true;
          const float4 q2 = s_q2[j];
          hit_update(p, g, dx, dy, G, alpha, q1.y, q2.x, q2.y, q2.z);
        }
      }
      if (__any_sync(0xffffffffu, hit)) {
        float m8;
        const float tot = warp_sum9(g, lane, m8);
        finish_and_add(a.acc + (size_t)s_ids[j] * ACC_STRIDE, tot, m8, role, q0.z, q0.w, q1.x, q1.y, ddelx_dx, ddely_dy);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------
// Masked backward: where each tile's walk may stop. One warp per tile scans the list front to back in chunks of 32,
// positions [0, min(tile_last, list length)), loads grad_mask of each instance's Gaussian and takes a ballot:
// first[tile] = 1-based position of the first edited instance, GRAD_MASK_NONE when there is none. At most 4 + 1 bytes
// per walked instance, and a tile stops reading at its first edited instance.
// ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BW_WARPS * 32) grad_mask_first_kernel(const uint2* __restrict__ ranges,
                                                                        const uint32_t* __restrict__ point_list,
                                                                        const uint32_t* __restrict__ tile_last,
                                                                        const uint8_t* __restrict__ grad_mask,
                                                                        uint32_t* __restrict__ first, int ntiles) {
  const int lane = threadIdx.x & 31;
  const int tile = blockIdx.x * BW_WARPS + (threadIdx.x >> 5);
  if (tile >= ntiles) return;
  const uint2 range = ranges[tile];
  const uint32_t n = min(tile_last[tile], range.y > range.x ? range.y - range.x : 0u);
  uint32_t f = GRAD_MASK_NONE;
  for (uint32_t b = 0; b < n; b += 32) {
    const uint32_t i = b + lane;
    const bool e = i < n && __ldg(grad_mask + __ldg(point_list + range.x + i)) != 0;
    const uint32_t hit = __ballot_sync(0xffffffffu, e);
    if (hit) {
      f = b + (uint32_t)__ffs(hit);  // __ffs is 1-based: the 1-based position
      break;
    }
  }
  if (lane == 0) first[tile] = f;
}

// grad_mask_first_kernel for a tile owner of the Gaussian-sharded path: warp n walks the n-th OWNED tile (owned_tile, as
// the masked walk reads first[]), and an instance is edited when its record's edit word q1.w is nonzero. The entries of
// the tiles this rank does not own are neither read nor written.
__global__ void __launch_bounds__(BW_WARPS * 32) grad_mask_first_owner_kernel(const uint2* __restrict__ ranges,
                                                                              const uint32_t* __restrict__ point_list,
                                                                              const uint32_t* __restrict__ tile_last,
                                                                              const SplatRecord* __restrict__ records,
                                                                              uint32_t* __restrict__ first, int ntiles,
                                                                              int gx, int own_stride, int own_phase) {
  const int lane = threadIdx.x & 31;
  const int n_own = blockIdx.x * BW_WARPS + (threadIdx.x >> 5);
  if (n_own >= ntiles) return;
  const int tile = owned_tile(n_own, gx, own_stride, own_phase);
  const uint2 range = ranges[tile];
  const uint32_t n = min(tile_last[tile], range.y > range.x ? range.y - range.x : 0u);
  uint32_t f = GRAD_MASK_NONE;
  for (uint32_t b = 0; b < n; b += 32) {
    const uint32_t i = b + lane;
    const bool e = i < n && __float_as_uint(__ldg(&records[__ldg(point_list + range.x + i)].q1.w)) != 0;
    const uint32_t hit = __ballot_sync(0xffffffffu, e);
    if (hit) {
      f = b + (uint32_t)__ffs(hit);
      break;
    }
  }
  if (lane == 0) first[tile] = f;
}

}  // namespace

size_t grad_mask_first_bytes(int W, int H) {
  const size_t ntiles = (size_t)((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
  return align_up((ntiles > 0 ? ntiles : 1) * sizeof(uint32_t));
}

// one MASK instantiation of variant 15: edit bits from grad_mask (single GPU) or from the records (gm.mask == null)
template <int MINB, bool DEPTH, bool DET>
static void launch_masked_form(const BwdMaskArgs<BwdArgsT<DEPTH, DET>>& ma, int blocks, int ntiles, cudaStream_t st) {
  if (ma.grad_mask != nullptr)
    render_bwd_masked_kernel<MINB, DEPTH, DET><<<blocks, BW_WARPS * 32, 0, st>>>(ma, ntiles);
  else
    render_bwd_recmask_kernel<MINB, DEPTH, DET><<<blocks, BW_WARPS * 32, 0, st>>>(ma, ntiles);
}

// The masked walk: first[] of every (owned) tile, then one of the four MASK instantiations of variant 15. 4 CTAs/SM for
// all four except the atomic colour kernel, which keeps the default's 5 (see DESIGN.md section 3 for the register counts).
// gm.mask == null: a tile owner of the sharded path, whose edit bits are the records' edit words.
static int launch_render_bwd_masked(const BwdArgs& a, int ntiles, const float* dL_ddepth, const DetWS* det,
                                    const GradMaskWS& gm, bool debug, cudaStream_t st) {
  if (gm.mask != nullptr)
    grad_mask_first_kernel<<<(ntiles + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(
        a.ranges, a.point_list, a.tile_last, gm.mask, gm.first, ntiles);
  else
    grad_mask_first_owner_kernel<<<(ntiles + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(
        a.ranges, a.point_list, a.tile_last, a.records, gm.first, ntiles, a.gx, a.own_stride, a.own_phase);
  g_launches++;
  int rc = check_launch("grad_mask_first", debug, st);
  if (rc) return rc;
  const int blocks = (ntiles * 2 + BW_WARPS - 1) / BW_WARPS;
  auto fill = [&](auto& ma) {
    ma.grad_mask = gm.mask;
    ma.first = gm.first;
  };
  if (det != nullptr) {
    if (dL_ddepth != nullptr) {
      BwdMaskArgs<BwdDetArgs<BwdDepthArgs>> ma;
      static_cast<BwdArgs&>(ma) = a;
      ma.dL_ddepth = dL_ddepth;
      ma.excl = det->excl; ma.rows = det->rows; ma.flags = det->flags;
      fill(ma);
      launch_masked_form<4, true, true>(ma, blocks, ntiles, st);
    } else {
      BwdMaskArgs<BwdDetArgs<BwdArgs>> ma;
      static_cast<BwdArgs&>(ma) = a;
      ma.excl = det->excl; ma.rows = det->rows; ma.flags = det->flags;
      fill(ma);
      launch_masked_form<4, false, true>(ma, blocks, ntiles, st);
    }
  } else if (dL_ddepth != nullptr) {
    BwdMaskArgs<BwdDepthArgs> ma;
    static_cast<BwdArgs&>(ma) = a;
    ma.dL_ddepth = dL_ddepth;
    fill(ma);
    launch_masked_form<4, true, false>(ma, blocks, ntiles, st);
  } else {
    BwdMaskArgs<BwdArgs> ma;
    static_cast<BwdArgs&>(ma) = a;
    fill(ma);
    launch_masked_form<5, false, false>(ma, blocks, ntiles, st);
  }
  g_launches++;
  return check_launch("render_bwd (masked)", debug, st);
}

int launch_render_bwd(const gsr_settings& s, const GeometryWS& g, const BinningWS& b, const ImageWS& im,
                      const float* dL_dpix, float* acc, cudaStream_t st, const TileOwner& own,
                      const float* dL_dalpha_img, const float* dL_ddepth, const DetWS* det, int P, int64_t R,
                      const GradMaskWS* gm) {
  BwdArgs a;
  a.dL_dalpha_img = dL_dalpha_img;
  a.own_stride = own.stride; a.own_phase = own.phase;
  a.ranges = im.ranges; a.point_list = b.point_list; a.records = g.records; a.tile_last = im.tile_last;
  a.W = s.image_width; a.H = s.image_height;
  a.gx = (a.W + TILE - 1) / TILE; a.gy = (a.H + TILE - 1) / TILE;
  a.bg = s.bg; a.final_T = im.final_T; a.n_contrib = im.n_contrib; a.dL_dpix = dL_dpix; a.acc = acc;
  const int ntiles = a.gx * own.owned_rows(a.gy);  // tiles this rank walks (all of them when own = {1,0})
  if (ntiles == 0) return GSR_OK;
  if (gm != nullptr) {  // masked backward: variant 15, atomic or deterministic
    int rc = det ? launch_det_prepare(P, R, 2, g, *det, st) : GSR_OK;
    if (rc) return rc;
    if ((rc = launch_render_bwd_masked(a, ntiles, dL_ddepth, det, *gm, s.debug != 0, st))) return rc;
    return det ? launch_det_reduce_acc(P, dL_ddepth != nullptr, g, *det, acc, st) : GSR_OK;
  }
  if (det != nullptr) {  // deterministic mode: variant 15 (or its depth form) writes rows, one kernel reduces them
    int rc = launch_det_prepare(P, R, 2, g, *det, st);
    if (rc) return rc;
    const int blocks = (ntiles * 2 + BW_WARPS - 1) / BW_WARPS;
    // 4 CTAs/SM for both: at 5 (96 registers) the colour-only DET kernel spills 8 bytes, as the depth kernel did 20
    if (dL_ddepth != nullptr) {
      BwdDetArgs<BwdDepthArgs> da;
      static_cast<BwdArgs&>(da) = a;
      da.dL_ddepth = dL_ddepth;
      da.excl = det->excl; da.rows = det->rows; da.flags = det->flags;
      render_bwd_flat_kernel<4, 4, true, false, true, true, true><<<blocks, BW_WARPS * 32, 0, st>>>(da, ntiles);
    } else {
      BwdDetArgs<BwdArgs> da;
      static_cast<BwdArgs&>(da) = a;
      da.excl = det->excl; da.rows = det->rows; da.flags = det->flags;
      render_bwd_flat_kernel<4, 4, true, false, true, false, true><<<blocks, BW_WARPS * 32, 0, st>>>(da, ntiles);
    }
    g_launches++;
    if ((rc = check_launch("render_bwd", s.debug != 0, st))) return rc;
    return launch_det_reduce_acc(P, dL_ddepth != nullptr, g, *det, acc, st);
  }
  int v = g_opt.render_bwd_variant;
  if (v == 0 && own.stride != 1) v = 4;  // the CTA-per-tile kernel maps blockIdx to tiles directly: single-GPU only
  if (dL_ddepth != nullptr) {  // the depth channel exists only in variant 15, whatever the option says. At 5 CTAs/SM
    // (96 registers) it spills 20 bytes; at 4 CTAs/SM it does not.
    BwdDepthArgs da;
    static_cast<BwdArgs&>(da) = a;
    da.dL_ddepth = dL_ddepth;
    render_bwd_flat_kernel<4, 4, true, false, true, true><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(da, ntiles);
  } else if (v == 0) {
    render_bwd_cta_kernel<<<dim3(a.gx, a.gy), dim3(TILE, TILE), 0, st>>>(a);
  } else if (v == 2) {
    const int warps = ntiles * 2;
    render_bwd_warp_kernel<4><<<(warps + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 3) {
    const int warps = ntiles * 4;
    render_bwd_warp_kernel<2><<<(warps + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 4) {
    render_bwd_flat_kernel<4, 1><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 5) {
    render_bwd_flat_kernel<4, 6><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 6) {
    render_bwd_flat_kernel<2, 1><<<(ntiles * 4 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 7) {
    render_bwd_flat_kernel<8, 1><<<(ntiles + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 8) {
    render_bwd_flat_kernel<4, 1, true><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 9) {
    render_bwd_flat_kernel<8, 1, true><<<(ntiles + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 12) {  // register caps: 5 / 6 CTAs per SM, with and without the hit-skip
    render_bwd_flat_kernel<4, 5><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 13) {
    render_bwd_flat_kernel<4, 6, true><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 14) {
    render_bwd_flat_kernel<4, 5, true><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 15) {  // variant 14 with the per-splat reduction batched through shared memory
    render_bwd_flat_kernel<4, 5, true, false, true><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 10) {  // variant 4 + sub-blocks outside the splat's mask skipped with warp-uniform branches
    render_bwd_flat_kernel<4, 1, false, true><<<(ntiles * 2 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else if (v == 11) {  // the same for the quarter-tile mapping
    render_bwd_flat_kernel<2, 1, false, true><<<(ntiles * 4 + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  } else {
    render_bwd_warp_kernel<8><<<(ntiles + BW_WARPS - 1) / BW_WARPS, BW_WARPS * 32, 0, st>>>(a, ntiles);
  }
  g_launches++;
  return check_launch("render_bwd", s.debug != 0, st);
}

}  // namespace gsr
