// Masked Adam for sm_90a: one optimizer step over every parameter group of a Gaussian cloud, restricted to the rows
// under edit (gsr_adam_masked, include/gsr_b200.h).
//
// Mapping: warp w owns rows [32w, 32w + 32) of every group. Its lanes read the 32 mask bytes and ballot them; a span
// without an edited row costs that one 32-byte read and nothing else. Otherwise the warp walks each group's
// 32 * D floats of the span with a lane stride (coalesced), and a lane touches element e only when its row e / D is
// edited: the loads of an unedited row are never issued, so its sectors are not fetched, and it is never stored.
// Reading the mask once per span for all groups (rather than once per (group, span)) keeps the mask traffic at P
// bytes. Each lane batches ADAM_UNROLL elements, all loads before any arithmetic, to keep 16 loads in flight.
// No shared memory, no atomics, no host synchronisation: a step can be captured in a CUDA graph.
#include <cmath>

#include "common.cuh"

namespace gsr {

namespace {

constexpr int ADAM_THREADS = 256;
constexpr int ADAM_UNROLL = 4;

struct AdamGroupDev {
  float* p;
  const float* g;
  float* m;
  float* v;
  float* step;  // capturable: device step (already advanced by adam_step_kernel), else nullptr
  int D;
  float omb1, b1, b2, omb2, eps, lr;  // omb = 1 - beta, rounded from double as torch passes Python scalars
  float step_size, bc2_sqrt;          // host-computed (step == nullptr)
};

struct AdamArgs {
  AdamGroupDev grp[GSR_ADAM_MAX_GROUPS];
  const uint8_t* mask;
  int n, P;
};

// capturable: every group's device step advances once, before the update reads it
__global__ void adam_step_kernel(const __grid_constant__ AdamArgs a) {
  const int i = threadIdx.x;
  if (i < a.n && a.grp[i].step) a.grp[i].step[0] += 1.f;
}

__global__ void __launch_bounds__(ADAM_THREADS) adam_masked_kernel(const __grid_constant__ AdamArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t row0 = (int64_t)blockIdx.x * ADAM_THREADS + (threadIdx.x & ~31);
  if (row0 >= a.P) return;  // warp-uniform
  const int rows = a.P - row0 < 32 ? (int)(a.P - row0) : 32;
  const unsigned edited = __ballot_sync(0xffffffffu, lane < rows && __ldg(a.mask + row0 + lane) != 0);
  if (!edited) return;
  for (int gi = 0; gi < a.n; gi++) {
    const AdamGroupDev& G = a.grp[gi];
    const int D = G.D;
    if (D == 0) continue;
    float step_size = G.step_size, bc2_sqrt = G.bc2_sqrt;
    if (G.step) {  // _multi_tensor_adam(capturable=True): step_size = 1 / ((beta1^t - 1) / lr) negated
      const float t = *G.step;
      step_size = -(1.f / ((powf(G.b1, t) - 1.f) / G.lr));
      bc2_sqrt = sqrtf(-(powf(G.b2, t) - 1.f));
    }
    const size_t base = (size_t)row0 * (size_t)D;  // 64-bit: P * D passes 2^31 for f_rest at 48M Gaussians
    float* __restrict__ p = G.p + base;
    const float* __restrict__ g = G.g + base;
    float* __restrict__ m = G.m + base;
    float* __restrict__ v = G.v + base;
    const unsigned n = (unsigned)rows * (unsigned)D;  // < 2^29: D <= GSR_ADAM_MAX_D
    for (unsigned e0 = lane; e0 < n; e0 += 32 * ADAM_UNROLL) {
      float gv[ADAM_UNROLL], mv[ADAM_UNROLL], vv[ADAM_UNROLL], pv[ADAM_UNROLL];
      bool on[ADAM_UNROLL];
#pragma unroll
      for (int u = 0; u < ADAM_UNROLL; u++) {
        const unsigned e = e0 + 32u * u;
        on[u] = e < n && ((edited >> (e / (unsigned)D)) & 1u);
        if (on[u]) {
          gv[u] = __ldcs(g + e);
          mv[u] = m[e];
          vv[u] = v[e];
          pv[u] = p[e];
        }
      }
#pragma unroll
      for (int u = 0; u < ADAM_UNROLL; u++) {
        if (!on[u]) continue;
        const unsigned e = e0 + 32u * u;
        const float gr = gv[u];
        const float mn = mv[u] + G.omb1 * (gr - mv[u]);                      // lerp(m, g, 1 - beta1), weight < 0.5
        const float vn = fmaf(G.omb2, __fmul_rn(gr, gr), __fmul_rn(vv[u], G.b2));  // mul_(beta2), addcmul_(g, g)
        const float den = __fadd_rn(__fdiv_rn(sqrtf(vn), bc2_sqrt), G.eps);
        m[e] = mn;
        v[e] = vn;
        p[e] = pv[u] - step_size * __fdiv_rn(mn, den);
      }
    }
  }
}

}  // namespace

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_adam_masked(const gsr_adam_group* groups, int32_t n_groups, int32_t P, const uint8_t* mask, void* stream) {
  if (n_groups < 1 || n_groups > GSR_ADAM_MAX_GROUPS) {
    set_error("gsr_adam_masked: n_groups = %d outside [1, %d]", n_groups, GSR_ADAM_MAX_GROUPS);
    return GSR_ERR_INVALID;
  }
  if (!groups) { set_error("gsr_adam_masked: groups is null"); return GSR_ERR_INVALID; }
  if (!mask) { set_error("gsr_adam_masked: mask is null"); return GSR_ERR_INVALID; }
  if (P < 0) { set_error("gsr_adam_masked: P = %d < 0", P); return GSR_ERR_INVALID; }
  AdamArgs a{};
  a.mask = mask;
  a.n = n_groups;
  a.P = P;
  bool any_step = false;
  for (int i = 0; i < n_groups; i++) {
    const gsr_adam_group& G = groups[i];
    if (G.D < 0 || G.D > GSR_ADAM_MAX_D) {
      set_error("gsr_adam_masked: group %d has D = %d outside [0, %d]", i, G.D, GSR_ADAM_MAX_D);
      return GSR_ERR_INVALID;
    }
    if ((int64_t)P * G.D > 0 && (!G.p || !G.g || !G.m || !G.v)) {
      set_error("gsr_adam_masked: group %d has a null p, g, m or v", i);
      return GSR_ERR_INVALID;
    }
    if (!(G.beta1 >= 0.0 && G.beta1 < 1.0) || !(G.beta2 >= 0.0 && G.beta2 < 1.0)) {
      set_error("gsr_adam_masked: group %d has beta1 = %g, beta2 = %g outside [0, 1)", i, G.beta1, G.beta2);
      return GSR_ERR_INVALID;
    }
    if (!(G.eps >= 0.0)) { set_error("gsr_adam_masked: group %d has eps = %g < 0", i, G.eps); return GSR_ERR_INVALID; }
    if (!G.step_dev && !(G.step >= 1.0)) {
      set_error("gsr_adam_masked: group %d has step = %g < 1 and no device step", i, G.step);
      return GSR_ERR_INVALID;
    }
    AdamGroupDev& d = a.grp[i];
    d.p = G.p; d.g = G.g; d.m = G.m; d.v = G.v; d.step = G.step_dev;
    d.D = (int)G.D;
    d.omb1 = (float)(1.0 - G.beta1);
    d.b1 = (float)G.beta1;
    d.b2 = (float)G.beta2;
    d.omb2 = (float)(1.0 - G.beta2);
    d.eps = (float)G.eps;
    d.lr = (float)G.lr;
    if (!G.step_dev) {  // torch's CPU-step path: Python doubles lr / (1 - beta1**t) and (1 - beta2**t)**0.5
      d.step_size = (float)(G.lr / (1.0 - std::pow(G.beta1, G.step)));
      d.bc2_sqrt = (float)std::pow(1.0 - std::pow(G.beta2, G.step), 0.5);
    }
    any_step |= G.step_dev != nullptr;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (any_step) {
    adam_step_kernel<<<1, 32, 0, st>>>(a);
    g_launches++;
    if (int rc = check_launch("adam_step", false, st)) return rc;
  }
  if (P == 0) return GSR_OK;
  const unsigned blocks = (unsigned)(((int64_t)P + ADAM_THREADS - 1) / ADAM_THREADS);
  adam_masked_kernel<<<blocks, ADAM_THREADS, 0, st>>>(a);
  g_launches++;
  return check_launch("adam_masked", false, st);
}

}  // extern "C"
