// Anchor loss for sm_90a: GaussianEditor's per-step "hierarchical" regularizer (GaussianModel.anchor_loss), forward and
// backward (gsr_anchor_loss_forward / gsr_anchor_loss_backward, include/gsr_b200.h).
//
//   w_i = schedule[generation[i]]                      (NaN when the generation is outside [0, n_schedule))
//   L_k = sum over edited rows i and j < D_k of w_i * (p_k[i, j] - a_k[i, j])^2  /  (N_m * D_k)
//   out = (L_dc + L_rest, L_xyz + L_rot, L_opacity, L_scale)
//
// Mapping (that of masked_adam.cu): warp w owns rows [32w, 32w + 32) of every term. Its lanes read the span's 32 mask
// bytes and ballot them; a span without an edited row costs that one 32-byte read in the forward and a vectorised zero
// store per term in the backward. Otherwise lane i loads the weight of row row0 + i, and the warp walks each term's
// 32 * D contiguous floats with a lane stride: a lane at element e takes its row's weight from lane e / D with a
// shuffle, and reads p and a only when that row is edited.
//
// The forward accumulates in fp64 per lane, reduces warp and block in a fixed order into per-block partials, and a
// one-CTA kernel sums the partials in a fixed order. The grid depends on P only and nothing is accumulated with
// atomics, so the result is bit-reproducible. The edited-row count N_m stays on the device (scratch header) for the
// backward. No host synchronisation: forward and backward can be captured in a CUDA graph.
#include <cstdint>

#include "common.cuh"

namespace gsr {

namespace {

constexpr int ANCHOR_THREADS = 256;
constexpr int ANCHOR_WARPS = ANCHOR_THREADS / 32;
constexpr int ANCHOR_UNROLL = 4;
constexpr int ANCHOR_FWD_MAX_BLOCKS = 1024;   // forward grid-strides beyond this: the finish kernel reads <= 1024 rows
constexpr int ANCHOR_SLOTS = 8;               // doubles per partial row: six term sums, the edited-row count, padding
constexpr int ANCHOR_FINISH_THREADS = 256;

struct AnchorTermDev {
  const float* p;
  const float* a;
  float* g;
  int D;
  int group;   // index into out4 / grad_out4
};

struct AnchorArgs {
  AnchorTermDev t[GSR_ANCHOR_TERMS];
  const uint8_t* mask;
  const int64_t* gen;
  const float* sched;
  int n_sched;
  int P;
  double* scratch;        // [ANCHOR_SLOTS] header (N_m at [0]), then [blocks][ANCHOR_SLOTS] partials
  int fwd_blocks;
  float* out;             // forward
  const float* grad_out;  // backward
};

// term -> group of out4 = (color, geo, opacity, scale), for the terms in GaussianModel.update_anchor's order
constexpr int kGroupOfTerm[GSR_ANCHOR_TERMS] = {1, 0, 0, 3, 1, 2};

int fwd_blocks(int32_t P) {
  const int64_t b = ((int64_t)P + ANCHOR_THREADS - 1) / ANCHOR_THREADS;
  return b < 1 ? 1 : (b > ANCHOR_FWD_MAX_BLOCKS ? ANCHOR_FWD_MAX_BLOCKS : (int)b);
}

__device__ __forceinline__ float row_weight(const AnchorArgs& a, int64_t row) {
  const int64_t g = __ldg(a.gen + row);
  // torch.gather would trap on an out-of-range index; a NaN weight poisons the loss instead
  return (g >= 0 && g < a.n_sched) ? __ldg(a.sched + g) : __int_as_float(0x7fc00000);
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(ANCHOR_THREADS) anchor_fwd_kernel(const __grid_constant__ AnchorArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc[GSR_ANCHOR_TERMS];
#pragma unroll
  for (int k = 0; k < GSR_ANCHOR_TERMS; k++) acc[k] = 0.0;
  int count = 0;
  const int64_t stride = (int64_t)gridDim.x * ANCHOR_THREADS;
  for (int64_t row0 = (int64_t)blockIdx.x * ANCHOR_THREADS + warp * 32; row0 < a.P; row0 += stride) {
    const int rows = a.P - row0 < 32 ? (int)(a.P - row0) : 32;
    const bool on = lane < rows && __ldg(a.mask + row0 + lane) != 0;
    const unsigned edited = __ballot_sync(0xffffffffu, on);
    if (!edited) continue;
    count += __popc(edited);
    const float w = on ? row_weight(a, row0 + lane) : 0.f;
#pragma unroll
    for (int k = 0; k < GSR_ANCHOR_TERMS; k++) {   // unrolled: acc[] stays in registers
      const unsigned D = (unsigned)a.t[k].D;
      if (D == 0) continue;
      const size_t base = (size_t)row0 * D;   // 64-bit: P * D passes 2^31 for f_rest at 48M Gaussians
      const float* __restrict__ p = a.t[k].p + base;
      const float* __restrict__ q = a.t[k].a + base;
      const unsigned n = (unsigned)rows * D;   // < 2^29: D <= GSR_ADAM_MAX_D
      double s = 0.0;
      for (unsigned e0 = lane; e0 - lane < n; e0 += 32 * ANCHOR_UNROLL) {
        float pv[ANCHOR_UNROLL], qv[ANCHOR_UNROLL], wv[ANCHOR_UNROLL];
        bool use[ANCHOR_UNROLL];
#pragma unroll
        for (int u = 0; u < ANCHOR_UNROLL; u++) {
          const unsigned e = e0 + 32u * u;
          const unsigned r = (e < n ? e : n - 1) / D;
          wv[u] = __shfl_sync(0xffffffffu, w, r);
          use[u] = e < n && ((edited >> r) & 1u);
          if (use[u]) {
            pv[u] = __ldg(p + e);
            qv[u] = __ldg(q + e);
          }
        }
#pragma unroll
        for (int u = 0; u < ANCHOR_UNROLL; u++) {
          if (!use[u]) continue;
          const double d = (double)pv[u] - (double)qv[u];
          s = fma((double)wv[u] * d, d, s);
        }
      }
      acc[k] += s;
    }
  }
  __shared__ double red[ANCHOR_WARPS][ANCHOR_SLOTS];
#pragma unroll
  for (int k = 0; k < GSR_ANCHOR_TERMS; k++) {
    const double v = warp_sum(acc[k]);
    if (lane == 0) red[warp][k] = v;
  }
  if (lane == 0) red[warp][GSR_ANCHOR_TERMS] = (double)count;   // every lane holds the warp's count
  __syncthreads();
  if (threadIdx.x < GSR_ANCHOR_TERMS + 1) {
    double v = 0.0;
    for (int i = 0; i < ANCHOR_WARPS; i++) v += red[i][threadIdx.x];
    a.scratch[ANCHOR_SLOTS * (1 + (int64_t)blockIdx.x) + threadIdx.x] = v;
  }
}

__global__ void __launch_bounds__(ANCHOR_FINISH_THREADS) anchor_finish_kernel(const __grid_constant__ AnchorArgs a) {
  __shared__ double red[GSR_ANCHOR_TERMS + 1][ANCHOR_FINISH_THREADS];
  const int tid = threadIdx.x;
  const double* part = a.scratch + ANCHOR_SLOTS;
  for (int k = 0; k <= GSR_ANCHOR_TERMS; k++) {
    double v = 0.0;
    for (int b = tid; b < a.fwd_blocks; b += ANCHOR_FINISH_THREADS) v += part[(int64_t)b * ANCHOR_SLOTS + k];
    red[k][tid] = v;
  }
  for (int s = ANCHOR_FINISH_THREADS / 2; s > 0; s >>= 1) {
    __syncthreads();
    if (tid < s)
      for (int k = 0; k <= GSR_ANCHOR_TERMS; k++) red[k][tid] += red[k][tid + s];
  }
  if (tid != 0) return;
  const double N = red[GSR_ANCHOR_TERMS][0];
  float L[GSR_ANCHOR_TERMS];
#pragma unroll
  for (int k = 0; k < GSR_ANCHOR_TERMS; k++)   // mean of an empty term (N_m == 0 or D == 0) is 0 / 0 = NaN, as torch's
    L[k] = (float)(red[k][0] / (N * (double)a.t[k].D));
  // the groups add in fp32, as the reference's dict entries do (kGroupOfTerm)
  a.out[0] = __fadd_rn(L[1], L[2]);   // color = dc + rest
  a.out[1] = __fadd_rn(L[0], L[4]);   // geo = xyz + rotation
  a.out[2] = L[5];                    // opacity
  a.out[3] = L[3];                    // scale
  a.scratch[0] = N;
}

__device__ __forceinline__ void zero_span(float* __restrict__ g, unsigned n, int lane) {
  unsigned done = 0;
  if ((reinterpret_cast<uintptr_t>(g) & 15u) == 0) {
    float4* g4 = reinterpret_cast<float4*>(g);
    const unsigned n4 = n >> 2;
    for (unsigned i = lane; i < n4; i += 32) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    done = n4 << 2;
  }
  for (unsigned e = done + lane; e < n; e += 32) g[e] = 0.f;
}

__global__ void __launch_bounds__(ANCHOR_THREADS) anchor_bwd_kernel(const __grid_constant__ AnchorArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t row0 = (int64_t)blockIdx.x * ANCHOR_THREADS + (threadIdx.x & ~31);
  if (row0 >= a.P) return;   // warp-uniform
  const int rows = a.P - row0 < 32 ? (int)(a.P - row0) : 32;
  const bool on = lane < rows && __ldg(a.mask + row0 + lane) != 0;
  const unsigned edited = __ballot_sync(0xffffffffu, on);
  const float w = on ? row_weight(a, row0 + lane) : 0.f;
  const double N = edited ? a.scratch[0] : 0.0;
#pragma unroll 1
  for (int k = 0; k < GSR_ANCHOR_TERMS; k++) {
    const unsigned D = (unsigned)a.t[k].D;
    if (D == 0) continue;
    const size_t base = (size_t)row0 * D;
    float* __restrict__ g = a.t[k].g + base;
    const unsigned n = (unsigned)rows * D;
    if (!edited) {
      zero_span(g, n, lane);
      continue;
    }
    const float* __restrict__ p = a.t[k].p + base;
    const float* __restrict__ q = a.t[k].a + base;
    // torch: mean backward go / numel, times w (the in-place weight), then mse backward (p - a) * 2 * grad
    const float c = __fdiv_rn(__ldg(a.grad_out + a.t[k].group), (float)(N * (double)D));
    for (unsigned e0 = lane; e0 - lane < n; e0 += 32 * ANCHOR_UNROLL) {
      float pv[ANCHOR_UNROLL], qv[ANCHOR_UNROLL], wv[ANCHOR_UNROLL];
      bool use[ANCHOR_UNROLL];
#pragma unroll
      for (int u = 0; u < ANCHOR_UNROLL; u++) {
        const unsigned e = e0 + 32u * u;
        const unsigned r = (e < n ? e : n - 1) / D;
        wv[u] = __shfl_sync(0xffffffffu, w, r);
        use[u] = e < n && ((edited >> r) & 1u);
        if (use[u]) {
          pv[u] = __ldg(p + e);
          qv[u] = __ldg(q + e);
        }
      }
#pragma unroll
      for (int u = 0; u < ANCHOR_UNROLL; u++) {
        const unsigned e = e0 + 32u * u;
        if (e >= n) continue;
        float gv = 0.f;
        if (use[u]) {
          const float d2 = __fmul_rn(__fsub_rn(pv[u], qv[u]), 2.f);
          // + 0: the boolean-index backward accumulates into zeros, which turns a -0 into +0
          gv = __fadd_rn(__fmul_rn(d2, __fmul_rn(c, wv[u])), 0.f);
        }
        g[e] = gv;
      }
    }
  }
}

int validate(const char* fn, const gsr_anchor_term* terms, int32_t P, const uint8_t* mask, const int64_t* generation,
             const float* schedule, int32_t n_schedule, bool need_g) {
  if (!terms) { set_error("%s: terms is null", fn); return GSR_ERR_INVALID; }
  if (P < 0) { set_error("%s: P = %d < 0", fn, P); return GSR_ERR_INVALID; }
  if (n_schedule < 1) { set_error("%s: n_schedule = %d < 1", fn, n_schedule); return GSR_ERR_INVALID; }
  if (!schedule) { set_error("%s: schedule is null", fn); return GSR_ERR_INVALID; }
  if (P > 0 && (!mask || !generation)) { set_error("%s: mask or generation is null", fn); return GSR_ERR_INVALID; }
  for (int k = 0; k < GSR_ANCHOR_TERMS; k++) {
    const gsr_anchor_term& T = terms[k];
    if (T.D < 0 || T.D > GSR_ADAM_MAX_D) {
      set_error("%s: term %d has D = %d outside [0, %d]", fn, k, T.D, GSR_ADAM_MAX_D);
      return GSR_ERR_INVALID;
    }
    if ((int64_t)P * T.D > 0 && (!T.p || !T.a || (need_g && !T.g))) {
      set_error("%s: term %d has a null %s", fn, k, need_g ? "p, a or g" : "p or a");
      return GSR_ERR_INVALID;
    }
  }
  return GSR_OK;
}

AnchorArgs make_args(const gsr_anchor_term* terms, int32_t P, const uint8_t* mask, const int64_t* generation,
                     const float* schedule, int32_t n_schedule, void* scratch) {
  AnchorArgs a{};
  for (int k = 0; k < GSR_ANCHOR_TERMS; k++) {
    a.t[k].p = terms[k].p;
    a.t[k].a = terms[k].a;
    a.t[k].g = terms[k].g;
    a.t[k].D = (int)terms[k].D;
    a.t[k].group = kGroupOfTerm[k];
  }
  a.mask = mask;
  a.gen = generation;
  a.sched = schedule;
  a.n_sched = n_schedule;
  a.P = P;
  a.scratch = static_cast<double*>(scratch);
  a.fwd_blocks = fwd_blocks(P);
  return a;
}

}  // namespace

}  // namespace gsr

using namespace gsr;

extern "C" {

size_t gsr_anchor_loss_scratch_bytes(int32_t P) {
  if (P < 0) P = 0;
  return sizeof(double) * ANCHOR_SLOTS * (1 + (size_t)fwd_blocks(P));
}

int gsr_anchor_loss_forward(const gsr_anchor_term* terms, int32_t P, const uint8_t* mask, const int64_t* generation,
                            const float* schedule, int32_t n_schedule, void* scratch, size_t scratch_bytes, float* out4,
                            void* stream) {
  const char* fn = "gsr_anchor_loss_forward";
  if (int rc = validate(fn, terms, P, mask, generation, schedule, n_schedule, false)) return rc;
  if (!out4) { set_error("%s: out4 is null", fn); return GSR_ERR_INVALID; }
  if (!scratch || scratch_bytes < gsr_anchor_loss_scratch_bytes(P)) {
    set_error("%s: scratch of %zu bytes, %zu needed", fn, scratch ? scratch_bytes : (size_t)0,
              gsr_anchor_loss_scratch_bytes(P));
    return GSR_ERR_INVALID;
  }
  AnchorArgs a = make_args(terms, P, mask, generation, schedule, n_schedule, scratch);
  a.out = out4;
  cudaStream_t st = (cudaStream_t)stream;
  anchor_fwd_kernel<<<a.fwd_blocks, ANCHOR_THREADS, 0, st>>>(a);
  g_launches++;
  if (int rc = check_launch("anchor_fwd", false, st)) return rc;
  anchor_finish_kernel<<<1, ANCHOR_FINISH_THREADS, 0, st>>>(a);
  g_launches++;
  return check_launch("anchor_finish", false, st);
}

int gsr_anchor_loss_backward(const gsr_anchor_term* terms, int32_t P, const uint8_t* mask, const int64_t* generation,
                             const float* schedule, int32_t n_schedule, const void* scratch, size_t scratch_bytes,
                             const float* grad_out4, void* stream) {
  const char* fn = "gsr_anchor_loss_backward";
  if (int rc = validate(fn, terms, P, mask, generation, schedule, n_schedule, true)) return rc;
  if (!grad_out4) { set_error("%s: grad_out4 is null", fn); return GSR_ERR_INVALID; }
  if (!scratch || scratch_bytes < gsr_anchor_loss_scratch_bytes(P)) {
    set_error("%s: scratch of %zu bytes, %zu needed", fn, scratch ? scratch_bytes : (size_t)0,
              gsr_anchor_loss_scratch_bytes(P));
    return GSR_ERR_INVALID;
  }
  if (P == 0) return GSR_OK;
  AnchorArgs a = make_args(terms, P, mask, generation, schedule, n_schedule, const_cast<void*>(scratch));
  a.grad_out = grad_out4;
  const unsigned blocks = (unsigned)(((int64_t)P + ANCHOR_THREADS - 1) / ANCHOR_THREADS);
  anchor_bwd_kernel<<<blocks, ANCHOR_THREADS, 0, (cudaStream_t)stream>>>(a);
  g_launches++;
  return check_launch("anchor_bwd", false, (cudaStream_t)stream);
}

}  // extern "C"
