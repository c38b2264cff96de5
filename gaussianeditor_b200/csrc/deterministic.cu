// Deterministic mode for sm_90a: the per-Gaussian reduction that replaces the float atomics of render_bwd and
// apply_weights (common.cuh: DetWS).
//
// The DET kernels store each finished (instance, tile half) row -- each instance row for apply_weights -- with plain
// stores at the instance's emission slot and set a one-byte flag; rows that no hit produced are never written. The
// slots of Gaussian g are [excl[g], excl[g] + tiles_touched[g]), so its rows are one contiguous run and
// det_reduce_kernel adds the flagged ones in a schedule that depends only on the run length:
//   * runs of at most SHORT_ROWS rows: one thread, rows in ascending slot order;
//   * longer runs: the whole warp, lane l adds rows l, l+32, ... in ascending order, then a fixed xor butterfly.
// No float atomics, and no order that depends on timing: two calls on the same inputs give the same bits.
#include "common.cuh"

namespace gsr {

namespace {

constexpr int DET_THREADS = 256;
constexpr int SHORT_ROWS = 64;

// excl[order[r]] = offsets[r] - tiles_touched[order[r]]: the inverse of the depth order folded with the exclusive scan
__global__ void __launch_bounds__(DET_THREADS) det_excl_kernel(int P, const uint32_t* __restrict__ order,
                                                               const uint32_t* __restrict__ offsets,
                                                               const uint32_t* __restrict__ tiles_touched,
                                                               uint32_t* __restrict__ excl) {
  const int r = blockIdx.x * DET_THREADS + threadIdx.x;
  if (r >= P) return;
  const uint32_t g = __ldg(order + r);
  excl[g] = __ldg(offsets + r) - __ldg(tiles_touched + g);
}

// ROWS rows per instance of STRIDE floats, the first NV of which are summed. ADD: out[g*OUT + v] += sum (only when g
// has a flagged row), else out[g*OUT + v] = sum for v < NV and 0 for NV <= v < OUT.
template <int ROWS, int STRIDE, int NV, int OUT, bool ADD>
__global__ void __launch_bounds__(DET_THREADS) det_reduce_kernel(int P, const uint32_t* __restrict__ excl,
                                                                 const uint32_t* __restrict__ tiles_touched,
                                                                 const float* __restrict__ rows,
                                                                 const uint8_t* __restrict__ flags,
                                                                 float* __restrict__ out) {
  const unsigned F = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * DET_THREADS + threadIdx.x;
  uint32_t n = 0;
  size_t b = 0;
  if (g < P) {
    n = __ldg(tiles_touched + g) * (uint32_t)ROWS;
    if (n) b = (size_t)__ldg(excl + g) * ROWS;
  }
  float s[NV];
#pragma unroll
  for (int v = 0; v < NV; v++) s[v] = 0.f;
  bool any = false;
  if (n <= (uint32_t)SHORT_ROWS) {
    for (uint32_t i = 0; i < n; i++) {
      if (!__ldg(flags + b + i)) continue;
      any = true;
      const float* row = rows + (b + i) * STRIDE;
#pragma unroll
      for (int v = 0; v < NV; v++) s[v] += __ldg(row + v);
    }
  }
  // long runs, one at a time in lane order, by the whole warp
  uint32_t longs = __ballot_sync(F, n > (uint32_t)SHORT_ROWS);
  while (longs) {
    const int src = __ffs(longs) - 1;
    longs &= longs - 1;
    const uint32_t ln = __shfl_sync(F, n, src);
    const size_t lb = ((size_t)__shfl_sync(F, (uint32_t)(b >> 32), src) << 32) | __shfl_sync(F, (uint32_t)b, src);
    float t[NV];
#pragma unroll
    for (int v = 0; v < NV; v++) t[v] = 0.f;
    bool la = false;
    for (uint32_t i = lane; i < ln; i += 32) {
      if (!__ldg(flags + lb + i)) continue;
      la = true;
      const float* row = rows + (lb + i) * STRIDE;
#pragma unroll
      for (int v = 0; v < NV; v++) t[v] += __ldg(row + v);
    }
#pragma unroll
    for (int v = 0; v < NV; v++) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t[v] += __shfl_xor_sync(F, t[v], o);
    }
    la = __any_sync(F, la);
    if (lane == src) {
      any = la;
#pragma unroll
      for (int v = 0; v < NV; v++) s[v] = t[v];
    }
  }
  if (g >= P) return;
  float* o = out + (size_t)g * OUT;
  if constexpr (ADD) {
    if (any) {
#pragma unroll
      for (int v = 0; v < NV; v++) o[v] += s[v];
    }
  } else {
#pragma unroll
    for (int v = 0; v < OUT; v++) o[v] = v < NV ? s[v] : 0.f;
  }
}

}  // namespace

bool carve_det(void* base, int P, int64_t R, int CH, DetWS& ws) {
  if (P < 0 || R < 0 || CH < 0) return false;
  const size_t rows_bwd = (size_t)R * 2 * ACC_STRIDE * sizeof(float);
  const size_t rows_aw = (size_t)R * (size_t)CH * sizeof(float);
  const size_t e = align_up((size_t)(P > 0 ? P : 1) * sizeof(uint32_t));
  const size_t f = align_up((size_t)(R > 0 ? 2 * R : 1));
  const size_t r = align_up(rows_bwd > rows_aw ? rows_bwd : rows_aw);
  char* p = (char*)base;
  ws.excl = (uint32_t*)p;
  ws.flags = (uint8_t*)(p ? p + e : nullptr);
  ws.rows = (float*)(p ? p + e + f : nullptr);
  ws.total = e + f + r;
  return true;
}

int launch_det_prepare(int P, int64_t R, int rows_per, const GeometryWS& g, const DetWS& d, cudaStream_t st) {
  if (R > 0) {
    cudaError_t e = cudaMemsetAsync(d.flags, 0, (size_t)R * rows_per, st);
    if (e != cudaSuccess) return check_cuda(e, "deterministic flags memset");
  }
  if (P <= 0) return GSR_OK;
  det_excl_kernel<<<(P + DET_THREADS - 1) / DET_THREADS, DET_THREADS, 0, st>>>(P, g.depth_order, g.offsets,
                                                                             g.tiles_touched, d.excl);
  g_launches++;
  return check_launch("det_excl", false, st);
}

int launch_det_reduce_acc(int P, bool depth, const GeometryWS& g, const DetWS& d, float* acc, cudaStream_t st) {
  if (P <= 0) return GSR_OK;
  const int blocks = (P + DET_THREADS - 1) / DET_THREADS;
  if (depth)
    det_reduce_kernel<2, ACC_STRIDE, 10, ACC_STRIDE, false><<<blocks, DET_THREADS, 0, st>>>(P, d.excl, g.tiles_touched,
                                                                                            d.rows, d.flags, acc);
  else
    det_reduce_kernel<2, ACC_STRIDE, 9, ACC_STRIDE, false><<<blocks, DET_THREADS, 0, st>>>(P, d.excl, g.tiles_touched,
                                                                                           d.rows, d.flags, acc);
  g_launches++;
  return check_launch("det_reduce_acc", false, st);
}

int launch_det_reduce_weights(int P, int CH, const GeometryWS& g, const DetWS& d, float* weights, cudaStream_t st) {
  if (P <= 0) return GSR_OK;
  const int blocks = (P + DET_THREADS - 1) / DET_THREADS;
  if (CH == 1)
    det_reduce_kernel<1, 1, 1, 1, true><<<blocks, DET_THREADS, 0, st>>>(P, d.excl, g.tiles_touched, d.rows, d.flags, weights);
  else if (CH == 2)
    det_reduce_kernel<1, 2, 2, 2, true><<<blocks, DET_THREADS, 0, st>>>(P, d.excl, g.tiles_touched, d.rows, d.flags, weights);
  else
    det_reduce_kernel<1, 3, 3, 3, true><<<blocks, DET_THREADS, 0, st>>>(P, d.excl, g.tiles_touched, d.rows, d.flags, weights);
  g_launches++;
  return check_launch("det_reduce_weights", false, st);
}

}  // namespace gsr
