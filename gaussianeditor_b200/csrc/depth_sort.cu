// Depth order of the P Gaussians and the scan of their tile counts in that order, without CUB (sm_90a).
//
// Contract (binning.cu / tile_binning.cu rely on it; the reference gets the same order from the low 32 bits of its
// 64-bit keys and the stability of its radix sort, cuda_rasterizer/rasterizer_impl.cu:67-100,253-261):
//   depth_order[r]  = Gaussian indices ascending in (fp32 view-depth bits, index); culled ones (key 0xFFFFFFFF) last
//   offsets[r]      = inclusive sum of tiles_touched[depth_order[0..r]]
//
// Four stable LSD radix passes over 8-bit digits with the machinery of tile_binning.cu (4096 keys per CTA, atomic
// ticket, decoupled look-back with a window of independent loads, one ballot per digit bit for the stable ranking,
// reorder through shared memory), one histogram kernel for all four digits, and a single-pass chained scan for the
// offsets. Replaces cub::DeviceRadixSort::SortPairs (6 launches) + cub::DeviceScan::InclusiveSum (2 launches).
#include "common.cuh"

namespace gsr {

namespace {

constexpr int DS_THREADS = 256;
constexpr int DS_WARPS = DS_THREADS / 32;
constexpr int DS_ITEMS = 16;
constexpr int DS_TILE = DS_THREADS * DS_ITEMS;  // 4096
constexpr int DS_NB = 256;
constexpr uint32_t DS_AGG = 1u << 30, DS_INC = 2u << 30, DS_VAL = (1u << 30) - 1u;

// all four digit histograms in one pass over the keys (shared-memory privatised, flushed with global atomics)
__global__ void __launch_bounds__(DS_THREADS) depth_hist_kernel(int P, const uint32_t* __restrict__ keys, uint32_t* __restrict__ hist) {
  __shared__ uint32_t s_h[4][DS_NB];
  for (int i = threadIdx.x; i < 4 * DS_NB; i += DS_THREADS) (&s_h[0][0])[i] = 0;
  __syncthreads();
  for (int i = blockIdx.x * DS_THREADS + threadIdx.x; i < P; i += gridDim.x * DS_THREADS) {
    const uint32_t k = __ldg(keys + i);
    atomicAdd(&s_h[0][k & 255u], 1u);
    atomicAdd(&s_h[1][(k >> 8) & 255u], 1u);
    atomicAdd(&s_h[2][(k >> 16) & 255u], 1u);
    atomicAdd(&s_h[3][k >> 24], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 4 * DS_NB; i += DS_THREADS) {
    const uint32_t v = (&s_h[0][0])[i];
    if (v) atomicAdd(hist + i, v);
  }
}

// exclusive scan of each of the four histograms (one warp per histogram, 8 bins per lane), in place
__global__ void depth_base_kernel(uint32_t* __restrict__ hist) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t v[8], sum = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) { v[k] = hist[w * DS_NB + lane * 8 + k]; sum += v[k]; }
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  uint32_t base = inc - sum;
#pragma unroll
  for (int k = 0; k < 8; k++) { hist[w * DS_NB + lane * 8 + k] = base; base += v[k]; }
}

struct DepthPassArgs {
  int P;
  const uint32_t* keys_in;
  const uint32_t* vals_in;   // null in the first pass: the value of element e is e
  uint32_t* keys_out;
  uint32_t* vals_out;
  int shift;
  uint32_t* ticket;
  uint32_t* state;             // [ntiles, DS_NB]
  const uint32_t* digit_base;  // [DS_NB]
};

__global__ void __launch_bounds__(DS_THREADS, 4) depth_sort_pass_kernel(const DepthPassArgs a) {
  __shared__ uint32_t s_whist[DS_WARPS][DS_NB];
  __shared__ uint32_t s_off[DS_NB];
  __shared__ uint32_t s_wsum[DS_WARPS];
  __shared__ uint32_t s_keys[DS_TILE];
  __shared__ uint32_t s_vals[DS_TILE];
  __shared__ uint32_t s_tile;
  const unsigned F = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(a.ticket, 1u);
  for (int i = tid; i < DS_WARPS * DS_NB; i += DS_THREADS) (&s_whist[0][0])[i] = 0;
  __syncthreads();
  const uint32_t tile = s_tile;
  const uint32_t R = (uint32_t)a.P;
  const uint32_t tile_base = tile * (uint32_t)DS_TILE;
  if (tile_base >= R) return;
  const uint32_t nvalid = min((uint32_t)DS_TILE, R - tile_base);
  uint32_t* whist = s_whist[warp];
  const uint32_t s_begin = tile_base + (uint32_t)warp * (32u * DS_ITEMS);

  uint32_t key[DS_ITEMS];
  uint32_t rk[DS_ITEMS / 2];  // rank of the digit inside the warp (< 512), two per register
#pragma unroll
  for (int i = 0; i < DS_ITEMS; i++) {
    const uint32_t e = s_begin + 32u * i + lane;
    key[i] = e < R ? __ldg(a.keys_in + e) : 0xFFFFFFFFu;
  }
#pragma unroll
  for (int i = 0; i < DS_ITEMS; i++) {
    const bool valid = s_begin + 32u * i + lane < R;
    const uint32_t d = (key[i] >> a.shift) & 255u;
    uint32_t peers = __ballot_sync(F, valid);
#pragma unroll
    for (int b = 0; b < 8; b++) {
      const uint32_t bal = __ballot_sync(F, (d >> b) & 1u);
      peers &= ((d >> b) & 1u) ? bal : ~bal;
    }
    const uint32_t lt = peers & ((1u << lane) - 1u);
    uint32_t prev = 0;
    if (valid) prev = whist[d];
    __syncwarp();
    if (valid && lt == 0) whist[d] = prev + __popc(peers);
    __syncwarp();
    const uint32_t r = prev + __popc(lt);
    if (i & 1) rk[i >> 1] |= r << 16; else rk[i >> 1] = r;
  }
  __syncthreads();

  uint32_t cta_hist = 0;
  {
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < DS_WARPS; w++) {
      const uint32_t t = s_whist[w][tid];
      s_whist[w][tid] = run;
      run += t;
    }
    cta_hist = run;
  }
  uint32_t incl = cta_hist;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(F, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_wsum[warp] = incl;
  __syncthreads();
  uint32_t wbase = 0;
#pragma unroll
  for (int w = 0; w < DS_WARPS; w++) wbase += w < warp ? s_wsum[w] : 0u;
  const uint32_t cta_excl = incl - cta_hist + wbase;
  s_off[tid] = cta_excl;
  __syncthreads();

  {
    uint32_t v[DS_ITEMS];
#pragma unroll
    for (int i = 0; i < DS_ITEMS; i++) {
      const uint32_t e = s_begin + 32u * i + lane;
      v[i] = e;                                     // first pass: the value IS the element index
      if (a.vals_in != nullptr && e < R) v[i] = __ldg(a.vals_in + e);
    }
#pragma unroll
    for (int i = 0; i < DS_ITEMS; i++) {
      const uint32_t e = s_begin + 32u * i + lane;
      if (e < R) {
        const uint32_t d = (key[i] >> a.shift) & 255u;
        const uint32_t pos = s_off[d] + s_whist[warp][d] + ((rk[i >> 1] >> (16 * (i & 1))) & 0xFFFFu);
        s_keys[pos] = key[i];
        s_vals[pos] = v[i];
      }
    }
  }
  __syncthreads();
  uint32_t excl = 0;
  {
    volatile uint32_t* st = a.state + (size_t)tile * DS_NB + tid;
    if (tile == 0) {
      *st = cta_hist | DS_INC;
    } else {
      *st = cta_hist | DS_AGG;
      constexpr int LB_WINDOW = 16;
      bool done = false;
      for (int p = (int)tile - 1; !done && p >= 0; p -= LB_WINDOW) {
        uint32_t v[LB_WINDOW];
#pragma unroll
        for (int k = 0; k < LB_WINDOW; k++)
          v[k] = p - k >= 0 ? *(const volatile uint32_t*)(a.state + (size_t)(p - k) * DS_NB + tid) : DS_INC;
#pragma unroll
        for (int k = 0; k < LB_WINDOW; k++) {
          if (!done) {
            uint32_t x = v[k];
            while ((x >> 30) == 0u) x = *(const volatile uint32_t*)(a.state + (size_t)(p - k) * DS_NB + tid);
            excl += x & DS_VAL;
            done = (x >> 30) == 2u;
          }
        }
      }
      *st = ((excl + cta_hist) & DS_VAL) | DS_INC;
    }
    excl += __ldg(a.digit_base + tid);
  }
  s_off[tid] = excl - cta_excl;
  __syncthreads();
  for (uint32_t p = tid; p < nvalid; p += DS_THREADS) {
    const uint32_t k = s_keys[p];
    const uint32_t out = s_off[(k >> a.shift) & 255u] + p;
    a.keys_out[out] = k;
    a.vals_out[out] = s_vals[p];
  }
}

// offsets[r] = inclusive sum of tiles_touched[order[0..r]]: one pass, 4096 ranks per CTA (ticket order), block scan +
// decoupled look-back on one status word per CTA (low 62 bits value, top 2 bits flag)
__global__ void __launch_bounds__(DS_THREADS) offsets_scan_kernel(int P, const uint32_t* __restrict__ order,
                                                                 const uint32_t* __restrict__ tiles_touched,
                                                                 uint32_t* __restrict__ offsets, uint32_t* ticket,
                                                                 unsigned long long* state) {
  __shared__ uint32_t s_wsum[DS_WARPS];
  __shared__ uint32_t s_tile, s_prefix;
  const unsigned F = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const uint32_t tile = s_tile;
  const uint32_t base = tile * (uint32_t)DS_TILE + (uint32_t)tid * DS_ITEMS;  // 16 consecutive ranks per thread
  if (tile * (uint32_t)DS_TILE >= (uint32_t)P) return;
  uint32_t t[DS_ITEMS], sum = 0;
#pragma unroll
  for (int i = 0; i < DS_ITEMS; i++) {
    const uint32_t r = base + i;
    t[i] = r < (uint32_t)P ? __ldg(tiles_touched + __ldg(order + r)) : 0u;
    sum += t[i];
  }
  uint32_t incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(F, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_wsum[warp] = incl;
  __syncthreads();
  uint32_t wbase = 0, total = 0;
#pragma unroll
  for (int w = 0; w < DS_WARPS; w++) { wbase += w < warp ? s_wsum[w] : 0u; total += s_wsum[w]; }
  if (warp == 0) {
    // warp-parallel decoupled look-back: lane l inspects tile - 1 - l (32 predecessors per round, independent loads)
    const unsigned long long AGG = 1ull << 62, INC = 2ull << 62, VAL = (1ull << 62) - 1ull;
    volatile unsigned long long* st = state + tile;
    unsigned long long excl = 0;
    if (tile == 0) {
      if (lane == 0) *st = (unsigned long long)total | INC;
    } else {
      if (lane == 0) *st = (unsigned long long)total | AGG;
      int p = (int)tile - 1;
      bool done = false;
      while (!done) {
        const int q = p - lane;
        unsigned long long x = INC;  // before the first tile: an inclusive prefix of zero
        if (q >= 0) {
          do { x = *(const volatile unsigned long long*)(state + q); } while ((x >> 62) == 0ull);
        }
        const unsigned incmask = __ballot_sync(F, (x >> 62) == 2ull);
        const int first = incmask ? __ffs(incmask) - 1 : 32;   // nearest predecessor with an inclusive prefix
        unsigned long long v = lane <= first ? (x & VAL) : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(F, v, o);
        excl += v;
        done = incmask != 0u;
        p -= 32;
      }
      if (lane == 0) *st = ((excl + total) & VAL) | INC;
    }
    if (lane == 0) s_prefix = (uint32_t)excl;
  }
  __syncthreads();
  uint32_t run = s_prefix + wbase + incl - sum;
#pragma unroll
  for (int i = 0; i < DS_ITEMS; i++) {
    run += t[i];
    if (base + i < (uint32_t)P) offsets[base + i] = run;
  }
}

}  // namespace

// scratch layout (uint32 words): [0..3] pass tickets | [4] scan ticket | [16 .. 16+1024) histograms -> digit bases |
// [2048 ..) 4 x ntiles x 256 status words | scan status (ntiles x u64) | ping-pong keys [P] | ping-pong values [P]
size_t depth_sort_scratch_bytes(int P) {
  const size_t n = (size_t)(P > 0 ? P : 1), ntiles = (n + DS_TILE - 1) / DS_TILE;
  return (2048 + 4 * ntiles * DS_NB + 2 * ntiles + 16) * sizeof(uint32_t) + align_up(n * 4) * 2 + 512;
}

int run_depth_sort_own(int P, const GeometryWS& g, cudaStream_t st, bool debug) {
  const size_t n = (size_t)P, ntiles = (n + DS_TILE - 1) / DS_TILE;
  if (g.cub_temp_bytes < depth_sort_scratch_bytes(P)) { set_error("depth sort scratch too small"); return GSR_ERR_WORKSPACE; }
  uint32_t* w = reinterpret_cast<uint32_t*>(g.cub_temp);
  uint32_t* tickets = w;
  uint32_t* hist = w + 16;
  uint32_t* state = w + 2048;
  unsigned long long* scan_state = reinterpret_cast<unsigned long long*>(state + 4 * ntiles * DS_NB);
  const size_t ctrl_words = 2048 + 4 * ntiles * DS_NB + 2 * ntiles;
  char* after = reinterpret_cast<char*>(w) + align_up(ctrl_words * sizeof(uint32_t));
  uint32_t* keys_b = reinterpret_cast<uint32_t*>(after);
  uint32_t* vals_b = reinterpret_cast<uint32_t*>(after + align_up(n * 4));
  cudaError_t e = cudaMemsetAsync(w, 0, ctrl_words * sizeof(uint32_t), st);
  if (e != cudaSuccess) return check_cuda(e, "depth-sort state memset");
  depth_hist_kernel<<<296, DS_THREADS, 0, st>>>(P, g.depth_keys, hist);
  depth_base_kernel<<<1, 128, 0, st>>>(hist);
  DepthPassArgs a;
  a.P = P;
  const uint32_t* kin[4] = {g.depth_keys, keys_b, g.depth_keys_sorted, keys_b};
  const uint32_t* vin[4] = {nullptr, vals_b, g.depth_order, vals_b};
  uint32_t* kout[4] = {keys_b, g.depth_keys_sorted, keys_b, g.depth_keys_sorted};
  uint32_t* vout[4] = {vals_b, g.depth_order, vals_b, g.depth_order};
  for (int p = 0; p < 4; p++) {
    a.keys_in = kin[p]; a.vals_in = vin[p]; a.keys_out = kout[p]; a.vals_out = vout[p];
    a.shift = 8 * p; a.ticket = tickets + p; a.state = state + (size_t)p * ntiles * DS_NB; a.digit_base = hist + p * DS_NB;
    depth_sort_pass_kernel<<<(unsigned)ntiles, DS_THREADS, 0, st>>>(a);
  }
  offsets_scan_kernel<<<(unsigned)ntiles, DS_THREADS, 0, st>>>(P, g.depth_order, g.tiles_touched, g.offsets, tickets + 4, scan_state);
  g_launches += 7;
  return check_launch("depth sort (own)", debug, st);
}

}  // namespace gsr
