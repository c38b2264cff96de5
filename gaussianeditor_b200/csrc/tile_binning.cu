// Tile binning for sm_90a without CUB: per-tile ranges from a 2-D difference array, and the stable sort of the R
// (Gaussian, tile) instances by tile id as TWO hand-written radix passes with decoupled look-back, the first of which
// generates its input on the fly (instance emission fused in).
//
// Result contract (asserted bit-for-bit against the reference in the GPU tests): `point_list` and `ranges` equal what
// the reference obtains from duplicateWithKeys + a stable 64-bit radix sort + identifyTileRanges
// (cuda_rasterizer/rasterizer_impl.cu:67-125,227-270): instances ordered by (tile id, depth bits, Gaussian index).
// As in binning.cu the P Gaussians are already in (depth bits, index) order (`depth_order`, with `offsets` = inclusive
// scan of their tile counts in that order), so what is left is a STABLE sort of the emission sequence by tile id.
//
//   tile_prefix_kernel  the preprocess kernel added the four corners of every visible Gaussian's tile rectangle to a
//                       (gy+1) x (gx+1) difference array; its 2-D prefix sum is the instance count of every tile ->
//                       `ranges` (exclusive scan; (0,0) for empty tiles like the reference's memset), and the digit
//                       histograms of both radix passes. No pass over the R instances, no sorted keys needed.
//   tile_sort_pass<1>   CTA = 4096 consecutive emission slots: each warp finds the Gaussians of its 512 slots in the
//                       offsets array (32-ary cooperative search, then shuffle-only), forms (tile id, index) in
//                       registers, ranks the low digit (match_any + per-warp counters), obtains its global bin offsets
//                       by decoupled look-back over the preceding CTAs, reorders through shared memory and writes
//                       coalesced runs.  The 8*R bytes the separate emit kernel wrote and the sort re-read are gone, and
//                       so is the histogram pass over the keys.
//   tile_sort_pass<2>   the same kernel on the high digit, reading pass 1's output.
//
// The CTAs take their tile through an atomic ticket, so every predecessor a CTA waits for in the look-back is already
// running: no deadlock regardless of the block scheduling order.
#include "common.cuh"

namespace gsr {

namespace {

constexpr int SORT_THREADS = 256;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int SORT_ITEMS = SORT_TILE / SORT_THREADS;  // 16 per thread; a warp owns 512 consecutive slots
constexpr int NB = 256;                               // status words per sort tile (digits are at most 8 bits)
static_assert(SORT_ITEMS == 16 && SORT_TILE == SORT_WARPS * 32 * SORT_ITEMS, "tile shape");

constexpr uint32_t FLAG_AGG = 1u << 30, FLAG_INC = 2u << 30, VAL_MASK = (1u << 30) - 1u;

// rasterizer_impl.cu:36-49
uint32_t higher_msb(uint32_t n) {
  uint32_t msb = sizeof(n) * 4, step = msb;
  while (step > 1) {
    step /= 2;
    if (n >> msb) msb += step; else msb -= step;
  }
  if (n >> msb) msb++;
  return msb;
}

__device__ __forceinline__ void tile_rect(float px, float py, int radius, int gx, int gy, uint2& rmin, uint2& rmax) {
  // auxiliary.h:46-56
  rmin.x = (unsigned)min(gx, max((int)0, (int)((px - radius) / TILE)));
  rmin.y = (unsigned)min(gy, max((int)0, (int)((py - radius) / TILE)));
  rmax.x = (unsigned)min(gx, max((int)0, (int)((px + radius + TILE - 1) / TILE)));
  rmax.y = (unsigned)min(gy, max((int)0, (int)((py + radius + TILE - 1) / TILE)));
}
__device__ __forceinline__ void owned_rows(uint32_t ymin, uint32_t ymax, int stride, int phase, uint32_t& y0, uint32_t& ny) {
  if (stride == 1) { y0 = ymin; ny = ymax - ymin; return; }
  int d = (phase - (int)ymin) % stride;
  if (d < 0) d += stride;
  y0 = ymin + (uint32_t)d;
  ny = y0 < ymax ? (ymax - y0 + (uint32_t)stride - 1u) / (uint32_t)stride : 0u;
}

// ---------------------------------------------------------------------------------------------------------------
// ranges + digit bases from the difference array (one CTA; the arrays are a few tens of KB and L2-resident)
// ---------------------------------------------------------------------------------------------------------------
constexpr int PREFIX_THREADS = 1024;

// rows ty >= y of a gy-row grid that this rank owns (ty % stride == phase)
__device__ __forceinline__ int owned_rows_from(int y, int gy, int stride, int phase) {
  if (stride == 1) return max(gy - y, 0);
  int d = (phase - y) % stride;
  if (d < 0) d += stride;
  const int first = y + d;
  return first < gy ? (gy - first + stride - 1) / stride : 0;
}

// One thread per entry of the difference array: adds up the replicas (-> `sum`, what tile_prefix_kernel reads) and
// accumulates R without any prefix sum: an entry (x, y) is seen by every tile (tx >= x, ty >= y), so
//   R = sum_entries diff[y][x] * (gx - x) * #owned rows >= y.
// Every Gaussian's four corners cancel to its own instance count, so each block's partial sum is non-negative.
constexpr int COUNT_THREADS = 256;
__global__ void __launch_bounds__(COUNT_THREADS)
tile_count_kernel(int gx, int gy, int own_stride, int own_phase, const int32_t* __restrict__ diff, int copies,
                  int32_t* __restrict__ sum, uint32_t* __restrict__ R_dev) {
  __shared__ long long s_part[COUNT_THREADS / 32];
  const int stride = gx + 1, nent = stride * (gy + 1);
  const int i = blockIdx.x * COUNT_THREADS + threadIdx.x;
  long long acc = 0;
  if (i < nent) {
    int v = 0;
    for (int c = 0; c < copies; c++) v += diff[(size_t)c * nent + i];  // independent coalesced loads
    sum[i] = v;
    if (v != 0) {
      const int y = i / stride, x = i - y * stride;
      acc = (long long)v * (long long)(gx - x) * (long long)owned_rows_from(y, gy, own_stride, own_phase);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    long long v = threadIdx.x < COUNT_THREADS / 32 ? s_part[threadIdx.x] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    // signed partial sums of different blocks add up to R >= 0 (two's complement wrap-around is harmless)
    if (threadIdx.x == 0 && v != 0) atomicAdd(R_dev, (uint32_t)v);
  }
}

__global__ void __launch_bounds__(PREFIX_THREADS)
tile_prefix_kernel(int gx, int gy, int own_stride, int own_phase, const int32_t* __restrict__ diff, int32_t* cnt_global,
                   uint2* __restrict__ ranges, uint32_t* __restrict__ digit_base, int bits1, const uint32_t* __restrict__ R_dev,
                   uint32_t cap) {
  constexpr int SMEM_CNT = 10240;  // 40 KB: grids up to ~1600x1600 pixels keep the 2-D prefix in shared memory
  __shared__ int32_t s_cnt[SMEM_CNT];
  __shared__ uint32_t s_h[2][NB];
  __shared__ uint32_t s_warp[PREFIX_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int stride = gx + 1;
  int32_t* cnt = stride * (gy + 1) <= SMEM_CNT ? s_cnt : cnt_global;
  for (int i = tid; i < 2 * NB; i += PREFIX_THREADS) (&s_h[0][0])[i] = 0;
  // prefix along x: one warp per row, 32 entries per step with a shuffle scan and a running carry. With the array in
  // shared memory the difference array is first copied in with independent coalesced loads (one exposed latency).
  const int nent = stride * (gy + 1);
  // the summed difference array (tile_count_kernel) -> shared memory, or -> the global scratch for very large grids
  for (int i = tid; i < nent; i += PREFIX_THREADS) cnt[i] = diff[i];
  __syncthreads();
  const int32_t* src = cnt;
  for (int r = warp; r <= gy; r += PREFIX_THREADS / 32) {
    int carry = 0;
    for (int x0 = 0; x0 <= gx; x0 += 32) {
      const int x = x0 + lane;
      int v = x <= gx ? src[r * stride + x] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
      }
      v += carry;
      if (x <= gx) cnt[r * stride + x] = v;
      carry = __shfl_sync(0xffffffffu, v, 31);
    }
  }
  __syncthreads();
  // prefix along y: one thread per column (coalesced across the threads; the loads do not depend on the running sum)
  for (int c = tid; c <= gx; c += PREFIX_THREADS) {
    int acc = 0;
#pragma unroll 8
    for (int y = 0; y <= gy; y++) {
      acc += cnt[y * stride + c];
      cnt[y * stride + c] = acc;
    }
  }
  __syncthreads();
  // exclusive scan of the counts over the tiles (row-major) -> ranges, digit histograms
  const int ntile = gx * gy;
  const int per = (ntile + PREFIX_THREADS - 1) / PREFIX_THREADS;
  const int t0 = min(ntile, tid * per), t1 = min(ntile, t0 + per);
  auto count_of = [&](int t) -> uint32_t {
    const int ty = t / gx, tx = t - ty * gx;
    if (own_stride != 1 && (ty % own_stride) != own_phase) return 0u;  // sharded path: only the owned tile rows are binned
    return (uint32_t)cnt[ty * stride + tx];
  };
  uint32_t mine = 0;
  for (int t = t0; t < t1; t++) mine += count_of(t);
  uint32_t incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t v = s_warp[lane];
    uint32_t inc2 = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, inc2, o);
      if (lane >= o) inc2 += u;
    }
    s_warp[lane] = inc2 - v;
  }
  __syncthreads();
  uint32_t run = incl - mine + s_warp[warp];
  const uint32_t mask1 = (1u << bits1) - 1u;
  // speculative launch whose capacity guess was too small: the sort passes skip their work and the host redoes the
  // second half; empty ranges keep the (discarded) render of this launch away from the unsorted list
  const bool overflow = R_dev != nullptr && __ldcg(R_dev) > cap;
  // ranges + histogram of the HIGH digit: a thread's consecutive tiles share it except at a boundary -> one shared
  // atomic per run instead of one per tile (7500 atomics into 64 bins serialised this kernel)
  uint32_t hi_bin = 0xFFFFFFFFu, hi_sum = 0;
  for (int t = t0; t < t1; t++) {
    const uint32_t c = overflow ? 0u : count_of(t);
    ranges[t] = c ? make_uint2(run, run + c) : make_uint2(0u, 0u);
    const uint32_t b = (uint32_t)t >> bits1;
    if (b != hi_bin) {
      if (hi_sum) atomicAdd(&s_h[1][hi_bin], hi_sum);
      hi_bin = b; hi_sum = 0;
    }
    hi_sum += c;
    run += c;
  }
  if (hi_sum) atomicAdd(&s_h[1][hi_bin], hi_sum);
  // histogram of the LOW digit: thread `tid` adds up the tiles t = tid, tid + 1024, ... -- they all have the low digit
  // tid & mask1 (1024 is a multiple of 2^bits1) -> one shared atomic per thread
  if (!overflow) {
    uint32_t lo_sum = 0;
    for (int t = tid; t < ntile; t += PREFIX_THREADS) lo_sum += count_of(t);
    if (lo_sum) atomicAdd(&s_h[0][tid & mask1], lo_sum);
  }
  __syncthreads();
  if (warp < 2) {  // exclusive scan of one 256-bin histogram per warp (8 bins per lane)
    uint32_t v[8], sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) { v[k] = s_h[warp][lane * 8 + k]; sum += v[k]; }
    uint32_t inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    uint32_t base = inc - sum;
#pragma unroll
    for (int k = 0; k < 8; k++) { digit_base[warp * NB + lane * 8 + k] = base; base += v[k]; }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// one radix pass
// ---------------------------------------------------------------------------------------------------------------
struct SortArgs {
  int P;
  uint32_t cap;            // slots the grid was sized for (== R unless speculative)
  const uint32_t* R_dev;   // instance count on the device (speculative launches), or null: R = cap
  // pass 1: emission inputs
  const uint32_t* order;
  const uint32_t* offsets;
  const uint32_t* tiles_touched;
  const SplatRecord* records;
  const int32_t* radii;
  int gx, gy, own_stride, own_phase;
  // pass 2: input arrays
  const uint16_t* keys_in;
  const uint32_t* vals_in;
  uint16_t* keys_out;
  uint32_t* vals_out;
  int shift, nbits;
  uint32_t* ticket;
  uint32_t* state;              // [ntiles, NB]
  const uint32_t* digit_base;   // [NB] exclusive scan of this pass's global digit histogram
};

template <bool EMIT, int NBITS>
__global__ void __launch_bounds__(SORT_THREADS, 4) tile_sort_pass_kernel(const SortArgs a) {
  __shared__ uint32_t s_whist[SORT_WARPS][NB];
  __shared__ uint32_t s_off[NB];    // CTA-exclusive prefix over the digits, later the global offset of the digit's run
  __shared__ uint32_t s_wsum[SORT_WARPS];
  __shared__ uint16_t s_keys[SORT_TILE];
  __shared__ uint32_t s_vals[SORT_TILE];
  __shared__ uint32_t s_tile;
  const unsigned F = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(a.ticket, 1u);
  for (int i = tid; i < SORT_WARPS * NB; i += SORT_THREADS) (&s_whist[0][0])[i] = 0;
  __syncthreads();
  const uint32_t tile = s_tile;
  const uint32_t R_true = a.R_dev ? __ldcg(a.R_dev) : a.cap;
  if (R_true > a.cap) return;  // speculative capacity too small: nothing is sorted, the host redoes the second half
  const uint32_t R = R_true;
  const uint32_t tile_base = tile * (uint32_t)SORT_TILE;
  if (tile_base >= R) return;  // CTA-uniform
  const uint32_t nvalid = min((uint32_t)SORT_TILE, R - tile_base);
  constexpr uint32_t dmask = (1u << NBITS) - 1u;  // digit width is a template parameter: the ranking below is straight-line code
  uint32_t* whist = s_whist[warp];

  // Register diet (64 registers -> 4 CTAs per SM): one word per item = key (low 16 bits) | rank of its digit inside the
  // warp (high 16 bits, < 512); the values are not held at all until the reorder step -- pass 1 leaves them in shared
  // memory where the transposition put them, pass 2 loads them then.
  uint32_t kr[SORT_ITEMS];
  const uint32_t s_begin = tile_base + (uint32_t)warp * (32u * SORT_ITEMS);  // first slot of this warp

  if (EMIT) {
    if (s_begin < R) {  // warp-uniform
      // Depth ranks of this warp's 512 slots: r_lo = smallest rank with offsets[rank] > s_begin (32-ary cooperative
      // search, 4 dependent loads at P = 1M); every visible rank owns >= 1 slot, so the 512 slots span at most 512
      // ranks: their offsets are staged in the warp's part of s_vals (16 independent coalesced loads per lane) and
      // each slot finishes with a binary search in shared memory. All global loads of the 16 items are independent.
      int lo = 0, n = a.P;
      while (n > 1) {
        const int stride = (n + 31) >> 5;
        const int pos = min(lo + (lane + 1) * stride - 1, lo + n - 1);
        const unsigned gt = __ballot_sync(F, __ldg(a.offsets + pos) > s_begin);
        const int j = __ffs(gt) - 1;
        lo += j * stride;
        n = min(stride, n - j * stride);
      }
      const int r_lo = lo;
      uint32_t* sval = s_vals + warp * (32 * SORT_ITEMS);   // this warp's 512 values (swizzled, warp-striped)
      uint16_t* skey = s_keys + warp * (32 * SORT_ITEMS);   // first the staged offsets, then this warp's 512 keys
      // offsets relative to the warp's first slot, saturated to 16 bits: only "<= slot" with slot - s_begin < 512 is
      // ever asked of them, so 512 of them fit the warp's key area and the value area stays free for the results
#pragma unroll
      for (int i = 0; i < SORT_ITEMS; i++)
        skey[i * 32 + lane] = (uint16_t)min(__ldg(a.offsets + min(r_lo + i * 32 + lane, a.P - 1)) - s_begin, 0xFFFFu);
      __syncwarp();
      // BLOCKED generation: lane l walks the 16 consecutive slots s_begin + 16 l ... -- one binary search for its first
      // slot, then tile ids by incrementing (column, row) inside the Gaussian's rectangle; a new Gaussian is fetched
      // only when the walk crosses the end of the current one (every visible rank owns >= 1 slot: one step).
      const uint32_t first = (uint32_t)(SORT_ITEMS * lane);           // relative to s_begin
      const uint32_t last_rel = R - 1 - s_begin;                       // last valid slot, relative
      const uint32_t sc = min(first, last_rel);
      int j = 0;  // smallest j with skey[j] > sc
#pragma unroll
      for (int step = 256; step > 0; step >>= 1)
        if ((uint32_t)skey[j + step - 1] <= sc) j += step;
      uint32_t idx, end, w, xmin, ybase, rx, ry;
      auto fetch = [&](int jj) {
        end = skey[jj];
        idx = __ldg(a.order + min(r_lo + jj, a.P - 1));
        const float4 q0 = __ldg(reinterpret_cast<const float4*>(a.records + idx));
        uint2 rmin, rmax;
        tile_rect(q0.x, q0.y, __ldg(a.radii + idx), a.gx, a.gy, rmin, rmax);
        w = max(rmax.x - rmin.x, 1u);
        xmin = rmin.x;
        uint32_t y0, ny;
        owned_rows(rmin.y, rmax.y, a.own_stride, a.own_phase, y0, ny);
        ybase = y0;
      };
      fetch(j);
      {
        // absolute arithmetic for the position inside the first Gaussian (its start may lie before s_begin)
        const uint32_t end_abs = __ldg(a.offsets + min(r_lo + j, a.P - 1));
        const uint32_t k = (s_begin + sc) - (end_abs - __ldg(a.tiles_touched + idx));
        ry = k / w;
        rx = k - ry * w;
      }
      uint32_t bk[SORT_ITEMS / 2];  // two 16-bit keys per register
#pragma unroll
      for (int i = 0; i < SORT_ITEMS; i++) {
        const uint32_t sl = first + i;
        if (sl <= last_rel && sl >= end) {  // crossed into the next depth rank
          j++;
          fetch(j);
          rx = 0; ry = 0;
        }
        const uint32_t kk = ((ybase + ry * (uint32_t)a.own_stride) * a.gx + (xmin + rx)) & 0xFFFFu;
        if (i & 1) bk[i >> 1] |= kk << 16; else bk[i >> 1] = kk;
        // blocked -> warp-striped through shared memory (the stable ranking below needs item i of lane l to be slot
        // 32 i + l); the XOR swizzle makes both the writes (stride 16) and the reads (stride 1) bank-conflict free
        const int pl = SORT_ITEMS * lane + i;
        sval[pl ^ ((pl >> 5) & 15)] = idx;
        rx++;
        if (rx == w) { rx = 0; ry++; }
      }
      __syncwarp();  // everybody is done with the staged offsets: the key area now takes the keys
#pragma unroll
      for (int i = 0; i < SORT_ITEMS; i++) {
        const int pl = SORT_ITEMS * lane + i;
        skey[pl ^ ((pl >> 5) & 15)] = (uint16_t)(bk[i >> 1] >> (16 * (i & 1)));
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < SORT_ITEMS; i++) {
        const int pl = 32 * i + lane;
        kr[i] = skey[pl ^ ((pl >> 5) & 15)];
      }
    } else {
#pragma unroll
      for (int i = 0; i < SORT_ITEMS; i++) kr[i] = 0;
    }
  } else {
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; i++) {
      const uint32_t e = s_begin + 32u * i + lane;
      kr[i] = e < R ? (uint32_t)a.keys_in[e] : 0u;
    }
  }
  // ---- stable rank of every item's digit among the warp's earlier slots (match_any + per-warp counters) ----
#pragma unroll
  for (int i = 0; i < SORT_ITEMS; i++) {
    const bool valid = s_begin + 32u * i + lane < R;
    const uint32_t d = valid ? ((kr[i] >> a.shift) & dmask) : 0xFFFFFFFFu;
    // lanes with the same digit: one ballot per digit bit (MATCH.ANY measured ~100 cycles of SM time per warp
    // instruction here: 16 of them per thread were 40 % of this kernel's stall samples)
    uint32_t peers = __ballot_sync(F, valid);
#pragma unroll
    for (int b = 0; b < NBITS; b++) {
      const uint32_t bal = __ballot_sync(F, (d >> b) & 1u);
      peers &= ((d >> b) & 1u) ? bal : ~bal;
    }
    const uint32_t lt = peers & ((1u << lane) - 1u);
    uint32_t prev = 0;
    if (valid) prev = whist[d];
    __syncwarp();
    if (valid && lt == 0) whist[d] = prev + __popc(peers);
    __syncwarp();
    kr[i] |= (prev + __popc(lt)) << 16;
  }
  __syncthreads();

  // ---- per digit (thread d): exclusive prefix over the warps, CTA total ----
  uint32_t cta_hist = 0;
  {
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < SORT_WARPS; w++) {
      const uint32_t t = s_whist[w][tid];
      s_whist[w][tid] = run;
      run += t;
    }
    cta_hist = run;
  }
  // ---- CTA-exclusive scan over the digits ----
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
  for (int w = 0; w < SORT_WARPS; w++) wbase += w < warp ? s_wsum[w] : 0u;
  const uint32_t cta_excl = incl - cta_hist + wbase;

  s_off[tid] = cta_excl;
  __syncthreads();

  // ---- reorder inside the CTA (before the look-back: it frees the registers) ----
  {
    uint32_t v[SORT_ITEMS];
    const uint32_t* sval_w = s_vals + warp * (32 * SORT_ITEMS);
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; i++) {
      const uint32_t e = s_begin + 32u * i + lane;
      const int pl = 32 * i + lane;
      v[i] = 0;
      if (e < R) v[i] = EMIT ? sval_w[pl ^ ((pl >> 5) & 15)] : a.vals_in[e];
    }
    __syncthreads();  // pass 1: every value has left the staging area before it is overwritten
#pragma unroll
    for (int i = 0; i < SORT_ITEMS; i++) {
      const uint32_t e = s_begin + 32u * i + lane;
      if (e < R) {
        const uint32_t k = kr[i] & 0xFFFFu;
        const uint32_t d = (k >> a.shift) & dmask;
        const uint32_t pos = s_off[d] + s_whist[warp][d] + (kr[i] >> 16);
        s_keys[pos] = (uint16_t)k;
        s_vals[pos] = v[i];
      }
    }
  }
  __syncthreads();
  // ---- decoupled look-back: global offset of this CTA's run of digit `tid` ----
  uint32_t excl = 0;
  if ((uint32_t)tid <= dmask) {
    volatile uint32_t* st = a.state + (size_t)tile * NB + tid;
    if (tile == 0) {
      *st = cta_hist | FLAG_INC;
    } else {
      *st = cta_hist | FLAG_AGG;
      // Windowed look-back: the status words of LB_WINDOW predecessors are fetched with independent loads before any
      // of them is inspected. The "inclusive" front can only advance LB_WINDOW tiles per L2 round trip (a tile that
      // sees nothing but aggregates in its window has to go one window further back), and with ~1600 tiles of a few
      // microseconds each that chain, not the sorting work, was the critical path (measured: 8 -> 0.34 us per round).
      constexpr int LB_WINDOW = 16;
      bool done = false;
      for (int p = (int)tile - 1; !done && p >= 0; p -= LB_WINDOW) {
        uint32_t v[LB_WINDOW];
#pragma unroll
        for (int k = 0; k < LB_WINDOW; k++)
          v[k] = p - k >= 0 ? *(const volatile uint32_t*)(a.state + (size_t)(p - k) * NB + tid) : FLAG_INC;
#pragma unroll
        for (int k = 0; k < LB_WINDOW; k++) {
          if (!done) {
            uint32_t x = v[k];
            while ((x >> 30) == 0u) x = *(const volatile uint32_t*)(a.state + (size_t)(p - k) * NB + tid);
            excl += x & VAL_MASK;
            done = (x >> 30) == 2u;
          }
        }
      }
      *st = ((excl + cta_hist) & VAL_MASK) | FLAG_INC;
    }
    excl += __ldg(a.digit_base + tid);
  }

  s_off[tid] = excl - cta_excl;  // global position of local position p of digit tid = s_off + p   (mod 2^32)
  __syncthreads();
  for (uint32_t p = tid; p < nvalid; p += SORT_THREADS) {
    const uint16_t k = s_keys[p];
    const uint32_t d = ((uint32_t)k >> a.shift) & dmask;
    const uint32_t out = s_off[d] + p;
    a.keys_out[out] = k;
    a.vals_out[out] = s_vals[p];
  }
}

template <bool EMIT>
void launch_pass(int nbits, int ntiles, const SortArgs& a, cudaStream_t st) {
  switch (nbits) {
    case 1: tile_sort_pass_kernel<EMIT, 1><<<ntiles, SORT_THREADS, 0, st>>>(a); break;
    case 2: tile_sort_pass_kernel<EMIT, 2><<<ntiles, SORT_THREADS, 0, st>>>(a); break;
    case 3: tile_sort_pass_kernel<EMIT, 3><<<ntiles, SORT_THREADS, 0, st>>>(a); break;
    case 4: tile_sort_pass_kernel<EMIT, 4><<<ntiles, SORT_THREADS, 0, st>>>(a); break;
    case 5: tile_sort_pass_kernel<EMIT, 5><<<ntiles, SORT_THREADS, 0, st>>>(a); break;
    case 6: tile_sort_pass_kernel<EMIT, 6><<<ntiles, SORT_THREADS, 0, st>>>(a); break;
    case 7: tile_sort_pass_kernel<EMIT, 7><<<ntiles, SORT_THREADS, 0, st>>>(a); break;
    default: tile_sort_pass_kernel<EMIT, 8><<<ntiles, SORT_THREADS, 0, st>>>(a); break;
  }
}

}  // namespace

bool tile_binning_supported(int gx, int gy) {
  return g_opt.binning_variant == 1 && g_opt.tile_key_bits == 16 && (int64_t)gx * gy < 65536 &&
         (int64_t)(gx + 1) * (gy + 1) <= MAX_TILE_DIFF;
}

int clear_tile_counts(const GeometryWS& g, int gx, int gy, cudaStream_t st) {
  // R_dev (16 bytes) sits directly in front of the difference array
  const size_t bytes = 16 + (size_t)tile_diff_copies(gx, gy) * (gx + 1) * (gy + 1) * sizeof(int32_t);
  return check_cuda(cudaMemsetAsync(g.R_dev, 0, bytes, st), "tile-count memset");
}

int launch_tile_count(const GeometryWS& g, int gx, int gy, const TileOwner& own, cudaStream_t st) {
  const int copies = tile_diff_copies(gx, gy), nent = (gx + 1) * (gy + 1);
  tile_count_kernel<<<(nent + COUNT_THREADS - 1) / COUNT_THREADS, COUNT_THREADS, 0, st>>>(
      gx, gy, own.stride, own.phase, g.tile_diff, copies, g.tile_diff + (size_t)copies * nent, g.R_dev);
  g_launches++;
  return check_launch("tile_count", false, st);
}

int run_tile_binning(const gsr_settings& s, int P, int R, bool speculative, const GeometryWS& g, const BinningWS& b,
                     const ImageWS& im, const int32_t* radii, cudaStream_t st, const TileOwner& own) {
  const int W = s.image_width, H = s.image_height;
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  const bool debug = s.debug != 0;
  const int bits = (int)higher_msb((uint32_t)(gx * gy));
  const int bits1 = (bits + 1) / 2, bits2 = bits - bits1;
  const int ntiles = (R + SORT_TILE - 1) / SORT_TILE;
  // sort_state layout: [0..1] tickets | [16 .. 16+2*NB) digit bases | [1024 ..) pass-1 status, pass-2 status | counts
  uint32_t* ticket = b.sort_state;
  uint32_t* digit_base = b.sort_state + 16;
  uint32_t* state = b.sort_state + 1024;
  const size_t state_words = (size_t)2 * (ntiles > 0 ? ntiles : 1) * NB;
  int32_t* cnt = reinterpret_cast<int32_t*>(state + state_words);
  {
    StageScope t(ST_RANGES, st);
    cudaError_t e = cudaMemsetAsync(b.sort_state, 0, (1024 + state_words) * sizeof(uint32_t), st);
    if (e != cudaSuccess) return check_cuda(e, "sort-state memset");
    const int32_t* diff_sum = g.tile_diff + (size_t)tile_diff_copies(gx, gy) * (gx + 1) * (gy + 1);
    tile_prefix_kernel<<<1, PREFIX_THREADS, 0, st>>>(gx, gy, own.stride, own.phase, diff_sum, cnt, im.ranges, digit_base,
                                                    bits1, speculative ? g.R_dev : nullptr, (uint32_t)R);
    g_launches++;
    int rc = check_launch("tile_prefix", debug, st);
    if (rc) return rc;
  }
  if (R <= 0) return GSR_OK;
  StageScope t(ST_TILE_SORT, st);
  SortArgs a;
  a.P = P; a.cap = (uint32_t)R; a.R_dev = speculative ? g.R_dev : nullptr;
  a.order = g.depth_order; a.offsets = g.offsets; a.tiles_touched = g.tiles_touched; a.records = g.records; a.radii = radii;
  a.gx = gx; a.gy = gy; a.own_stride = own.stride; a.own_phase = own.phase;
  a.keys_in = nullptr; a.vals_in = nullptr;
  a.keys_out = reinterpret_cast<uint16_t*>(b.keys_unsorted); a.vals_out = b.vals_unsorted;
  a.shift = 0; a.nbits = bits1;
  a.ticket = ticket; a.state = state; a.digit_base = digit_base;
  launch_pass<true>(a.nbits, ntiles, a, st);
  g_launches++;
  int rc = check_launch("tile_sort_pass1", debug, st);
  if (rc) return rc;
  if (bits2 == 0) {  // at most 2 tiles... a single digit covers the ids: pass 1's output is final
    cudaError_t e = cudaMemcpyAsync(b.keys_sorted, b.keys_unsorted, (size_t)R * sizeof(uint16_t), cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(b.point_list, b.vals_unsorted, (size_t)R * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st);
    return check_cuda(e, "single-digit tile sort copy");
  }
  a.keys_in = reinterpret_cast<const uint16_t*>(b.keys_unsorted); a.vals_in = b.vals_unsorted;
  a.keys_out = reinterpret_cast<uint16_t*>(b.keys_sorted); a.vals_out = b.point_list;
  a.shift = bits1; a.nbits = bits2;
  a.ticket = ticket + 1; a.state = state + (size_t)(ntiles > 0 ? ntiles : 1) * NB; a.digit_base = digit_base + NB;
  launch_pass<false>(a.nbits, ntiles, a, st);
  g_launches++;
  return check_launch("tile_sort_pass2", debug, st);
}

}  // namespace gsr
