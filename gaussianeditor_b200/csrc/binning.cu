// Binning for sm_90a: turn per-Gaussian tile rectangles into per-tile, depth-ordered splat lists.
//
// The reference (cuda_rasterizer/rasterizer_impl.cu:227-270) emits one 64-bit key  tile<<32 | depth_bits  per
// (Gaussian, tile) instance in Gaussian-index order and radix-sorts all R instances over 32+bit key bits
// (6 eight-bit passes over 12 B/instance).  Its result -- point_list and the tile ranges -- is fully
// determined by the order  (tile, depth bits, Gaussian index)  because the sort is stable.
//
// Here the same permutation is produced with a quarter of the traffic by splitting the key:
//   1. stable radix sort of the P Gaussians by depth bits (32-bit keys, P items, culled ones keyed 0xFFFFFFFF),
//   2. inclusive scan of the tile counts IN THAT ORDER -> instance offsets, R,
//   3. emission of (tile id, Gaussian index) in depth order, one thread per instance (load-balanced search),
//   4. stable radix sort of the R instances by tile id only (`bit` = getHigherMsb(Ntile) bits -> 2 passes over
//      8 B/instance) -- ties keep emission order = (depth bits, index),
//   5. tile ranges from the sorted tile ids.
// Equality of point_list / ranges / R with the reference is asserted bit-for-bit in the GPU tests.
#include <cub/cub.cuh>

#include <mutex>
#include <unordered_map>

#include "common.cuh"

namespace gsr {

namespace {

// rasterizer_impl.cu:36-49 (number of key bits that cover the tile ids)
uint32_t higher_msb(uint32_t n) {
  uint32_t msb = sizeof(n) * 4;
  uint32_t step = msb;
  while (step > 1) {
    step /= 2;
    if (n >> msb)
      msb += step;
    else
      msb -= step;
  }
  if (n >> msb) msb++;
  return msb;
}

// tiles_touched gathered through the depth order, as a CUB input iterator
struct GatherTilesOp {
  const uint32_t* tiles;
  const uint32_t* order;
  __host__ __device__ __forceinline__ uint32_t operator()(uint32_t rank) const { return tiles[order[rank]]; }
};

// Sharded path, after the all-gather of the splat records: rebuild the per-Gaussian arrays of all P Gaussians from
// the records (radius = q2.w, depth key = bits of q1.z), count the OWNED tiles and write the identity permutation the
// depth sort carries. A Gaussian that touches none of this rank's tile rows gets the "culled" depth key, so that --
// as on a single GPU -- every Gaussian with a zero count sorts behind all the others (emit_instances_kernel relies on
// it: 32 consecutive instance slots then span at most 32 depth ranks). Its position in the order is irrelevant: it
// emits nothing.
__global__ void retouch_kernel(int P, const SplatRecord* __restrict__ records, int gx, int gy, int stride, int phase,
                               int32_t* __restrict__ radii, uint32_t* __restrict__ tiles_touched,
                               uint32_t* __restrict__ ident, uint32_t* __restrict__ depth_keys,
                               int32_t* __restrict__ tile_diff, int diff_copies) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t n = 0;
  if (idx < P) {
    const float4* r = reinterpret_cast<const float4*>(records + idx);
    const int radius = __float_as_int(__ldg(r + 2).w);
    uint32_t key = 0xFFFFFFFFu;
    if (radius > 0) {
      const float4 q0 = __ldg(r);
      uint2 rmin, rmax;
      tile_rect(q0.x, q0.y, radius, gx, gy, rmin, rmax);
      uint32_t y0, ny;
      owned_rows(rmin.y, rmax.y, stride, phase, y0, ny);
      n = ny * (rmax.x - rmin.x);
      if (n != 0) {
        key = __float_as_uint(__ldg(r + 1).z);
        // full rectangle: tile_prefix_kernel keeps the owned rows
        if (tile_diff) add_tile_rect(tile_diff, gx, gy, diff_copies, (uint32_t)idx, rmin.x, rmin.y, rmax.x, rmax.y);
      }
    }
    radii[idx] = radius;
    tiles_touched[idx] = n;
    ident[idx] = (uint32_t)idx;
    depth_keys[idx] = key;
  }
}

// One thread per OUTPUT slot (instance): perfectly balanced no matter how the tile counts are distributed --
// in depth order the few huge near-camera splats (thousands of tiles each) are adjacent ranks, so any
// rank-to-thread or rank-to-warp assignment serialises them. Finding the owner rank of a slot is a search over the
// inclusive offsets; a per-thread binary search is a chain of ~20 dependent loads, so each WARP instead locates the
// rank of its first slot with a 32-ary cooperative search (4 dependent loads for P = 1M), probes the next 32 offsets
// once (32 consecutive slots span at most 32 visible ranks) and the lanes finish with a shuffle-only search.
// Stores are fully coalesced.
constexpr int EMIT_THREADS = 256;
constexpr int EMIT_CHUNKS = 8;  // consecutive 32-slot chunks per warp: the 32-ary search is paid once per 256 slots
template <typename KeyT>
__global__ void __launch_bounds__(EMIT_THREADS)
emit_instances_kernel(int P, uint32_t cap, const uint32_t* __restrict__ R_dev, KeyT pad_key,
                      const uint32_t* __restrict__ order, const uint32_t* __restrict__ offsets,
                      const uint32_t* __restrict__ tiles_touched, const SplatRecord* __restrict__ records,
                      const int32_t* __restrict__ radii, int gx, int gy, int own_stride, int own_phase,
                      KeyT* __restrict__ keys, uint32_t* __restrict__ vals) {
  const unsigned F = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const uint32_t warp_id = (blockIdx.x * EMIT_THREADS + threadIdx.x) >> 5;
  const uint32_t s_begin = warp_id * (32u * EMIT_CHUNKS);
  if (s_begin >= cap) return;
  // Speculative launches size the grid for a capacity `cap` >= R that the host guessed before R was known; R itself is
  // read from the scan result on the device and the slots [R, cap) get a key that sorts behind every tile.
  const uint32_t R = R_dev ? min(__ldg(R_dev), cap) : cap;
  int r_base = 0;
  if (s_begin < R) {
    // smallest rank with offsets[rank] > s_begin; invariant: answer in [lo, lo+n), offsets[lo+n-1] > s_begin
    int lo = 0, n = P;
    while (n > 1) {  // warp-uniform
      const int stride = (n + 31) >> 5;
      const int pos = min(lo + (lane + 1) * stride - 1, lo + n - 1);
      const unsigned gt = __ballot_sync(F, __ldg(offsets + pos) > s_begin);
      const int j = __ffs(gt) - 1;
      lo += j * stride;
      n = min(stride, n - j * stride);
    }
    r_base = lo;
  }
#pragma unroll 1
  for (int ch = 0; ch < EMIT_CHUNKS; ch++) {
    const uint32_t s0 = s_begin + 32u * ch;
    if (s0 >= cap) break;
    if (s0 >= R) {  // padding only
      if (s0 + lane < cap) { keys[s0 + lane] = pad_key; vals[s0 + lane] = 0u; }
      continue;
    }
    // r_base = smallest rank with offsets[r_base] > s0; 32 consecutive slots span at most 32 visible ranks
    const uint32_t oj = __ldg(offsets + min(r_base + lane, P - 1));
    const uint32_t s = min(s0 + lane, R - 1);
    int c = 0;  // number of probed offsets <= s  (0..31)
#pragma unroll
    for (int step = 16; step > 0; step >>= 1) {
      const uint32_t e = __shfl_sync(F, oj, c + step - 1);
      if (e <= s) c += step;
    }
    const uint32_t end = __shfl_sync(F, oj, c);
    const int rank = min(r_base + c, P - 1);
    const uint32_t idx = order[rank];
    const uint32_t start = end - tiles_touched[idx];
    const float4 q0 = __ldg(reinterpret_cast<const float4*>(records + idx));
    uint2 rmin, rmax;
    tile_rect(q0.x, q0.y, radii[idx], gx, gy, rmin, rmax);
    const uint32_t w = max(rmax.x - rmin.x, 1u);
    const uint32_t k = s - start;
    const uint32_t ry = k / w, rx = k - ry * w;
    uint32_t y0, ny;
    owned_rows(rmin.y, rmax.y, own_stride, own_phase, y0, ny);
    if (s0 + lane < R) {
      keys[s] = (KeyT)((y0 + ry * (uint32_t)own_stride) * gx + (rmin.x + rx));
      vals[s] = idx;
    } else if (s0 + lane < cap) {
      keys[s0 + lane] = pad_key;
      vals[s0 + lane] = 0u;
    }
    // next chunk starts at s0 + 32: the owner of slot s0+31 still owns it unless its range ends exactly there
    const uint32_t end31 = __shfl_sync(F, end, 31);
    const int rank31 = __shfl_sync(F, rank, 31);
    r_base = rank31 + (end31 <= s0 + 32u ? 1 : 0);
  }
}

// rasterizer_impl.cu:105-125 on 16/32-bit tile keys; ranges must be zeroed beforehand (:263-265). Each thread owns
// RANGE_ITEMS consecutive keys (one 128-bit load for 16-bit keys) plus its left neighbour.
constexpr int RANGE_ITEMS = 8;
template <typename KeyT>
__global__ void tile_ranges_kernel(int cap, const uint32_t* __restrict__ R_dev, const KeyT* __restrict__ keys,
                                   uint2* __restrict__ ranges) {
  const int L = R_dev ? (int)min(__ldg(R_dev), (uint32_t)cap) : cap;  // padding slots [L, cap) carry no tile
  const int base = (blockIdx.x * blockDim.x + threadIdx.x) * RANGE_ITEMS;
  if (base >= L) return;
  KeyT k[RANGE_ITEMS];
  if (sizeof(KeyT) == 2 && base + RANGE_ITEMS <= cap) {  // workspace arrays are 256-byte aligned, base*2 is 16-byte aligned
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(keys + base));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < RANGE_ITEMS; i++) k[i] = (KeyT)((w[i >> 1] >> (16 * (i & 1))) & 0xFFFFu);
  } else {
#pragma unroll
    for (int i = 0; i < RANGE_ITEMS; i++) k[i] = base + i < L ? keys[base + i] : (KeyT)0;
  }
  uint32_t prev = base > 0 ? (uint32_t)keys[base - 1] : 0u;
#pragma unroll
  for (int i = 0; i < RANGE_ITEMS; i++) {
    const int idx = base + i;
    if (idx < L) {
      const uint32_t cur = (uint32_t)k[i];
      if (idx == 0)
        ranges[cur].x = 0;
      else if (cur != prev) {
        ranges[prev].y = idx;
        ranges[cur].x = idx;
      }
      if (idx == L - 1) ranges[cur].y = L;
      prev = cur;
    }
  }
}

// Static-capacity forward: the host never learns R, so the device reports it. When R exceeds the capacity the lists
// were sized for, the tile-binning path has already left every range empty (tile_prefix_kernel) but the CUB path holds
// the first `cap` instances in sorted order; both are reduced to the same empty frame here, before the render: zero
// ranges (colour = background, depth = 0, alpha = 0) and zero per-Gaussian tile counts, so that the deterministic
// reduction, whose runs [excl, excl + tiles_touched) would reach past the capacity, has nothing to read.
constexpr int STATUS_THREADS = 256;
__global__ void __launch_bounds__(STATUS_THREADS)
static_status_kernel(int P, int ntile, uint32_t cap, const uint32_t* __restrict__ R_dev, uint2* __restrict__ ranges,
                     uint32_t* __restrict__ tiles_touched, int32_t* __restrict__ status) {
  const uint32_t R = __ldg(R_dev);
  const bool overflow = R > cap;
  const int i0 = blockIdx.x * STATUS_THREADS + threadIdx.x;
  if (i0 == 0) {
    status[0] = (int32_t)R;
    status[1] = overflow ? 1 : 0;
  }
  if (!overflow) return;
  for (int i = i0; i < max(P, ntile); i += gridDim.x * STATUS_THREADS) {
    if (i < ntile) ranges[i] = make_uint2(0u, 0u);
    if (i < P) tiles_touched[i] = 0u;
  }
}

// Static-capacity sharded forward: static_status_kernel for one rank's owned tiles, plus (sparse exchange,
// counts_matrix != null) the segment check: a segment of more than seg_cap records was truncated by the push, so this
// rank's candidate lists are incomplete. The matrix is the same on every rank after the barrier that carried its rows,
// so every rank finds a segment overflow alike; an R overflow is local and is made global by the gate below.
// status = {R, overflow, largest segment (0 without a matrix), 0}; word 3 is the gate's.
__global__ void __launch_bounds__(STATUS_THREADS)
shard_static_status_kernel(int P, int ntile, uint32_t cap, const uint32_t* __restrict__ R_dev,
                           const int32_t* __restrict__ counts_matrix, int world, int seg_cap, uint2* __restrict__ ranges,
                           uint32_t* __restrict__ tiles_touched, int32_t* __restrict__ status) {
  const uint32_t R = __ldg(R_dev);
  int max_count = 0;
  if (counts_matrix)
    for (int k = 0; k < world * GSR_MAX_PEERS; k++) max_count = max(max_count, counts_matrix[k]);
  const bool overflow = R > cap || max_count > seg_cap;
  const int i0 = blockIdx.x * STATUS_THREADS + threadIdx.x;
  if (i0 == 0) {
    status[0] = (int32_t)R;
    status[1] = overflow ? 1 : 0;
    status[2] = max_count;
    status[3] = 0;
  }
  if (!overflow) return;
  for (int i = i0; i < max(P, ntile); i += gridDim.x * STATUS_THREADS) {
    if (i < ntile) ranges[i] = make_uint2(0u, 0u);
    if (i < P) tiles_touched[i] = 0u;
  }
}

// The overflow consensus of the static sharded forward, after the frame exchange: `flags` [nflags] (the ranks' overflow
// words, delivered through the frame barrier) or `flag_sum` (the exact float sum of the ranks' 0/1 flags that rode the
// frame all-reduce). If any rank overflowed, every rank gets the same empty frame -- colour = background, depth and
// alpha 0 -- and its owned tiles are emptied, so every backward writes zeros: zero ranges and tile counts, and zero
// tile_last, where the blending backward starts its walk (the forward has already run on the full lists here).
// status[1] = the global flag, status[3] = the barrier error word (0 without one).
__global__ void __launch_bounds__(STATUS_THREADS)
shard_static_gate_kernel(int P, int ntile, int npix, int planes, const int32_t* __restrict__ flags, int nflags,
                         const float* __restrict__ flag_sum, const uint32_t* __restrict__ error_word,
                         const float* __restrict__ bg, uint2* __restrict__ ranges, uint32_t* __restrict__ tile_last,
                         uint32_t* __restrict__ tiles_touched, float* __restrict__ frame, int32_t* __restrict__ status) {
  bool any = flag_sum != nullptr && *flag_sum != 0.f;
  for (int r = 0; r < nflags; r++) any |= flags[r] != 0;
  const int i0 = blockIdx.x * STATUS_THREADS + threadIdx.x;
  if (i0 == 0) {
    status[1] = any ? 1 : 0;
    status[3] = error_word ? (int32_t)*error_word : 0;
  }
  if (!any) return;
  const long long nframe = (long long)npix * planes;
  const long long n = max((long long)max(P, ntile), nframe);
  for (long long i = i0; i < n; i += (long long)gridDim.x * STATUS_THREADS) {
    if (i < ntile) {
      ranges[i] = make_uint2(0u, 0u);
      tile_last[i] = 0u;
    }
    if (i < P) tiles_touched[i] = 0u;
    if (i < nframe) {
      const int plane = (int)(i / npix);
      frame[i] = plane < 3 ? __ldg(bg + plane) : 0.f;
    }
  }
}

// CUB's temp-size queries depend only on the item count but cost several runtime calls each; every C-ABI entry point
// re-derives the workspace layout, so they are memoised (single-threaded callers per the ABI; a mutex keeps it safe).
struct SizeCache {
  std::mutex mu;
  std::unordered_map<long long, size_t> m;
  template <typename Fn> size_t get(int kind, long long n, Fn fn) {
    std::lock_guard<std::mutex> lk(mu);
    const long long key = n * 4 + kind;
    auto it = m.find(key);
    if (it != m.end()) return it->second;
    const size_t v = fn();
    if (cudaPeekAtLastError() == cudaSuccess) m[key] = v;
    return v;
  }
};
SizeCache g_sizes;

size_t depth_sort_temp_bytes(int P) {
  return g_sizes.get(0, P, [&] {
    size_t n = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, n, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, P);
    return n;
  });
}
size_t scan_temp_bytes(int P) {
  return g_sizes.get(1, P, [&] {
    size_t n = 0;
    cub::TransformInputIterator<uint32_t, GatherTilesOp, cub::CountingInputIterator<uint32_t>> it(
        cub::CountingInputIterator<uint32_t>(0), GatherTilesOp{nullptr, nullptr});
    cub::DeviceScan::InclusiveSum(nullptr, n, it, (uint32_t*)nullptr, P);
    return n;
  });
}
// R changes with every frame: the CUB size is queried for R rounded up to a 64K bucket (monotone in the item count),
// so a long session fills a handful of cache entries instead of one per frame.
size_t tile_sort_temp_bytes(int64_t R_exact) {
  const int64_t R = (R_exact + 65535) / 65536 * 65536;
  return g_sizes.get(2, R, [&] {
    size_t n = 0, m = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, n, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)R, 0, 32);
    cub::DeviceRadixSort::SortPairs(nullptr, m, (const uint16_t*)nullptr, (uint16_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)R, 0, 16);
    return n > m ? n : m;
  });
}

template <typename KeyT>
int bin_typed(const gsr_cloud& c, int R, bool speculative, int gx, int gy, const GeometryWS& g, const BinningWS& b,
              const ImageWS& im, const int32_t* radii, cudaStream_t st, bool debug, const TileOwner& own) {
  const uint32_t* R_dev = speculative ? g.offsets + (c.P - 1) : nullptr;
  const int bit = (int)higher_msb((uint32_t)(gx * gy));
  const KeyT pad_key = (KeyT)((1u << bit) - 1u);  // > every tile id (ids <= Ntile-1 <= 2^bit - 2), inside the sorted bits
  KeyT* ku = reinterpret_cast<KeyT*>(b.keys_unsorted);
  KeyT* ks = reinterpret_cast<KeyT*>(b.keys_sorted);
  int rc;
  {
    StageScope t(ST_EMIT, st);
    emit_instances_kernel<KeyT><<<(R + EMIT_THREADS * EMIT_CHUNKS - 1) / (EMIT_THREADS * EMIT_CHUNKS), EMIT_THREADS, 0, st>>>(
        c.P, (uint32_t)R, R_dev, pad_key, g.depth_order, g.offsets, g.tiles_touched, g.records, radii, gx, gy, own.stride,
        own.phase, ku, b.vals_unsorted);
    g_launches++;
    rc = check_launch("emit_instances", debug, st);
    if (rc) return rc;
  }
  {
    StageScope t(ST_TILE_SORT, st);
    size_t tb = b.cub_temp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(b.cub_temp, tb, (const KeyT*)ku, ks, (const uint32_t*)b.vals_unsorted,
                                                    b.point_list, R, 0, bit, st);
    g_launches += 4;
    if (e != cudaSuccess) return check_cuda(e, "tile sort");
  }
  StageScope t(ST_RANGES, st);
  tile_ranges_kernel<KeyT><<<(R + 256 * RANGE_ITEMS - 1) / (256 * RANGE_ITEMS), 256, 0, st>>>(R, R_dev, ks, im.ranges);
  g_launches++;
  return check_launch("tile_ranges", debug, st);
}

}  // namespace

bool carve_geometry(void* base, int P, GeometryWS& ws) {
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) {
    void* p = b ? (void*)(b + off) : nullptr;
    off += align_up(bytes ? bytes : 1);
    return p;
  };
  const size_t n = (size_t)(P > 0 ? P : 1);
  ws.records = (SplatRecord*)take(n * sizeof(SplatRecord));
  ws.tiles_touched = (uint32_t*)take(n * 4);
  ws.clamped = (uint8_t*)take(n);
  ws.depth_keys = (uint32_t*)take(n * 4);
  ws.ident = (uint32_t*)take(n * 4);
  ws.depth_keys_sorted = (uint32_t*)take(n * 4);
  ws.depth_order = (uint32_t*)take(n * 4);
  ws.offsets = (uint32_t*)take(n * 4);
  ws.R_dev = (uint32_t*)take(16 + (size_t)MAX_TILE_DIFF * sizeof(int32_t));  // one block: R, then the array
  ws.tile_diff = reinterpret_cast<int32_t*>(ws.R_dev + 4);
  size_t t1 = depth_sort_temp_bytes((int)n), t2 = scan_temp_bytes((int)n);
  if (cudaPeekAtLastError() != cudaSuccess) {
    check_cuda(cudaGetLastError(), "CUB temp-size query");
    return false;
  }
  ws.cub_temp_bytes = t1 > t2 ? t1 : t2;
  const size_t t3 = depth_sort_scratch_bytes((int)n);  // depth_sort.cu (default depth order): status words + ping-pong arrays
  if (t3 > ws.cub_temp_bytes) ws.cub_temp_bytes = t3;
  ws.cub_temp = take(ws.cub_temp_bytes);
  ws.total = off;
  return true;
}

bool carve_binning(void* base, int P, int64_t R, int W, int H, BinningWS& ws) {
  (void)P;
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) {
    void* p = b ? (void*)(b + off) : nullptr;
    off += align_up(bytes ? bytes : 1);
    return p;
  };
  const size_t n = (size_t)(R > 0 ? R : 1);
  ws.keys_unsorted = (uint32_t*)take(n * 4);
  ws.keys_sorted = (uint32_t*)take(n * 4);
  ws.vals_unsorted = (uint32_t*)take(n * 4);
  ws.point_list = (uint32_t*)take(n * 4);
  ws.cub_temp_bytes = tile_sort_temp_bytes((int64_t)n);
  if (cudaPeekAtLastError() != cudaSuccess) {
    check_cuda(cudaGetLastError(), "CUB temp-size query");
    return false;
  }
  ws.cub_temp = take(ws.cub_temp_bytes);
  // tile_binning.cu: tickets + digit bases (1024 words), two passes of per-sort-tile status words, 2-D count scratch
  const size_t gx = (size_t)(W + TILE - 1) / TILE, gy = (size_t)(H + TILE - 1) / TILE;
  const size_t ntiles = (n + SORT_TILE - 1) / SORT_TILE;
  ws.sort_state_bytes = (1024 + 2 * ntiles * 256 + (gx + 1) * (gy + 1)) * sizeof(uint32_t);
  ws.sort_state = (uint32_t*)take(ws.sort_state_bytes);
  ws.total = off;
  return true;
}

void carve_image(void* base, int W, int H, ImageWS& ws) {
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) {
    void* p = b ? (void*)(b + off) : nullptr;
    off += align_up(bytes ? bytes : 1);
    return p;
  };
  const size_t npix = (size_t)W * H;
  const size_t ntile = (size_t)((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
  ws.final_T = (float*)take(npix * 4);
  ws.n_contrib = (uint32_t*)take(npix * 4);
  ws.ranges = (uint2*)take(ntile * 8);
  ws.tile_last = (uint32_t*)take(ntile * 4);
  ws.total = off;
}

int run_depth_order_and_scan(const gsr_cloud& c, const GeometryWS& g, int32_t* num_rendered_host, cudaStream_t st,
                             bool debug) {
  // num_rendered_host == nullptr: the caller already fetched the count from g.R_dev (tile_binning path)
  const int P = c.P;
  if (g_opt.depth_sort_variant == 1) {
    int rc = run_depth_sort_own(P, g, st, debug);
    if (rc) return rc;
    if (num_rendered_host) {
      cudaError_t e2 = cudaMemcpyAsync(num_rendered_host, g.offsets + (P - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st);
      if (e2 != cudaSuccess) return check_cuda(e2, "num_rendered readback");
    }
    return GSR_OK;
  }
  size_t tb = g.cub_temp_bytes;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(g.cub_temp, tb, (const uint32_t*)g.depth_keys, g.depth_keys_sorted,
                                                  (const uint32_t*)g.ident, g.depth_order, P, 0, 32, st);
  g_launches += 5;
  if (e != cudaSuccess) return check_cuda(e, "depth sort");
  cub::TransformInputIterator<uint32_t, GatherTilesOp, cub::CountingInputIterator<uint32_t>> it(
      cub::CountingInputIterator<uint32_t>(0), GatherTilesOp{g.tiles_touched, g.depth_order});
  tb = g.cub_temp_bytes;
  e = cub::DeviceScan::InclusiveSum(g.cub_temp, tb, it, g.offsets, P, st);
  g_launches += 2;
  if (e != cudaSuccess) return check_cuda(e, "tile-count scan");
  if (num_rendered_host) {
    e = cudaMemcpyAsync(num_rendered_host, g.offsets + (P - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return check_cuda(e, "num_rendered readback");
  }
  return check_launch("depth order + scan", debug, st);
}

int run_binning(const gsr_settings& s, const gsr_cloud& c, int R, bool speculative, const GeometryWS& g,
                const BinningWS& b, const ImageWS& im, const int32_t* radii, cudaStream_t st, const TileOwner& own) {
  const int W = s.image_width, H = s.image_height;
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  const bool debug = s.debug != 0;
  if (R > 0 && R < (1 << 30) && tile_binning_supported(gx, gy)) return run_tile_binning(s, c.P, R, speculative, g, b, im, radii, st, own);
  cudaError_t e = cudaMemsetAsync(im.ranges, 0, (size_t)gx * gy * sizeof(uint2), st);
  if (e != cudaSuccess) return check_cuda(e, "ranges memset");
  if (R <= 0) return GSR_OK;
  // tile ids (and the padding key 2^bit - 1 > Ntile - 1) fit 16 bits up to 65535 tiles: half the key traffic of the sort
  if ((int64_t)gx * gy < 65536 && g_opt.tile_key_bits == 16)
    return bin_typed<uint16_t>(c, R, speculative, gx, gy, g, b, im, radii, st, debug, own);
  return bin_typed<uint32_t>(c, R, speculative, gx, gy, g, b, im, radii, st, debug, own);
}

int launch_static_status(const gsr_settings& s, int P, uint32_t capacity, const GeometryWS& g, const ImageWS& im,
                         int32_t* status, cudaStream_t st) {
  const int gx = (s.image_width + TILE - 1) / TILE, gy = (s.image_height + TILE - 1) / TILE;
  // the count run_binning compared against the capacity: tile_count_kernel's on the tile-binning path, else the scan's
  const uint32_t* R_dev = tile_binning_supported(gx, gy) ? g.R_dev : g.offsets + (P - 1);
  const int n = P > gx * gy ? P : gx * gy;
  const int blocks = std::min((n + STATUS_THREADS - 1) / STATUS_THREADS, 1024);
  static_status_kernel<<<blocks, STATUS_THREADS, 0, st>>>(P, gx * gy, capacity, R_dev, im.ranges, g.tiles_touched, status);
  g_launches++;
  return check_launch("static_status", s.debug != 0, st);
}

int launch_shard_static_status(const gsr_settings& s, int P, uint32_t capacity, const GeometryWS& g, const ImageWS& im,
                               const int32_t* counts_matrix, int world, int seg_cap, int32_t* status, cudaStream_t st) {
  const int gx = (s.image_width + TILE - 1) / TILE, gy = (s.image_height + TILE - 1) / TILE;
  const uint32_t* R_dev = tile_binning_supported(gx, gy) ? g.R_dev : g.offsets + (P - 1);  // as launch_static_status
  const int n = P > gx * gy ? P : gx * gy;
  const int blocks = std::min((n + STATUS_THREADS - 1) / STATUS_THREADS, 1024);
  shard_static_status_kernel<<<blocks, STATUS_THREADS, 0, st>>>(P, gx * gy, capacity, R_dev, counts_matrix, world,
                                                                seg_cap, im.ranges, g.tiles_touched, status);
  g_launches++;
  return check_launch("shard_static_status", s.debug != 0, st);
}

int launch_shard_static_gate(const gsr_settings& s, int P, const GeometryWS& g, const ImageWS& im, const int32_t* flags,
                             int nflags, const float* flag_sum, const uint32_t* error_word, float* frame, int planes,
                             int32_t* status, cudaStream_t st) {
  const int gx = (s.image_width + TILE - 1) / TILE, gy = (s.image_height + TILE - 1) / TILE;
  const long long npix = (long long)s.image_width * s.image_height;
  const long long n = std::max<long long>(std::max(P, gx * gy), npix * planes);
  const int blocks = (int)std::min<long long>((n + STATUS_THREADS - 1) / STATUS_THREADS, 1024);
  shard_static_gate_kernel<<<blocks, STATUS_THREADS, 0, st>>>(P, gx * gy, (int)npix, planes, flags, nflags, flag_sum,
                                                              error_word, s.bg, im.ranges, im.tile_last, g.tiles_touched, frame,
                                                              status);
  g_launches++;
  return check_launch("shard_static_gate", s.debug != 0, st);
}

int launch_retouch(const gsr_settings& s, int P, const GeometryWS& g, int32_t* radii, const TileOwner& own,
                   cudaStream_t st) {
  const int gx = (s.image_width + TILE - 1) / TILE, gy = (s.image_height + TILE - 1) / TILE;
  const bool v2 = tile_binning_supported(gx, gy);
  if (v2) {
    int rc = clear_tile_counts(g, gx, gy, st);
    if (rc) return rc;
  }
  retouch_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, g.records, gx, gy, own.stride, own.phase, radii, g.tiles_touched,
                                                  g.ident, g.depth_keys, v2 ? g.tile_diff : nullptr, tile_diff_copies(gx, gy));
  g_launches++;
  return check_launch("retouch", s.debug != 0, st);
}

}  // namespace gsr
