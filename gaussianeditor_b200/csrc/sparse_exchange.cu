// Sparse exchange of the Gaussian-sharded multi-GPU path (BASELINE config 4, SURVEY.md 8(e)) for sm_90a.
//
// The dense scheme of gsr_shard_* sends every 48-byte splat record to every rank, depth-sorts all P keys on every
// rank and reduce-scatters all P gradient rows (three P-sized steps that do not shrink with the number of GPUs).
// Here a record travels only to the ranks whose tile rows its rectangle touches:
//
//   owner s (index decomposition)                              tile owner d (tile-row decomposition)
//   preprocess shard -> records[n_s], dest_mask[n_s]
//   scan: ordered slot of Gaussian i in the list L[s->d]
//   push: record -> cand_d[s*cap + slot]        ---NVLink--->  candidates = G segments of capacity `cap`, in
//                                                               (source, slot) = GLOBAL INDEX order; unused slots are
//                                                               holes ("culled" sort key) -> the stable 32-bit depth
//                                                               sort still yields the reference's (depth, index) order
//                                                               retouch -> depth sort -> scan -> bin -> blend  (existing
//                                                               stages on a cloud of G*cap candidates)
//   gather: acc_slice[i] = sum over d of ret[d][slot]  <------  blend backward -> acc[G*cap, 12] -> return push of the
//   (fixed rank order: deterministic)                           segment of source s into ret_s[d*cap ...]
//   fused preprocess backward of the shard
//
// Counts n[s->d] travel in one [G,G] int matrix: every rank writes its row into every peer's copy inside the
// cross-rank barrier that follows the push (gsr_peer_barrier, flag words in peer memory; virtual ranks and the gloo
// tests sum the rows on the host instead); a segment that overflows `cap` is detected from that matrix on every rank
// alike and the step is redone with a larger capacity.
//
// Everything except the peer transport is testable with VIRTUAL ranks on one GPU: peer pointers are then just other
// buffers of the same device (tests/test_sharded.py).
#include <algorithm>
#include <cstddef>

#include "common.cuh"

namespace gsr {

namespace {

constexpr int SP_THREADS = 128;  // Gaussians per block in every per-Gaussian kernel below (one partition for all)

struct SparseLocal {   // extra per-owner arrays behind the GeometryWS of the shard
  uint8_t* dest_mask;  // [n]   bit d: the Gaussian's tile rectangle has a row owned by rank d (0 = culled)
  uint32_t* blk_base;  // [nblocks, 8] exclusive prefix (over blocks, index order) of the per-dest counts
  int32_t* counts;     // [8]   totals n[this rank -> d]
  size_t total;
};

size_t carve_sparse_local(void* base, int n, const GeometryWS& g, SparseLocal& sl) {
  size_t off = g.total;
  char* b = (char*)base;
  auto take = [&](size_t bytes) {
    void* p = b ? (void*)(b + off) : nullptr;
    off += align_up(bytes ? bytes : 1);
    return p;
  };
  const size_t nb = (size_t)(n + SP_THREADS - 1) / SP_THREADS;
  sl.dest_mask = (uint8_t*)take((size_t)(n > 0 ? n : 1));
  sl.blk_base = (uint32_t*)take((nb ? nb : 1) * GSR_MAX_PEERS * sizeof(uint32_t));
  sl.counts = (int32_t*)take(GSR_MAX_PEERS * sizeof(int32_t));
  sl.total = off;
  return off;
}

// candidate workspace = GeometryWS(world*cap) | ret [world*cap, 12] floats (written by the tile owners in the backward)
struct SparseCand {
  GeometryWS g;
  float* ret;
  size_t total;
};
bool carve_sparse_cand(void* base, int world, int cap, SparseCand& sc) {
  const int M = world * cap;
  if (!carve_geometry(base, M, sc.g)) return false;
  size_t off = sc.g.total;
  sc.ret = base ? (float*)((char*)base + off) : nullptr;
  off += align_up((size_t)(M > 0 ? M : 1) * ACC_STRIDE * sizeof(float));
  sc.total = off;
  return true;
}

__device__ __forceinline__ void tile_rect_rows(float py, int radius, int gy, uint32_t& ymin, uint32_t& ymax) {
  ymin = (unsigned)min(gy, max((int)0, (int)((py - radius) / TILE)));
  ymax = (unsigned)min(gy, max((int)0, (int)((py + radius + TILE - 1) / TILE)));
}

// ---- owner side, forward -------------------------------------------------------------------------------
// dest_mask from the records the preprocess kernel wrote (radius in q2.w, centre in q0), and the per-destination counts
// of this block of SP_THREADS Gaussians (-> blk_base[block], turned into an exclusive prefix by sparse_scan_kernel).
__global__ void __launch_bounds__(SP_THREADS)
sparse_mask_kernel(int n, const SplatRecord* __restrict__ records, int gx, int gy, int world, uint8_t* __restrict__ dest_mask,
                   uint32_t* __restrict__ blk_cnt) {
  __shared__ uint32_t s_cnt[SP_THREADS / 32][GSR_MAX_PEERS];
  const int idx = blockIdx.x * SP_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t m = 0;
  if (idx < n) {
    const float4* r = reinterpret_cast<const float4*>(records + idx);
    const int radius = __float_as_int(__ldg(r + 2).w);
    if (radius > 0) {
      const float4 q0 = __ldg(r);
      uint32_t ymin, ymax;
      tile_rect_rows(q0.y, radius, gy, ymin, ymax);
      const uint32_t xmin = (unsigned)min(gx, max((int)0, (int)((q0.x - radius) / TILE)));
      const uint32_t xmax = (unsigned)min(gx, max((int)0, (int)((q0.x + radius + TILE - 1) / TILE)));
      if (xmax > xmin && ymax > ymin) {
        if (ymax - ymin >= (uint32_t)world) m = (1u << world) - 1u;
        else
          for (uint32_t y = ymin; y < ymax; y++) m |= 1u << (y % (uint32_t)world);
      }
    }
    dest_mask[idx] = (uint8_t)m;
  }
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) {
    const uint32_t bal = __ballot_sync(0xffffffffu, (m >> d) & 1u);
    if (lane == 0) s_cnt[warp][d] = __popc(bal);
  }
  __syncthreads();
  if (threadIdx.x < GSR_MAX_PEERS) {
    uint32_t c = 0;
#pragma unroll
    for (int w = 0; w < SP_THREADS / 32; w++) c += s_cnt[w][threadIdx.x];
    blk_cnt[(size_t)blockIdx.x * GSR_MAX_PEERS + threadIdx.x] = c;
  }
}

// One CTA: exclusive scan (over the blocks, in index order) of the per-block per-destination counts, in place.
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS)
sparse_scan_kernel(int n, int world, uint32_t* __restrict__ blk_base, int32_t* __restrict__ counts) {
  __shared__ uint32_t s_warp[SCAN_THREADS / 32][GSR_MAX_PEERS];
  __shared__ uint32_t s_carry[GSR_MAX_PEERS];
  const int nblocks = (n + SP_THREADS - 1) / SP_THREADS;
  const int per = (nblocks + SCAN_THREADS - 1) / SCAN_THREADS;  // consecutive blocks per thread
  const int b0 = threadIdx.x * per, b1 = min(nblocks, b0 + per);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto block_counts = [&](int b, uint32_t* c) {
    const uint4 v0 = *reinterpret_cast<const uint4*>(blk_base + (size_t)b * GSR_MAX_PEERS);
    const uint4 v1 = *(reinterpret_cast<const uint4*>(blk_base + (size_t)b * GSR_MAX_PEERS) + 1);
    c[0] = v0.x; c[1] = v0.y; c[2] = v0.z; c[3] = v0.w; c[4] = v1.x; c[5] = v1.y; c[6] = v1.z; c[7] = v1.w;
  };
  uint32_t mine[GSR_MAX_PEERS];
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) mine[d] = 0;
  for (int b = b0; b < b1; b++) {
    uint32_t c[GSR_MAX_PEERS];
    block_counts(b, c);
#pragma unroll
    for (int d = 0; d < GSR_MAX_PEERS; d++) mine[d] += c[d];
  }
  // exclusive scan of `mine` over the threads
  uint32_t excl[GSR_MAX_PEERS];
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) {
    uint32_t v = mine[d];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    if (lane == 31) s_warp[warp][d] = v;
    excl[d] = v - mine[d];
  }
  __syncthreads();
  if (threadIdx.x < GSR_MAX_PEERS) {
    uint32_t run = 0;
    for (int w = 0; w < SCAN_THREADS / 32; w++) {
      const uint32_t t = s_warp[w][threadIdx.x];
      s_warp[w][threadIdx.x] = run;
      run += t;
    }
    s_carry[threadIdx.x] = run;
  }
  __syncthreads();
  uint32_t run[GSR_MAX_PEERS];
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) run[d] = excl[d] + s_warp[warp][d];
  for (int b = b0; b < b1; b++) {
    uint32_t c[GSR_MAX_PEERS];
    block_counts(b, c);
    uint4* o = reinterpret_cast<uint4*>(blk_base + (size_t)b * GSR_MAX_PEERS);
    o[0] = make_uint4(run[0], run[1], run[2], run[3]);
    o[1] = make_uint4(run[4], run[5], run[6], run[7]);
#pragma unroll
    for (int d = 0; d < GSR_MAX_PEERS; d++) run[d] += c[d];
  }
  if (threadIdx.x < GSR_MAX_PEERS) counts[threadIdx.x] = threadIdx.x < world ? (int32_t)s_carry[threadIdx.x] : 0;
}

// Ordered slot of this thread's Gaussian in each destination list: blk_base + rank inside the block. All SP_THREADS
// threads of the block must call it. slot[d] is only meaningful where bit d of `m` is set.
__device__ __forceinline__ void sparse_slots(uint32_t m, int world, const uint32_t* __restrict__ blk_base, uint32_t* slot,
                                             uint32_t (*s_cnt)[GSR_MAX_PEERS]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t in_warp[GSR_MAX_PEERS];
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) {
    const uint32_t bal = __ballot_sync(0xffffffffu, (m >> d) & 1u);
    in_warp[d] = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) s_cnt[warp][d] = __popc(bal);
  }
  __syncthreads();
  const uint4 b0 = __ldg(reinterpret_cast<const uint4*>(blk_base + (size_t)blockIdx.x * GSR_MAX_PEERS));
  const uint4 b1 = __ldg(reinterpret_cast<const uint4*>(blk_base + (size_t)blockIdx.x * GSR_MAX_PEERS) + 1);
  const uint32_t base[GSR_MAX_PEERS] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) {
    uint32_t before = 0;
#pragma unroll
    for (int w = 0; w < SP_THREADS / 32; w++) before += w < warp ? s_cnt[w][d] : 0u;
    slot[d] = base[d] + before + in_warp[d];
  }
  (void)world;
}

struct PushArgs {
  int n, world, rank, cap;
  const SplatRecord* records;
  const uint8_t* dest_mask;
  const uint32_t* blk_base;
  SplatRecord* peer_records[GSR_MAX_PEERS];  // candidate records array of every rank (as mapped here)
};

// The collective: every Gaussian's record goes to slot rank*cap + slot_d of every destination d in its mask, straight
// into that rank's memory over NVLink peer mappings. The records a warp sends to one destination occupy CONSECUTIVE
// slots there, so the warp first compacts them in its shared-memory stage and then copies the run with consecutive
// 16-byte chunks per lane: every store instruction covers 512 contiguous bytes (full 128-byte lines on the wire).
// The first version stored each thread's own record (three 16-byte stores at a 48-byte stride): 16-byte payloads in
// 32-byte sectors reached a third of the link rate (0.36 ms for 93 MB per rank at config 4 on 4 GPUs).
__global__ void __launch_bounds__(SP_THREADS) sparse_push_kernel(const PushArgs a) {
  __shared__ uint32_t s_cnt[SP_THREADS / 32][GSR_MAX_PEERS];
  __shared__ float4 s_stage[SP_THREADS / 32][32 * 3];
  const int idx = blockIdx.x * SP_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t m = idx < a.n ? a.dest_mask[idx] : 0u;
  uint32_t bal[GSR_MAX_PEERS];
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) {
    bal[d] = __ballot_sync(0xffffffffu, (m >> d) & 1u);
    if (lane == 0) s_cnt[warp][d] = __popc(bal[d]);
  }
  __syncthreads();
  float4 q0 = make_float4(0.f, 0.f, 0.f, 0.f), q1 = q0, q2 = q0;
  if (m != 0) {
    const float4* r = reinterpret_cast<const float4*>(a.records + idx);
    q0 = __ldg(r); q1 = __ldg(r + 1); q2 = __ldg(r + 2);
  }
  const uint4 b0 = __ldg(reinterpret_cast<const uint4*>(a.blk_base + (size_t)blockIdx.x * GSR_MAX_PEERS));
  const uint4 b1 = __ldg(reinterpret_cast<const uint4*>(a.blk_base + (size_t)blockIdx.x * GSR_MAX_PEERS) + 1);
  const uint32_t base[GSR_MAX_PEERS] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  float4* stage = s_stage[warp];
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) {
    if (bal[d] == 0) continue;  // warp-uniform
    uint32_t slot0 = base[d];   // first slot (in this destination's segment) of the run this warp sends
#pragma unroll
    for (int w = 0; w < SP_THREADS / 32; w++) slot0 += w < warp ? s_cnt[w][d] : 0u;
    if ((m >> d) & 1u) {
      const int r = __popc(bal[d] & ((1u << lane) - 1u));
      stage[3 * r] = q0; stage[3 * r + 1] = q1; stage[3 * r + 2] = q2;
    }
    __syncwarp();
    // overflow (slot >= cap): dropped here, detected from the counts on every rank alike
    const uint32_t room = slot0 < (uint32_t)a.cap ? (uint32_t)a.cap - slot0 : 0u;
    const uint32_t nrec = min((uint32_t)__popc(bal[d]), room);
    float4* dst = reinterpret_cast<float4*>(a.peer_records[d]) + ((size_t)a.rank * a.cap + slot0) * 3;
    for (uint32_t t = lane; t < 3u * nrec; t += 32) dst[t] = stage[t];
    __syncwarp();
  }
}

// ---- tile-owner side ------------------------------------------------------------------------------------
// Per candidate slot: valid slots (j < n[s -> me]) get radius / owned-tile count / depth key from the record, holes
// get the culled key and zero tiles (the depth sort then puts them behind every candidate that emits instances).
__global__ void retouch_sparse_kernel(int world, int cap, int me, const int32_t* __restrict__ counts_matrix,
                                      const SplatRecord* __restrict__ records, int gx, int gy, int32_t* __restrict__ radii,
                                      uint32_t* __restrict__ tiles_touched, uint32_t* __restrict__ ident,
                                      uint32_t* __restrict__ depth_keys, int32_t* __restrict__ tile_diff, int diff_copies) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = c < world * cap;
  const int s = live ? c / cap : 0, j = c - s * cap;
  const int cnt = live ? min(counts_matrix[s * GSR_MAX_PEERS + me], cap) : 0;
  int radius = 0;
  uint32_t n = 0, key = 0xFFFFFFFFu;
  if (live && j < cnt) {
    const float4* r = reinterpret_cast<const float4*>(records + c);
    radius = __float_as_int(__ldg(r + 2).w);
    if (radius > 0) {
      const float4 q0 = __ldg(r);
      uint32_t ymin, ymax;
      tile_rect_rows(q0.y, radius, gy, ymin, ymax);
      const uint32_t xmin = (unsigned)min(gx, max((int)0, (int)((q0.x - radius) / TILE)));
      const uint32_t xmax = (unsigned)min(gx, max((int)0, (int)((q0.x + radius + TILE - 1) / TILE)));
      int dd = (me - (int)ymin) % world;
      if (dd < 0) dd += world;
      const uint32_t y0 = ymin + (uint32_t)dd;
      const uint32_t ny = y0 < ymax ? (ymax - y0 + (uint32_t)world - 1u) / (uint32_t)world : 0u;
      n = ny * (xmax - xmin);
      if (n != 0) {
        key = __float_as_uint(__ldg(r + 1).z);
        // full rectangle; tile_prefix_kernel keeps the owned rows
        if (tile_diff) add_tile_rect(tile_diff, gx, gy, diff_copies, (uint32_t)c, xmin, ymin, xmax, ymax);
      }
    }
  }
  if (live) {
    radii[c] = n != 0 ? radius : 0;
    tiles_touched[c] = n;
    ident[c] = (uint32_t)c;
    depth_keys[c] = key;
  }
}

// overflow / bookkeeping word for the host: max over all (s, d) of n[s -> d]
__global__ void sparse_max_count_kernel(int world, const int32_t* __restrict__ counts_matrix, int32_t* __restrict__ out) {
  int m = 0;
  for (int i = threadIdx.x; i < world * GSR_MAX_PEERS; i += 32) m = max(m, counts_matrix[i]);
  m = __reduce_max_sync(0xffffffffu, m);
  if (threadIdx.x == 0) *out = m;
}

struct ReturnArgs {
  int world, cap, me;
  const int32_t* counts_matrix;
  const float* acc;                   // [world*cap, 12] this tile owner's partial sums per candidate
  float* peer_ret[GSR_MAX_PEERS];     // ret array of every rank (as mapped here)
};
// backward collective: the rows of segment s go to rank s, slot me*cap + j of its ret array (contiguous copy)
__global__ void sparse_return_kernel(const ReturnArgs a) {
  const size_t total = (size_t)a.world * a.cap * 3;  // float4 units
  for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < total; q += (size_t)gridDim.x * blockDim.x) {
    const size_t c = q / 3;
    const int s = (int)(c / a.cap), j = (int)(c - (size_t)s * a.cap);
    if (j >= min(a.counts_matrix[s * GSR_MAX_PEERS + a.me], a.cap)) continue;
    const float4 v = __ldg(reinterpret_cast<const float4*>(a.acc) + q);
    reinterpret_cast<float4*>(a.peer_ret[s])[((size_t)a.me * a.cap + j) * 3 + (q - c * 3)] = v;
  }
}

// ---- owner side, backward ---------------------------------------------------------------------------------
// acc_slice[i] = sum over the destinations d of Gaussian i (ascending rank: a fixed order) of ret[d*cap + slot_d(i)]
__global__ void __launch_bounds__(SP_THREADS)
sparse_gather_kernel(int n, int world, int cap, const uint8_t* __restrict__ dest_mask, const uint32_t* __restrict__ blk_base,
                     const float* __restrict__ ret, float* __restrict__ acc_slice) {
  __shared__ uint32_t s_cnt[SP_THREADS / 32][GSR_MAX_PEERS];
  const int idx = blockIdx.x * SP_THREADS + threadIdx.x;
  const uint32_t m = idx < n ? dest_mask[idx] : 0u;
  uint32_t slot[GSR_MAX_PEERS];
  sparse_slots(m, world, blk_base, slot, s_cnt);
  if (idx >= n) return;
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0;
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) {
    if (!((m >> d) & 1u) || slot[d] >= (uint32_t)cap) continue;
    const float4* p = reinterpret_cast<const float4*>(ret + ((size_t)d * cap + slot[d]) * ACC_STRIDE);
    const float4 v0 = __ldg(p), v1 = __ldg(p + 1), v2 = __ldg(p + 2);
    a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
    a1.x += v1.x; a1.y += v1.y; a1.z += v1.z; a1.w += v1.w;
    a2.x += v2.x; a2.y += v2.y; a2.z += v2.z; a2.w += v2.w;
  }
  float4* o = reinterpret_cast<float4*>(acc_slice + (size_t)idx * ACC_STRIDE);
  o[0] = a0; o[1] = a1; o[2] = a2;
}

// semantic tracing: weights[i, ch] += and cnt[i] += the returned rows of Gaussian i (same slots and order as above); the
// count travels as int32 bits in slot GSR_SPARSE_AW_CNT_SLOT of the row
static_assert(GSR_SPARSE_AW_CNT_SLOT >= 3 && GSR_SPARSE_AW_CNT_SLOT < ACC_STRIDE, "count slot");
__global__ void __launch_bounds__(SP_THREADS)
sparse_aw_gather_kernel(int n, int world, int cap, int CH, const uint8_t* __restrict__ dest_mask,
                        const uint32_t* __restrict__ blk_base, const float* __restrict__ ret, float* __restrict__ weights,
                        int32_t* __restrict__ cnt) {
  __shared__ uint32_t s_cnt[SP_THREADS / 32][GSR_MAX_PEERS];
  const int idx = blockIdx.x * SP_THREADS + threadIdx.x;
  const uint32_t m = idx < n ? dest_mask[idx] : 0u;
  uint32_t slot[GSR_MAX_PEERS];
  sparse_slots(m, world, blk_base, slot, s_cnt);
  if (idx >= n || m == 0) return;
  float w0 = 0.f, w1 = 0.f, w2 = 0.f;
  int32_t c = 0;
#pragma unroll
  for (int d = 0; d < GSR_MAX_PEERS; d++) {
    if (!((m >> d) & 1u) || slot[d] >= (uint32_t)cap) continue;
    const float* p = ret + ((size_t)d * cap + slot[d]) * ACC_STRIDE;
    const float4 v = __ldg(reinterpret_cast<const float4*>(p));
    w0 += v.x; w1 += v.y; w2 += v.z;
    c += __float_as_int(__ldg(p + GSR_SPARSE_AW_CNT_SLOT));
  }
  float* w = weights + (size_t)idx * CH;
  w[0] += w0;
  if (CH > 1) w[1] += w1;
  if (CH > 2) w[2] += w2;
  cnt[idx] += c;
}

// ---- frame broadcast: owned tile rows of the [4,H,W] frame -> every rank's frame ----------------------------------
struct FrameArgs {
  int W, H, gy, world, me, nrows;  // nrows = owned tile rows
  const float* frame;              // local [4,H,W] (only the owned rows are valid)
  float* peer_frame[GSR_MAX_PEERS];
};
__global__ void frame_broadcast_kernel(const FrameArgs a) {
  // blockIdx.y = owned tile row k (ty = me + k*world), blockIdx.z = channel * world + peer; x strides over the row band
  const int k = blockIdx.y, ch = blockIdx.z / a.world, peer = blockIdx.z % a.world;
  if (peer == a.me) return;
  const int ty = a.me + k * a.world;
  const int y0 = ty * TILE, y1 = min(a.H, y0 + TILE);
  const size_t begin = (size_t)ch * a.H * a.W + (size_t)y0 * a.W, count = (size_t)(y1 - y0) * a.W;
  const float* src = a.frame + begin;
  float* dst = a.peer_frame[peer] + begin;
  // rows are contiguous in memory: treat the band as a flat array; 128-bit where alignment allows
  if (((begin | count) & 3) == 0) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count / 4; i += (size_t)gridDim.x * blockDim.x) d4[i] = s4[i];
  } else {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
  }
}

// ---- small row all-gather: this rank's row -> slot [me] of every rank's slots (a barrier must follow) ----------------
struct RowPutArgs {
  const float* row;
  int n, me, world;
  float* peer_slots[GSR_MAX_PEERS];  // rank r's [GSR_MAX_PEERS][GSR_PEER_ROW_FLOATS] slots as mapped here
};
__global__ void peer_row_put_kernel(const RowPutArgs a) {
  // threadIdx.x = float of the row (plain copy: the bits travel unchanged); the unrolled loop over the destinations
  // indexes the parameter array with constants, so it is not copied to local memory
  if ((int)threadIdx.x >= a.n) return;
  const float v = a.row[threadIdx.x];
#pragma unroll
  for (int r = 0; r < GSR_MAX_PEERS; r++)
    if (r < a.world) a.peer_slots[r][a.me * GSR_PEER_ROW_FLOATS + threadIdx.x] = v;
}

// ---- cross-rank barrier over peer memory ---------------------------------------------------------------------------
// 512 bytes at the start of every rank's peer-visible block. flags[r] is written by rank r only (the number of the last
// barrier it has reached); matrix row s is written by rank s only (n[s -> d], the segment sizes of the sparse exchange).
// The device-epoch barrier (gsr_peer_barrier_device) adds two fields behind the matrix: `epoch`, the number of the last
// device barrier this rank ran on the block (written by this rank's own barrier kernel only), and status[r], the
// overflow word rank r sent with its last barrier.
struct PeerCtrl {
  uint32_t flags[GSR_MAX_PEERS];
  uint32_t error;
  uint32_t pad[7];
  int32_t matrix[GSR_MAX_PEERS][GSR_MAX_PEERS];
  uint32_t epoch;
  uint32_t pad2[7];
  int32_t status[GSR_MAX_PEERS];
};
static_assert(sizeof(PeerCtrl) <= GSR_PEER_CTRL_BYTES && offsetof(PeerCtrl, matrix) == GSR_PEER_CTRL_MATRIX_OFFSET &&
                  offsetof(PeerCtrl, error) == GSR_PEER_CTRL_ERROR_OFFSET &&
                  offsetof(PeerCtrl, epoch) == GSR_PEER_CTRL_EPOCH_OFFSET &&
                  offsetof(PeerCtrl, status) == GSR_PEER_CTRL_STATUS_OFFSET, "ctrl layout");

struct BarrierArgs {
  PeerCtrl* ctrl[GSR_MAX_PEERS];
  int world, me, with_row;
  uint32_t epoch;
  long long timeout_clocks;
};
// One warp, lane r talks to rank r: (optionally) copy this rank's matrix row into r's matrix, fence, raise this rank's flag
// in r's block, then wait until r's flag in the OWN block has reached the epoch. Stores of earlier kernels of this stream
// (the pushes) are complete before this kernel starts; the system fence orders the row in front of the flag. A peer
// that never arrives costs `timeout_clocks` and sets ctrl.error instead of hanging the GPU.
__global__ void peer_barrier_kernel(const BarrierArgs a) {
  const int r = threadIdx.x;
  if (r < a.world) {
    if (a.with_row && r != a.me) {
#pragma unroll
      for (int d = 0; d < GSR_MAX_PEERS; d++)
        *(volatile int32_t*)&a.ctrl[r]->matrix[a.me][d] = *(volatile int32_t*)&a.ctrl[a.me]->matrix[a.me][d];
    }
    __threadfence_system();
    *(volatile uint32_t*)&a.ctrl[r]->flags[a.me] = a.epoch;
    volatile uint32_t* f = &a.ctrl[a.me]->flags[r];
    const long long t0 = clock64();
    while ((int32_t)(*f - a.epoch) < 0) {
      if (clock64() - t0 > a.timeout_clocks) { *(volatile uint32_t*)&a.ctrl[a.me]->error = 1u; break; }
    }
  }
  __threadfence_system();
}

struct BarrierDeviceArgs {
  PeerCtrl* ctrl[GSR_MAX_PEERS];
  const int32_t* status_word;  // or null
  int world, me, with_row;
  long long timeout_clocks;
};
// peer_barrier_kernel with the epoch taken from the own block's counter instead of a kernel argument, so that a replayed
// CUDA graph advances it: every lane reads the counter before lane 0 stores counter + 1 at the end, and the next barrier
// on this block (a later kernel of the same stream) sees the new value. With `status_word` its value is stored into
// status[me] of every block, own included, in front of the fence and the flag, as the matrix row is.
__global__ void peer_barrier_device_kernel(const BarrierDeviceArgs a) {
  const int r = threadIdx.x;
  const uint32_t epoch = *(volatile uint32_t*)&a.ctrl[a.me]->epoch + 1u;
  __syncwarp();
  if (r < a.world) {
    if (a.with_row && r != a.me) {
#pragma unroll
      for (int d = 0; d < GSR_MAX_PEERS; d++)
        *(volatile int32_t*)&a.ctrl[r]->matrix[a.me][d] = *(volatile int32_t*)&a.ctrl[a.me]->matrix[a.me][d];
    }
    if (a.status_word) *(volatile int32_t*)&a.ctrl[r]->status[a.me] = *(volatile const int32_t*)a.status_word;
    __threadfence_system();
    *(volatile uint32_t*)&a.ctrl[r]->flags[a.me] = epoch;
    volatile uint32_t* f = &a.ctrl[a.me]->flags[r];
    const long long t0 = clock64();
    while ((int32_t)(*f - epoch) < 0) {
      if (clock64() - t0 > a.timeout_clocks) { *(volatile uint32_t*)&a.ctrl[a.me]->error = 1u; break; }
    }
  }
  __syncwarp();
  if (r == 0) *(volatile uint32_t*)&a.ctrl[a.me]->epoch = epoch;
  __threadfence_system();
}

int check_plan(const gsr_sparse_plan* p) {
  if (!p || p->world < 1 || p->world > GSR_MAX_PEERS || p->rank < 0 || p->rank >= p->world || p->slice_len < 0 ||
      p->seg_cap < 1) {
    set_error("sparse plan: need 1 <= world <= %d, 0 <= rank < world, slice_len >= 0, seg_cap >= 1", GSR_MAX_PEERS);
    return GSR_ERR_INVALID;
  }
  if ((int64_t)p->world * p->seg_cap > 0x7fffffffLL) { set_error("sparse plan: world*seg_cap overflows"); return GSR_ERR_INVALID; }
  return GSR_OK;
}

}  // namespace
}  // namespace gsr

using namespace gsr;

extern "C" {

size_t gsr_sparse_local_bytes(int32_t slice_len) {
  GeometryWS g;
  if (!carve_geometry(nullptr, slice_len, g)) return 0;
  SparseLocal sl;
  return carve_sparse_local(nullptr, slice_len, g, sl);
}

size_t gsr_sparse_candidate_bytes(int32_t world, int32_t seg_cap) {
  SparseCand sc;
  if (world < 1 || seg_cap < 1 || !carve_sparse_cand(nullptr, world, seg_cap, sc)) return 0;
  return sc.total;
}

// gsr_sparse_preprocess and, with `raw`, gsr_sparse_preprocess_raw (`shard` unused); with `grad_mask` their masked
// twins: the masked preprocess writes the records' edit words, and the push carries them with the records
static int sparse_preprocess_impl(const gsr_settings* s, const gsr_cloud* shard, const gsr_raw_cloud* raw,
                                  const gsr_sparse_plan* plan, void* local_ws, size_t local_bytes, int32_t* radii_local,
                                  void* const* peer_cand, size_t cand_bytes, int32_t* counts_row, void* stream,
                                  const uint8_t* grad_mask = nullptr) {
  int rc = check_plan(plan);
  if (rc) return rc;
  const int32_t P = raw ? raw->P : (shard ? shard->P : -1);
  if (!s || P < 0 || P > plan->slice_len) { set_error("sparse_preprocess: shard does not fit slice_len"); return GSR_ERR_INVALID; }
  if (!local_ws || !radii_local || !peer_cand || !counts_row) { set_error("sparse_preprocess: null buffer"); return GSR_ERR_INVALID; }
  gsr_cloud c;
  rc = shard_cloud(s, shard, raw, c);  // (P == 0 passes: nothing of the cloud is read)
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int n = P;
  GeometryWS g;
  if (!carve_geometry(local_ws, plan->slice_len, g)) return GSR_ERR_CUDA;
  SparseLocal sl;
  carve_sparse_local(local_ws, plan->slice_len, g, sl);
  if (sl.total > local_bytes) { set_error("local workspace too small: %zu < %zu", local_bytes, sl.total); return GSR_ERR_WORKSPACE; }
  PushArgs pa;
  pa.n = n; pa.world = plan->world; pa.rank = plan->rank; pa.cap = plan->seg_cap;
  for (int r = 0; r < GSR_MAX_PEERS; r++) pa.peer_records[r] = nullptr;
  for (int r = 0; r < plan->world; r++) {
    SparseCand sc;
    if (!peer_cand[r] || !carve_sparse_cand(peer_cand[r], plan->world, plan->seg_cap, sc)) { set_error("peer candidate workspace %d is null", r); return GSR_ERR_INVALID; }
    if (sc.total > cand_bytes) { set_error("candidate workspace too small: %zu < %zu", cand_bytes, sc.total); return GSR_ERR_WORKSPACE; }
    pa.peer_records[r] = sc.g.records;
  }
  const int W = s->image_width, H = s->image_height;
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (n == 0) return check_cuda(cudaMemsetAsync(counts_row, 0, GSR_MAX_PEERS * sizeof(int32_t), st), "counts memset");
  {
    StageScope t(ST_PRE_FWD, st);
    rc = launch_preprocess_fwd(*s, c, g, radii_local, st, nullptr, 0, raw != nullptr, raw ? raw->features_rest : nullptr,
                               false, grad_mask);
    if (rc) return rc;
    const int nblocks = (n + SP_THREADS - 1) / SP_THREADS;
    sparse_mask_kernel<<<nblocks, SP_THREADS, 0, st>>>(n, g.records, gx, gy, plan->world, sl.dest_mask, sl.blk_base);
    sparse_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(n, plan->world, sl.blk_base, counts_row);
    pa.records = g.records; pa.dest_mask = sl.dest_mask; pa.blk_base = sl.blk_base;
    sparse_push_kernel<<<nblocks, SP_THREADS, 0, st>>>(pa);
    g_launches += 3;
  }
  return check_launch("sparse_preprocess", s->debug != 0, st);
}

int gsr_sparse_preprocess(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan, void* local_ws,
                          size_t local_bytes, int32_t* radii_local, void* const* peer_cand, size_t cand_bytes,
                          int32_t* counts_row, void* stream) {
  return sparse_preprocess_impl(s, shard, nullptr, plan, local_ws, local_bytes, radii_local, peer_cand, cand_bytes,
                                counts_row, stream);
}

int gsr_sparse_preprocess_raw(const gsr_settings* s, const gsr_raw_cloud* shard, const gsr_sparse_plan* plan,
                              void* local_ws, size_t local_bytes, int32_t* radii_local, void* const* peer_cand,
                              size_t cand_bytes, int32_t* counts_row, void* stream) {
  return sparse_preprocess_impl(s, nullptr, shard, plan, local_ws, local_bytes, radii_local, peer_cand, cand_bytes,
                                counts_row, stream);
}

int gsr_sparse_preprocess_masked(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan,
                                 void* local_ws, size_t local_bytes, int32_t* radii_local, void* const* peer_cand,
                                 size_t cand_bytes, int32_t* counts_row, const uint8_t* grad_mask, void* stream) {
  const int rc = check_mask_args(grad_mask, nullptr);
  if (rc) return rc;
  return sparse_preprocess_impl(s, shard, nullptr, plan, local_ws, local_bytes, radii_local, peer_cand, cand_bytes,
                                counts_row, stream, grad_mask);
}

int gsr_sparse_preprocess_raw_masked(const gsr_settings* s, const gsr_raw_cloud* shard, const gsr_sparse_plan* plan,
                                     void* local_ws, size_t local_bytes, int32_t* radii_local, void* const* peer_cand,
                                     size_t cand_bytes, int32_t* counts_row, const uint8_t* grad_mask, void* stream) {
  const int rc = check_mask_args(grad_mask, nullptr);
  if (rc) return rc;
  return sparse_preprocess_impl(s, nullptr, shard, plan, local_ws, local_bytes, radii_local, peer_cand, cand_bytes,
                                counts_row, stream, grad_mask);
}

// gsr_sparse_order and, with host_out == nullptr, gsr_sparse_order_static (no host words: the static forward's status
// kernel reads the matrix and R on the device)
static int sparse_order_impl(const gsr_settings* s, const gsr_sparse_plan* plan, void* cand_ws, size_t cand_bytes,
                             const int32_t* counts_matrix, int32_t* radii_cand, int32_t* host_out, void* stream) {
  int rc = check_plan(plan);
  if (rc) return rc;
  if (!s || !cand_ws || !counts_matrix || !radii_cand) { set_error("sparse_order: null argument"); return GSR_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  SparseCand sc;
  if (!carve_sparse_cand(cand_ws, plan->world, plan->seg_cap, sc)) return GSR_ERR_CUDA;
  if (sc.total > cand_bytes) { set_error("candidate workspace too small: %zu < %zu", cand_bytes, sc.total); return GSR_ERR_WORKSPACE; }
  const int M = plan->world * plan->seg_cap;
  const int gx = (s->image_width + TILE - 1) / TILE, gy = (s->image_height + TILE - 1) / TILE;
  StageScope t(ST_DEPTH_SCAN, st);
  const bool v2 = tile_binning_supported(gx, gy);
  if (v2 && (rc = clear_tile_counts(sc.g, gx, gy, st))) return rc;
  retouch_sparse_kernel<<<(M + 255) / 256, 256, 0, st>>>(plan->world, plan->seg_cap, plan->rank, counts_matrix, sc.g.records,
                                                         gx, gy, radii_cand, sc.g.tiles_touched, sc.g.ident, sc.g.depth_keys,
                                                         v2 ? sc.g.tile_diff : nullptr, tile_diff_copies(gx, gy));
  g_launches++;
  if (host_out) {
    // host_out[1] (largest segment anywhere) is copied out BEFORE host_out[0] (num_rendered): a host that polls word 0
    // finds word 1 already in place. The device word is overwritten by the sort afterwards: read first.
    int32_t* dev_word = reinterpret_cast<int32_t*>(sc.g.depth_keys_sorted);
    sparse_max_count_kernel<<<1, 32, 0, st>>>(plan->world, counts_matrix, dev_word);
    g_launches++;
    cudaError_t e = cudaMemcpyAsync(host_out + 1, dev_word, sizeof(int32_t), cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return check_cuda(e, "max-count readback");
  }
  if (v2) {
    TileOwner own; own.stride = plan->world; own.phase = plan->rank;
    if ((rc = launch_tile_count(sc.g, gx, gy, own, st))) return rc;
    if (host_out) {
      cudaError_t e = cudaMemcpyAsync(host_out, sc.g.R_dev, sizeof(int32_t), cudaMemcpyDeviceToHost, st);
      if (e != cudaSuccess) return check_cuda(e, "num_rendered readback");
    }
  }
  gsr_cloud c{};
  c.P = M;
  return run_depth_order_and_scan(c, sc.g, v2 ? nullptr : host_out, st, s->debug != 0);
}

int gsr_sparse_order(const gsr_settings* s, const gsr_sparse_plan* plan, void* cand_ws, size_t cand_bytes,
                     const int32_t* counts_matrix, int32_t* radii_cand, int32_t* host_out, void* stream) {
  if (!host_out) { set_error("sparse_order: null argument"); return GSR_ERR_INVALID; }
  return sparse_order_impl(s, plan, cand_ws, cand_bytes, counts_matrix, radii_cand, host_out, stream);
}

int gsr_sparse_order_static(const gsr_settings* s, const gsr_sparse_plan* plan, void* cand_ws, size_t cand_bytes,
                            const int32_t* counts_matrix, int32_t* radii_cand, void* stream) {
  return sparse_order_impl(s, plan, cand_ws, cand_bytes, counts_matrix, radii_cand, nullptr, stream);
}

int gsr_sparse_return(const gsr_sparse_plan* plan, const void* acc_cand, const int32_t* counts_matrix,
                      void* const* peer_cand, void* stream) {
  int rc = check_plan(plan);
  if (rc) return rc;
  if (!acc_cand || !counts_matrix || !peer_cand) { set_error("sparse_return: null argument"); return GSR_ERR_INVALID; }
  ReturnArgs a;
  a.world = plan->world; a.cap = plan->seg_cap; a.me = plan->rank; a.counts_matrix = counts_matrix; a.acc = (const float*)acc_cand;
  for (int r = 0; r < GSR_MAX_PEERS; r++) a.peer_ret[r] = nullptr;
  for (int r = 0; r < plan->world; r++) {
    SparseCand sc;
    if (!peer_cand[r] || !carve_sparse_cand(peer_cand[r], plan->world, plan->seg_cap, sc)) { set_error("peer candidate workspace %d is null", r); return GSR_ERR_INVALID; }
    a.peer_ret[r] = sc.ret;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t total = (size_t)plan->world * plan->seg_cap * 3;
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)device_sm_count() * 16);
  sparse_return_kernel<<<blocks, 256, 0, st>>>(a);
  g_launches++;
  return check_launch("sparse_return", false, st);
}

// gsr_sparse_backward_preprocess, its DEPTH form and, with `raw` / `rgr`, gsr_sparse_backward_preprocess_raw (`shard`
// and `gr` unused)
static int sparse_backward_preprocess_impl(const gsr_settings* s, const gsr_cloud* shard, const gsr_raw_cloud* raw,
                                           const gsr_sparse_plan* plan, const void* local_ws, size_t local_bytes,
                                           const int32_t* radii_local, const void* cand_ws, size_t cand_bytes,
                                           void* acc_slice, size_t acc_bytes, const gsr_grads* gr,
                                           const gsr_raw_grads* rgr, bool depth, void* stream,
                                           const gsr_camera_grads* cam = nullptr, const uint8_t* grad_mask = nullptr) {
  int rc = check_plan(plan);
  if (rc) return rc;
  const int32_t P = raw ? raw->P : (shard ? shard->P : -1);
  if (!s || P < 0 || P > plan->slice_len) { set_error("sparse_backward: shard does not fit slice_len"); return GSR_ERR_INVALID; }
  if (cam && (rc = check_shard_camera(cam, P))) return rc;
  if (P == 0) return cam ? zero_shard_camera(cam, (cudaStream_t)stream) : GSR_OK;
  gsr_cloud c;
  rc = shard_cloud(s, shard, raw, c);
  if (rc) return rc;
  if ((raw ? !rgr : !gr) || !local_ws || !cand_ws || !radii_local || !acc_slice) { set_error("sparse_backward: null argument"); return GSR_ERR_INVALID; }
  if (raw) {
    if ((rc = check_raw_grads(s, rgr))) return rc;
    if (reinterpret_cast<uintptr_t>(acc_slice) & 15) { set_error("acc_slice must be 16-byte aligned"); return GSR_ERR_INVALID; }
  } else {
    if (!gr->dL_dmeans3D || !gr->dL_dmeans2D || !gr->dL_dcolors || !gr->dL_dopacity || !gr->dL_dcov3D ||
        !gr->dL_dscales || !gr->dL_drotations || (c.shs && !gr->dL_dsh)) {
      set_error("a gradient output pointer is null");
      return GSR_ERR_INVALID;
    }
    if ((reinterpret_cast<uintptr_t>(gr->dL_drotations) & 15) || (reinterpret_cast<uintptr_t>(acc_slice) & 15)) {
      set_error("dL_drotations / acc_slice must be 16-byte aligned");
      return GSR_ERR_INVALID;
    }
  }
  const int n = c.P;
  if (acc_bytes < (size_t)n * ACC_STRIDE * sizeof(float)) { set_error("acc_slice too small"); return GSR_ERR_WORKSPACE; }
  GeometryWS g;
  if (!carve_geometry(const_cast<void*>(local_ws), plan->slice_len, g)) return GSR_ERR_CUDA;
  SparseLocal sl;
  carve_sparse_local(const_cast<void*>(local_ws), plan->slice_len, g, sl);
  if (sl.total > local_bytes) { set_error("local workspace too small: %zu < %zu", local_bytes, sl.total); return GSR_ERR_WORKSPACE; }
  SparseCand sc;
  if (!carve_sparse_cand(const_cast<void*>(cand_ws), plan->world, plan->seg_cap, sc)) return GSR_ERR_CUDA;
  if (sc.total > cand_bytes) { set_error("candidate workspace too small: %zu < %zu", cand_bytes, sc.total); return GSR_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  StageScope t(ST_PRE_BWD, st);
  // the gather adds all 12 floats of each returned row, slot 9 (dL/dz of the depth gradient) included
  sparse_gather_kernel<<<(n + SP_THREADS - 1) / SP_THREADS, SP_THREADS, 0, st>>>(n, plan->world, plan->seg_cap, sl.dest_mask,
                                                                                 sl.blk_base, sc.ret, (float*)acc_slice);
  g_launches++;
  rc = check_launch("sparse_gather", s->debug != 0, st);
  if (rc) return rc;
  if (raw) {
    const RawBackward rb{raw->features_rest, rgr->dL_dfeatures_rest};
    return launch_preprocess_bwd(*s, c, g, radii_local, (const float*)acc_slice, raw_grads_as_full(*rgr), st, &rb,
                                 nullptr, depth, grad_mask);
  }
  if (cam) {
    const CameraBackward cb{cam->dL_dviewmatrix, cam->dL_dprojmatrix, cam->dL_dcampos, (float*)cam->scratch};
    return launch_preprocess_bwd(*s, c, g, radii_local, (const float*)acc_slice, *gr, st, nullptr, &cb, depth);
  }
  return launch_preprocess_bwd(*s, c, g, radii_local, (const float*)acc_slice, *gr, st, nullptr, nullptr, depth,
                               grad_mask);
}

int gsr_sparse_backward_preprocess_camera(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan,
                                          const void* local_ws, size_t local_bytes, const int32_t* radii_local,
                                          const void* cand_ws, size_t cand_bytes, void* acc_slice, size_t acc_bytes,
                                          const gsr_grads* gr, int32_t depth, const gsr_camera_grads* camera,
                                          void* stream) {
  if (!camera) { set_error("camera gradients: null struct"); return GSR_ERR_INVALID; }
  return sparse_backward_preprocess_impl(s, shard, nullptr, plan, local_ws, local_bytes, radii_local, cand_ws, cand_bytes,
                                         acc_slice, acc_bytes, gr, nullptr, depth != 0, stream, camera);
}

int gsr_sparse_backward_preprocess(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan,
                                   const void* local_ws, size_t local_bytes, const int32_t* radii_local,
                                   const void* cand_ws, size_t cand_bytes, void* acc_slice, size_t acc_bytes,
                                   const gsr_grads* gr, void* stream) {
  return sparse_backward_preprocess_impl(s, shard, nullptr, plan, local_ws, local_bytes, radii_local, cand_ws, cand_bytes,
                                         acc_slice, acc_bytes, gr, nullptr, false, stream);
}

int gsr_sparse_backward_preprocess_depth(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan,
                                         const void* local_ws, size_t local_bytes, const int32_t* radii_local,
                                         const void* cand_ws, size_t cand_bytes, void* acc_slice, size_t acc_bytes,
                                         const gsr_grads* gr, void* stream) {
  return sparse_backward_preprocess_impl(s, shard, nullptr, plan, local_ws, local_bytes, radii_local, cand_ws, cand_bytes,
                                         acc_slice, acc_bytes, gr, nullptr, true, stream);
}

int gsr_sparse_backward_preprocess_raw(const gsr_settings* s, const gsr_raw_cloud* shard, const gsr_sparse_plan* plan,
                                       const void* local_ws, size_t local_bytes, const int32_t* radii_local,
                                       const void* cand_ws, size_t cand_bytes, void* acc_slice, size_t acc_bytes,
                                       const gsr_raw_grads* gr, int32_t depth, void* stream) {
  return sparse_backward_preprocess_impl(s, nullptr, shard, plan, local_ws, local_bytes, radii_local, cand_ws, cand_bytes,
                                         acc_slice, acc_bytes, nullptr, gr, depth != 0, stream);
}

// masked twins: the rank's local workspace is indexed by its own rows, so grad_mask holds them [shard.P]
int gsr_sparse_backward_preprocess_masked(const gsr_settings* s, const gsr_cloud* shard, const gsr_sparse_plan* plan,
                                          const void* local_ws, size_t local_bytes, const int32_t* radii_local,
                                          const void* cand_ws, size_t cand_bytes, void* acc_slice, size_t acc_bytes,
                                          const gsr_grads* gr, int32_t depth, const gsr_camera_grads* camera,
                                          const uint8_t* grad_mask, void* stream) {
  const int rc = check_mask_args(grad_mask, camera);
  if (rc) return rc;
  return sparse_backward_preprocess_impl(s, shard, nullptr, plan, local_ws, local_bytes, radii_local, cand_ws, cand_bytes,
                                         acc_slice, acc_bytes, gr, nullptr, depth != 0, stream, nullptr, grad_mask);
}

int gsr_sparse_backward_preprocess_raw_masked(const gsr_settings* s, const gsr_raw_cloud* shard,
                                              const gsr_sparse_plan* plan, const void* local_ws, size_t local_bytes,
                                              const int32_t* radii_local, const void* cand_ws, size_t cand_bytes,
                                              void* acc_slice, size_t acc_bytes, const gsr_raw_grads* gr, int32_t depth,
                                              const uint8_t* grad_mask, void* stream) {
  const int rc = check_mask_args(grad_mask, nullptr);
  if (rc) return rc;
  return sparse_backward_preprocess_impl(s, nullptr, shard, plan, local_ws, local_bytes, radii_local, cand_ws, cand_bytes,
                                         acc_slice, acc_bytes, nullptr, gr, depth != 0, stream, nullptr, grad_mask);
}

int gsr_sparse_apply_weights_gather(const gsr_sparse_plan* plan, const void* local_ws, size_t local_bytes,
                                    const void* cand_ws, size_t cand_bytes, int32_t n, int32_t CH, float* weights,
                                    int32_t* cnt, void* stream) {
  int rc = check_plan(plan);
  if (rc) return rc;
  if (CH < 1 || CH > 3) { set_error("sparse_apply_weights_gather: num_channels %d outside 1..3", CH); return GSR_ERR_INVALID; }
  if (n < 0 || n > plan->slice_len) { set_error("sparse_apply_weights_gather: n = %d does not fit slice_len", n); return GSR_ERR_INVALID; }
  if (!local_ws || !cand_ws || !weights || !cnt) { set_error("sparse_apply_weights_gather: null argument"); return GSR_ERR_INVALID; }
  if (n == 0) return GSR_OK;
  GeometryWS g;
  if (!carve_geometry(const_cast<void*>(local_ws), plan->slice_len, g)) return GSR_ERR_CUDA;
  SparseLocal sl;
  carve_sparse_local(const_cast<void*>(local_ws), plan->slice_len, g, sl);
  if (sl.total > local_bytes) { set_error("local workspace too small: %zu < %zu", local_bytes, sl.total); return GSR_ERR_WORKSPACE; }
  SparseCand sc;
  if (!carve_sparse_cand(const_cast<void*>(cand_ws), plan->world, plan->seg_cap, sc)) return GSR_ERR_CUDA;
  if (sc.total > cand_bytes) { set_error("candidate workspace too small: %zu < %zu", cand_bytes, sc.total); return GSR_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  StageScope t(ST_APPLY_W, st);
  sparse_aw_gather_kernel<<<(n + SP_THREADS - 1) / SP_THREADS, SP_THREADS, 0, st>>>(n, plan->world, plan->seg_cap, CH,
                                                                                    sl.dest_mask, sl.blk_base, sc.ret,
                                                                                    weights, cnt);
  g_launches++;
  return check_launch("sparse_apply_weights_gather", false, st);
}

int gsr_sparse_view(void* cand_ws, int32_t world, int32_t seg_cap, gsr_sparse_view_t* out) {
  SparseCand sc;
  if (!out || world < 1 || seg_cap < 1 || !carve_sparse_cand(cand_ws, world, seg_cap, sc)) return GSR_ERR_INVALID;
  out->records = sc.g.records;
  out->ret = sc.ret;
  out->geometry_bytes = sc.g.total;
  return GSR_OK;
}

int gsr_peer_barrier(int32_t world, int32_t rank, void* const* peer_ctrl, uint32_t epoch, int32_t with_matrix_row,
                     void* stream) {
  if (world < 1 || world > GSR_MAX_PEERS || rank < 0 || rank >= world || !peer_ctrl) { set_error("peer_barrier: bad arguments"); return GSR_ERR_INVALID; }
  BarrierArgs a;
  for (int r = 0; r < GSR_MAX_PEERS; r++) a.ctrl[r] = r < world ? (PeerCtrl*)peer_ctrl[r] : nullptr;
  for (int r = 0; r < world; r++)
    if (!a.ctrl[r]) { set_error("peer_barrier: peer block %d is null", r); return GSR_ERR_INVALID; }
  a.world = world; a.me = rank; a.with_row = with_matrix_row; a.epoch = epoch;
  a.timeout_clocks = 4000000000LL;  // ~2 s at 2 GHz
  peer_barrier_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a);
  g_launches++;
  return check_launch("peer_barrier", false, (cudaStream_t)stream);
}

int gsr_peer_barrier_device(int32_t world, int32_t rank, void* const* peer_ctrl, int32_t with_matrix_row,
                            const int32_t* status_word, void* stream) {
  if (world < 1 || world > GSR_MAX_PEERS || rank < 0 || rank >= world || !peer_ctrl) { set_error("peer_barrier_device: bad arguments"); return GSR_ERR_INVALID; }
  BarrierDeviceArgs a;
  for (int r = 0; r < GSR_MAX_PEERS; r++) a.ctrl[r] = r < world ? (PeerCtrl*)peer_ctrl[r] : nullptr;
  for (int r = 0; r < world; r++)
    if (!a.ctrl[r]) { set_error("peer_barrier_device: peer block %d is null", r); return GSR_ERR_INVALID; }
  a.status_word = status_word;
  a.world = world; a.me = rank; a.with_row = with_matrix_row;
  a.timeout_clocks = 4000000000LL;  // ~2 s at 2 GHz, as gsr_peer_barrier
  peer_barrier_device_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a);
  g_launches++;
  return check_launch("peer_barrier_device", false, (cudaStream_t)stream);
}

int gsr_frame_broadcast_planes(const gsr_tile_owner* owner, int32_t W, int32_t H, int32_t planes, const float* frame,
                               void* const* peer_frames, void* stream) {
  if (!owner || owner->row_stride < 1 || owner->row_stride > GSR_MAX_PEERS || owner->row_phase < 0 ||
      owner->row_phase >= owner->row_stride || !frame || !peer_frames || W < 0 || H < 0) {
    set_error("frame_broadcast: bad arguments");
    return GSR_ERR_INVALID;
  }
  if (planes < 1 || planes > GSR_FRAME_MAX_PLANES) {
    set_error("frame_broadcast: planes = %d outside 1..%d", planes, GSR_FRAME_MAX_PLANES);
    return GSR_ERR_INVALID;
  }
  FrameArgs a;
  a.W = W; a.H = H; a.gy = (H + TILE - 1) / TILE; a.world = owner->row_stride; a.me = owner->row_phase;
  TileOwner own; own.stride = owner->row_stride; own.phase = owner->row_phase;
  a.nrows = own.owned_rows(a.gy);
  a.frame = frame;
  for (int r = 0; r < GSR_MAX_PEERS; r++) a.peer_frame[r] = r < a.world ? (float*)peer_frames[r] : nullptr;
  for (int r = 0; r < a.world; r++)
    if (!a.peer_frame[r]) { set_error("frame_broadcast: peer frame %d is null", r); return GSR_ERR_INVALID; }
  if (a.nrows == 0 || a.world == 1 || W * H == 0) return GSR_OK;
  dim3 grid(4, a.nrows, planes * a.world);
  frame_broadcast_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
  g_launches++;
  return check_launch("frame_broadcast", false, (cudaStream_t)stream);
}

int gsr_frame_broadcast(const gsr_tile_owner* owner, int32_t W, int32_t H, const float* frame, void* const* peer_frames,
                        void* stream) {
  return gsr_frame_broadcast_planes(owner, W, H, 4, frame, peer_frames, stream);
}

int gsr_peer_row_put(int32_t world, int32_t rank, const float* row, int32_t n, void* const* peer_slots, void* stream) {
  if (world < 1 || world > GSR_MAX_PEERS || rank < 0 || rank >= world || !row || !peer_slots) {
    set_error("peer_row_put: bad arguments");
    return GSR_ERR_INVALID;
  }
  if (n < 1 || n > GSR_PEER_ROW_FLOATS) { set_error("peer_row_put: n = %d outside 1..%d", n, GSR_PEER_ROW_FLOATS); return GSR_ERR_INVALID; }
  RowPutArgs a;
  for (int r = 0; r < GSR_MAX_PEERS; r++) a.peer_slots[r] = r < world ? (float*)peer_slots[r] : nullptr;
  for (int r = 0; r < world; r++)
    if (!a.peer_slots[r]) { set_error("peer_row_put: peer slots %d are null", r); return GSR_ERR_INVALID; }
  a.row = row; a.n = n; a.me = rank; a.world = world;
  peer_row_put_kernel<<<1, GSR_PEER_ROW_FLOATS, 0, (cudaStream_t)stream>>>(a);
  g_launches++;
  return check_launch("peer_row_put", false, (cudaStream_t)stream);
}

}  // extern "C"
