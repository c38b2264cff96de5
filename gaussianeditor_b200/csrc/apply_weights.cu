// Semantic tracing ("apply_weights") for sm_90a.
//
// Semantics: renderCUDA_apply_weights of GaussianEditor's fork (cuda_rasterizer/apply_weights.cu:240-356):
// the forward walk of a tile list with the forward's skip / stop rules, but instead of blending, every
// (pixel, splat) pair that WOULD be blended adds the pixel's 2-D mask value to the splat:
//     weights[id*CH + ch] += image_weights[ch, pixel];   cnt[id] += 1      (once per channel, :331-334)
// No image is written.  The reference issues 2*CH global atomics per hit; here the hits of a warp on the same
// splat are summed with shuffles first (one atomic pair per warp and splat). There is no tile culling: every
// pixel tests every splat of its tile's list with the reference's per-pixel alpha >= 1/255 test.
// Integer counts are exact; float sums differ from the reference only in summation order.
#include "common.cuh"

namespace gsr {

namespace {

struct AwArgs {
  const uint2* ranges;
  const uint32_t* point_list;
  const SplatRecord* records;
  int W, H, gx, gy;
  const float* image_weights;
  float* weights;
  int32_t* cnt;
};

// The walk of tile (blockIdx.x, ty). Splat id's hits go to weights[id*w_stride + ch] and cnt[id*c_stride].
template <int CH>
__device__ __forceinline__ void apply_weights_walk(const AwArgs& a, const unsigned ty, const size_t w_stride,
                                                   const size_t c_stride) {
  __shared__ float4 s_q0[TILE_PIX], s_q1[TILE_PIX];
  __shared__ uint32_t s_ids[TILE_PIX];
  const int tile = ty * a.gx + blockIdx.x;
  const int tid = threadIdx.y * TILE + threadIdx.x;
  const int lane = tid & 31;
  const uint2 pix = make_uint2(blockIdx.x * TILE + threadIdx.x, ty * TILE + threadIdx.y);
  const bool inside = pix.x < (unsigned)a.W && pix.y < (unsigned)a.H;
  const size_t pix_id = (size_t)a.W * pix.y + pix.x;
  const float2 pixf = make_float2((float)pix.x, (float)pix.y);
  const uint2 range = a.ranges[tile];
  const int rounds = ((range.y - range.x + TILE_PIX - 1) / TILE_PIX);
  int toDo = range.y - range.x;
  bool done = !inside;
  float T = 1.0f;
  float Cw[CH];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) Cw[ch] = inside ? a.image_weights[(size_t)ch * a.H * a.W + pix_id] : 0.f;

  for (int i = 0; i < rounds; i++, toDo -= TILE_PIX) {
    int num_done = __syncthreads_count(done);
    if (num_done == TILE_PIX) break;
    int progress = i * TILE_PIX + tid;
    if (range.x + progress < range.y) {
      const uint32_t id = a.point_list[range.x + progress];
      const float4* r = reinterpret_cast<const float4*>(a.records + id);
      s_q0[tid] = __ldg(r);
      s_q1[tid] = __ldg(r + 1);
      s_ids[tid] = id;
    }
    __syncthreads();
    const int n = min(TILE_PIX, toDo);
    for (int j = 0; j < n; j++) {
      bool hit = false;
      if (!done) {
        const float4 q0 = s_q0[j], q1 = s_q1[j];
        const float dx = q0.x - pixf.x, dy = q0.y - pixf.y;
        const float power = splat_power(dx, dy, q0.z, q0.w, q1.x);
        if (!(power > 0.0f)) {
          const float alpha = fminf(0.99f, __fmul_rn(q1.y, expf(power)));
          if (!(alpha < 1.0f / 255.0f)) {
            const float test_T = __fmul_rn(T, __fadd_rn(1.0f, -alpha));
            if (test_T < 0.0001f) {
              done = true;
            } else {
              hit = true;
              T = test_T;
            }
          }
        }
      }
      const unsigned hits = __ballot_sync(0xffffffffu, hit);
      if (hits) {
        const uint32_t id = s_ids[j];
#pragma unroll
        for (int ch = 0; ch < CH; ch++) {
          float v = hit ? Cw[ch] : 0.f;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          if (lane == 0) atomicAdd(a.weights + (size_t)id * w_stride + ch, v);
        }
        if (lane == 0) atomicAdd(a.cnt + (size_t)id * c_stride, CH * __popc(hits));
      }
    }
  }
}

template <int CH>
__global__ void __launch_bounds__(TILE_PIX) apply_weights_kernel(const AwArgs a) {
  apply_weights_walk<CH>(a, blockIdx.y, CH, 1);
}

// Gaussian-sharded path: blockIdx.y = k-th owned tile row (ty = own_phase + k*own_stride), and strided outputs so that
// the same walk fills a dense [P, CH] + [P] pair or the [M, 12] rows of the sparse return (cnt as int32 bits in a slot).
struct AwOwnerArgs : AwArgs {
  int own_stride, own_phase;
  int64_t w_stride, c_stride;
};

template <int CH>
__global__ void __launch_bounds__(TILE_PIX) apply_weights_owner_kernel(const AwOwnerArgs a) {
  apply_weights_walk<CH>(a, a.own_phase + blockIdx.y * a.own_stride, a.w_stride, a.c_stride);
}


// Deterministic mode (DetWS, deterministic.cu): the same walk, but the per-warp sums of a 256-splat round go to shared
// memory [8 warps][256][CH]. At the round boundary (where __syncthreads_count already synchronises, and so also before
// the early break) thread t adds the 8 warp entries of splat t in warp order and stores the row at that instance's
// emission slot, with its flag; the reduction kernel adds each Gaussian's rows to `weights`. `cnt` keeps its integer
// atomics, which are exact. Ownership as in apply_weights_owner_kernel: blockIdx.y = k-th owned tile row ({1, 0} on a
// single GPU), and the count of splat id goes to cnt[id*c_stride].
struct AwDetArgs : AwArgs {
  const uint32_t* excl;
  float* rows;     // [R, CH]
  uint8_t* flags;  // [R]
  int own_stride, own_phase;
  int64_t c_stride;
};

template <int CH>
__global__ void __launch_bounds__(TILE_PIX) apply_weights_det_kernel(const AwDetArgs a) {
  constexpr int NW = TILE_PIX / 32;
  __shared__ float4 s_q0[TILE_PIX], s_q1[TILE_PIX];
  __shared__ uint32_t s_ids[TILE_PIX];
  __shared__ uint32_t s_slot[TILE_PIX];
  __shared__ float s_w[NW][TILE_PIX][CH];
  const unsigned ty = a.own_phase + blockIdx.y * a.own_stride;
  const int tile = ty * a.gx + blockIdx.x;
  const int tid = threadIdx.y * TILE + threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const uint2 pix = make_uint2(blockIdx.x * TILE + threadIdx.x, ty * TILE + threadIdx.y);
  const bool inside = pix.x < (unsigned)a.W && pix.y < (unsigned)a.H;
  const size_t pix_id = (size_t)a.W * pix.y + pix.x;
  const float2 pixf = make_float2((float)pix.x, (float)pix.y);
  const uint2 range = a.ranges[tile];
  const int rounds = ((range.y - range.x + TILE_PIX - 1) / TILE_PIX);
  int toDo = range.y - range.x;
  bool done = !inside;
  float T = 1.0f;
  float Cw[CH];
#pragma unroll
  for (int ch = 0; ch < CH; ch++) Cw[ch] = inside ? a.image_weights[(size_t)ch * a.H * a.W + pix_id] : 0.f;
  // row of splat t of the round just finished (block-uniform count n)
  auto flush = [&](int n) {
    if (tid < n) {
      const size_t slot = s_slot[tid];
#pragma unroll
      for (int ch = 0; ch < CH; ch++) {
        float v = s_w[0][tid][ch];
#pragma unroll
        for (int w = 1; w < NW; w++) v += s_w[w][tid][ch];
        a.rows[slot * CH + ch] = v;
      }
      a.flags[slot] = 1;
    }
  };

  int prev_n = 0;
  for (int i = 0; i < rounds; i++, toDo -= TILE_PIX) {
    int num_done = __syncthreads_count(done);
    flush(prev_n);
    prev_n = 0;
    if (num_done == TILE_PIX) break;
    int progress = i * TILE_PIX + tid;
    if (range.x + progress < range.y) {
      const uint32_t id = a.point_list[range.x + progress];
      const float4* r = reinterpret_cast<const float4*>(a.records + id);
      const uint32_t ex = __ldg(a.excl + id);
      const float4 q0 = __ldg(r);
      s_q0[tid] = q0;
      s_q1[tid] = __ldg(r + 1);
      s_ids[tid] = id;
      s_slot[tid] = emission_slot(ex, q0.x, q0.y, __float_as_int(__ldg(r + 2).w), a.gx, a.gy, blockIdx.x, ty,
                                  a.own_stride, a.own_phase);
    }
    __syncthreads();
    const int n = min(TILE_PIX, toDo);
    for (int j = 0; j < n; j++) {
      bool hit = false;
      if (!done) {
        const float4 q0 = s_q0[j], q1 = s_q1[j];
        const float dx = q0.x - pixf.x, dy = q0.y - pixf.y;
        const float power = splat_power(dx, dy, q0.z, q0.w, q1.x);
        if (!(power > 0.0f)) {
          const float alpha = fminf(0.99f, __fmul_rn(q1.y, expf(power)));
          if (!(alpha < 1.0f / 255.0f)) {
            const float test_T = __fmul_rn(T, __fadd_rn(1.0f, -alpha));
            if (test_T < 0.0001f) {
              done = true;
            } else {
              hit = true;
              T = test_T;
            }
          }
        }
      }
      const unsigned hits = __ballot_sync(0xffffffffu, hit);
      if (hits) {
#pragma unroll
        for (int ch = 0; ch < CH; ch++) {
          float v = hit ? Cw[ch] : 0.f;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          if (lane == 0) s_w[warp][j][ch] = v;
        }
        if (lane == 0) atomicAdd(a.cnt + (size_t)s_ids[j] * a.c_stride, CH * __popc(hits));
      } else if (lane == 0) {
#pragma unroll
        for (int ch = 0; ch < CH; ch++) s_w[warp][j][ch] = 0.f;
      }
    }
    prev_n = n;
  }
  if (prev_n > 0) {  // block-uniform: the last round ran to its end
    __syncthreads();
    flush(prev_n);
  }
}

// Deterministic walk of the owned tile rows (grid.y of them) + the reduction into the packed weights [P, CH].
int launch_apply_weights_det(const gsr_settings& s, const GeometryWS& g, const AwArgs& a, int CH, int64_t c_stride,
                             const TileOwner& own, dim3 grid, cudaStream_t st, const DetWS& det, int P, int64_t R) {
  int rc = launch_det_prepare(P, R, 1, g, det, st);
  if (rc) return rc;
  AwDetArgs da;
  static_cast<AwArgs&>(da) = a;
  da.excl = det.excl; da.rows = det.rows; da.flags = det.flags;
  da.own_stride = own.stride; da.own_phase = own.phase; da.c_stride = c_stride;
  const dim3 block(TILE, TILE);
  if (CH == 1) apply_weights_det_kernel<1><<<grid, block, 0, st>>>(da);
  else if (CH == 2) apply_weights_det_kernel<2><<<grid, block, 0, st>>>(da);
  else apply_weights_det_kernel<3><<<grid, block, 0, st>>>(da);
  g_launches++;
  if ((rc = check_launch("apply_weights", s.debug != 0, st))) return rc;
  return launch_det_reduce_weights(P, CH, g, det, a.weights, st);
}

}  // namespace

int launch_apply_weights(const gsr_settings& s, const GeometryWS& g, const BinningWS& b, const ImageWS& im,
                         const float* image_weights, int CH, float* weights, int32_t* cnt, cudaStream_t st,
                         const DetWS* det, int P, int64_t R) {
  AwArgs a;
  a.ranges = im.ranges; a.point_list = b.point_list; a.records = g.records;
  a.W = s.image_width; a.H = s.image_height;
  a.gx = (a.W + TILE - 1) / TILE; a.gy = (a.H + TILE - 1) / TILE;
  a.image_weights = image_weights; a.weights = weights; a.cnt = cnt;
  if (a.gx * a.gy == 0) return GSR_OK;
  dim3 grid(a.gx, a.gy), block(TILE, TILE);
  if (det != nullptr && CH >= 1 && CH <= 3)
    return launch_apply_weights_det(s, g, a, CH, 1, TileOwner(), grid, st, *det, P, R);
  if (CH == 1) apply_weights_kernel<1><<<grid, block, 0, st>>>(a);
  else if (CH == 2) apply_weights_kernel<2><<<grid, block, 0, st>>>(a);
  else if (CH == 3) apply_weights_kernel<3><<<grid, block, 0, st>>>(a);
  else {
    set_error("apply_weights: unsupported number of channels %d (reference supports 1..3, apply_weights.cu:365-380)", CH);
    return GSR_ERR_INVALID;
  }
  g_launches++;
  return check_launch("apply_weights", s.debug != 0, st);
}

int launch_apply_weights_owner(const gsr_settings& s, const GeometryWS& g, const BinningWS& b, const ImageWS& im,
                               const float* image_weights, int CH, float* weights, int64_t w_stride, int32_t* cnt,
                               int64_t c_stride, const TileOwner& own, cudaStream_t st, const DetWS* det, int P,
                               int64_t R) {
  AwOwnerArgs a;
  a.ranges = im.ranges; a.point_list = b.point_list; a.records = g.records;
  a.W = s.image_width; a.H = s.image_height;
  a.gx = (a.W + TILE - 1) / TILE; a.gy = (a.H + TILE - 1) / TILE;
  a.image_weights = image_weights; a.weights = weights; a.cnt = cnt;
  a.own_stride = own.stride; a.own_phase = own.phase; a.w_stride = w_stride; a.c_stride = c_stride;
  const int rows = own.owned_rows(a.gy);
  if (a.gx * rows == 0) return GSR_OK;
  dim3 grid(a.gx, rows), block(TILE, TILE);
  if (det != nullptr && CH >= 1 && CH <= 3 && w_stride == CH)
    return launch_apply_weights_det(s, g, a, CH, c_stride, own, grid, st, *det, P, R);
  if (det != nullptr) {
    set_error("apply_weights: deterministic mode needs 1..3 channels and weights_stride == num_channels");
    return GSR_ERR_INVALID;
  }
  if (CH == 1) apply_weights_owner_kernel<1><<<grid, block, 0, st>>>(a);
  else if (CH == 2) apply_weights_owner_kernel<2><<<grid, block, 0, st>>>(a);
  else if (CH == 3) apply_weights_owner_kernel<3><<<grid, block, 0, st>>>(a);
  else {
    set_error("apply_weights: unsupported number of channels %d (reference supports 1..3, apply_weights.cu:365-380)", CH);
    return GSR_ERR_INVALID;
  }
  g_launches++;
  return check_launch("apply_weights", s.debug != 0, st);
}

}  // namespace gsr
