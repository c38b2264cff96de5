// Semantic tracing ("apply_weights") for sm_90a.
//
// Semantics: renderCUDA_apply_weights of GaussianEditor's fork (cuda_rasterizer/apply_weights.cu:240-356):
// the forward walk of a tile list with the forward's skip / stop rules, but instead of blending, every
// (pixel, splat) pair that WOULD be blended adds the pixel's 2-D mask value to the splat:
//     weights[id*CH + ch] += image_weights[ch, pixel];   cnt[id] += 1      (once per channel, :331-334)
// No image is written.  The reference issues 2*CH global atomics per hit; here the hits of a warp on the same
// splat are summed with shuffles first (one atomic pair per warp and splat) and the same opacity-aware tile
// culling as the render kernels drops splats that cannot reach alpha >= 1/255 inside the tile.
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

template <int CH>
__global__ void __launch_bounds__(TILE_PIX) apply_weights_kernel(const AwArgs a) {
  __shared__ float4 s_q0[TILE_PIX], s_q1[TILE_PIX];
  __shared__ uint32_t s_ids[TILE_PIX];
  const int tile = blockIdx.y * a.gx + blockIdx.x;
  const int tid = threadIdx.y * TILE + threadIdx.x;
  const int lane = tid & 31;
  const uint2 pix = make_uint2(blockIdx.x * TILE + threadIdx.x, blockIdx.y * TILE + threadIdx.y);
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
          if (lane == 0) atomicAdd(a.weights + (size_t)id * CH + ch, v);
        }
        if (lane == 0) atomicAdd(a.cnt + id, CH * __popc(hits));
      }
    }
  }
}

}  // namespace

int launch_apply_weights(const gsr_settings& s, const GeometryWS& g, const BinningWS& b, const ImageWS& im,
                         const float* image_weights, int CH, float* weights, int32_t* cnt, cudaStream_t st) {
  AwArgs a;
  a.ranges = im.ranges; a.point_list = b.point_list; a.records = g.records;
  a.W = s.image_width; a.H = s.image_height;
  a.gx = (a.W + TILE - 1) / TILE; a.gy = (a.H + TILE - 1) / TILE;
  a.image_weights = image_weights; a.weights = weights; a.cnt = cnt;
  if (a.gx * a.gy == 0) return GSR_OK;
  dim3 grid(a.gx, a.gy), block(TILE, TILE);
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

}  // namespace gsr
