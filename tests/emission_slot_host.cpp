// Host build of the emission-slot helpers of gaussianeditor_b200/csrc/common.cuh (tile_rect, owned_rows,
// emission_slot) for tests/test_sharded_deterministic.py: the deterministic kernels store their rows at these slots,
// so the test checks the header's own arithmetic. Built with -ffp-contract=off, so the host rounds like the device.
#include <stdint.h>

#include "../gaussianeditor_b200/csrc/common.cuh"

extern "C" {

// owned tile count of each splat on the rank that owns the tile rows ty % stride == phase (the sharded tiles_touched)
void owned_counts(int n, const float* px, const float* py, const int32_t* radius, int gx, int gy, int stride, int phase,
                  uint32_t* out) {
  for (int i = 0; i < n; i++) {
    if (radius[i] <= 0) { out[i] = 0; continue; }
    uint2 rmin, rmax;
    gsr::tile_rect(px[i], py[i], radius[i], gx, gy, rmin, rmax);
    uint32_t y0, ny;
    gsr::owned_rows(rmin.y, rmax.y, stride, phase, y0, ny);
    out[i] = ny * (rmax.x - rmin.x);
  }
}

// emission slot of each instance (splat at (px, py) with radius and exclusive prefix excl, tile (tx, ty))
void owner_slots(int n, const float* px, const float* py, const int32_t* radius, const uint32_t* excl,
                 const int32_t* tx, const int32_t* ty, int gx, int gy, int stride, int phase, uint32_t* out) {
  for (int i = 0; i < n; i++)
    out[i] = gsr::emission_slot(excl[i], px[i], py[i], radius[i], gx, gy, tx[i], ty[i], stride, phase);
}
}
