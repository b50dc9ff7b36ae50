// One pixel's ray (utils/render_helpers.py:96-123 == utils/ray_sampling.py:22-72), shared by the render path's
// raygen_kernel (geometry.cu) and the training batch kernel (train_data.cu) so a training ray is bit-identical to the
// render ray of the same camera and pixel.  Both files are compiled with -fmad=false: every product and sum rounds
// separately, as the reference's eager fp32 ops do.
#pragma once

namespace stnerf {

// c = normalize(K^-1 (px, py, 1)), kinv 3x3 row-major.  The tables are taken by reference to whatever holds them (kernel
// parameters, global memory), so the caller's loads are the ones it would have written itself.
template <class Kinv>
__device__ __forceinline__ void raygen_dir(const Kinv& kinv, float px, float py, float c[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = (kinv[3 * a] * px + kinv[3 * a + 1] * py) + kinv[3 * a + 2];
  const float nrm = sqrtf((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]);
  c[0] = c[0] / nrm; c[1] = c[1] / nrm; c[2] = c[2] / nrm;
}

// out[0..2] = camera origin, out[3..5] = R c, rot 3x3 row-major.
template <class Rot, class Org>
__device__ __forceinline__ void raygen_write(const Rot& rot, const Org& org, const float c[3], float* out) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    out[a] = org[a];
    out[3 + a] = (rot[3 * a] * c[0] + rot[3 * a + 1] * c[1]) + rot[3 * a + 2] * c[2];
  }
}

}  // namespace stnerf
