// Geometry extraction: the points of a layer's density field at one frame, and marching cubes on a sampled grid.
//
// field_points_kernel builds the network inputs of stnerf_layer_field / stnerf_layer_grid: a world point (given, or grid point
// origin + (i,j,k)*step), the inverse edit of the pass (inverse_edit, common.cuh), and the frame id as the
// time column.  api.cu then runs the context's MotionNet / SpaceNet on them (SRC_EXPLICIT), as stnerf_render does.
//
// Marching cubes (no context): a corner is inside when v > level (NaN is outside).  Every grid point owns the vertices of its
// +x/+y/+z edges, so neighbouring cells share vertex ids; the triangle table is mc_table.cuh (scripts/gen_mc_table.py).
//   mc_case_kernel   per cell: case index and triangle count
//   mc_edge_kernel   per grid point: crossing edges (bit a = the +a edge) and their count
//   cub::DeviceScan  exclusive sums of both counts -> vertex ids (grid-point-major), triangle offsets (cell-major)
//   mc_vert_kernel / mc_face_kernel   the emission
// Compiled with -fmad=false: grid points and edge interpolation round every product and sum on its own.
#include <cub/cub.cuh>
#include <math.h>
#include "common.cuh"
#include "mc_table.cuh"

namespace stnerf {

constexpr int EX_BLOCK = 256;

// ---------------------------------------------------------------------------------------------------------
// network inputs of a layer's field
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(EX_BLOCK)
field_points_kernel(const float* __restrict__ xyz, FieldGrid g, long long p0, long long n, FieldEdit e, float frame,
                    float* __restrict__ xyzt, const float* __restrict__ dirs, float* __restrict__ rdirs) {
  const long long j = (long long)blockIdx.x * EX_BLOCK + threadIdx.x;
  if (j >= n) return;
  const long long p = p0 + j;
  float v[3];
  if (xyz) {
    v[0] = xyz[3 * p]; v[1] = xyz[3 * p + 1]; v[2] = xyz[3 * p + 2];
  } else {                                          // x slowest: sigma[i][j][k] is meshgrid(indexing="ij")
    const long long nyz = (long long)g.dims[1] * g.dims[2];
    const int idx[3] = {(int)(p / nyz), (int)((p / g.dims[2]) % g.dims[1]), (int)(p % g.dims[2])};
#pragma unroll
    for (int a = 0; a < 3; ++a) v[a] = __fadd_rn(__fmul_rn((float)idx[a], g.step[a]), g.origin[a]);
  }
  // a rotated layer: back into the layer first, with the op order of rotate_rays_kernel (the render's o' = c + R^T (o - c))
  if (e.rot_on) {
    const float w[3] = {v[0], v[1], v[2]};
    rotate_back_point(e.rot, w, v);
    if (dirs) {
      const float d[3] = {dirs[3 * p], dirs[3 * p + 1], dirs[3 * p + 2]};
      float d2[3];
      rotate_back_dir(e.rot, d, d2);
      rdirs[3 * j] = d2[0]; rdirs[3 * j + 1] = d2[1]; rdirs[3 * j + 2] = d2[2];
    }
  }
  inverse_edit(e, v);
  reinterpret_cast<float4*>(xyzt)[j] = make_float4(v[0], v[1], v[2], frame);
}

int launch_field_points(const float* xyz, const FieldGrid& g, long long p0, long long n, const FieldEdit& e, float frame,
                        float* xyzt, const float* dirs, float* rdirs, cudaStream_t st) {
  if (n <= 0) return STNERF_OK;
  field_points_kernel<<<(unsigned)((n + EX_BLOCK - 1) / EX_BLOCK), EX_BLOCK, 0, st>>>(xyz, g, p0, n, e, frame, xyzt,
                                                                                     e.rot_on ? dirs : nullptr, rdirs);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// marching cubes
// ---------------------------------------------------------------------------------------------------------
// cube edge e (Bourke's numbering) = the +axis edge of the cell corner at offset (dx, dy, dz): packed as dx | dy<<1 | dz<<2 | axis<<3
__constant__ uint8_t c_mc_edge[12] = {0 | 0 << 3, 1 | 1 << 3, 2 | 0 << 3, 0 | 1 << 3, 4 | 0 << 3, 5 | 1 << 3,
                                      6 | 0 << 3, 4 | 1 << 3, 0 | 2 << 3, 1 | 2 << 3, 3 | 2 << 3, 2 | 2 << 3};

struct McDims {
  int n[3];
  long long points, cells;
};

__device__ __forceinline__ bool mc_inside(float v, float level) { return v > level; }     // false for NaN

__global__ void __launch_bounds__(EX_BLOCK)
mc_case_kernel(const float* __restrict__ sigma, McDims d, float level, uint8_t* __restrict__ cases, int* __restrict__ tcount) {
  const long long c = (long long)blockIdx.x * EX_BLOCK + threadIdx.x;
  if (c >= d.cells) return;
  const int cy = d.n[1] - 1, cz = d.n[2] - 1;
  const int i = (int)(c / ((long long)cy * cz)), j = (int)((c / cz) % cy), k = (int)(c % cz);
  const long long sx = (long long)d.n[1] * d.n[2], sy = d.n[2];
  const long long b = i * sx + j * sy + k;
  // corners in Bourke's order: (0,0,0) (1,0,0) (1,1,0) (0,1,0), then the same at z + 1
  const long long off[8] = {0, sx, sx + sy, sy, 1, sx + 1, sx + sy + 1, sy + 1};
  int cs = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) cs |= mc_inside(sigma[b + off[q]], level) ? (1 << q) : 0;
  cases[c] = (uint8_t)cs;
  tcount[c] = c_mc_ntri[cs];
}

__global__ void __launch_bounds__(EX_BLOCK)
mc_edge_kernel(const float* __restrict__ sigma, McDims d, float level, uint8_t* __restrict__ emask, int* __restrict__ vcount) {
  const long long p = (long long)blockIdx.x * EX_BLOCK + threadIdx.x;
  if (p >= d.points) return;
  const long long sx = (long long)d.n[1] * d.n[2], sy = d.n[2];
  const int i = (int)(p / sx), j = (int)((p / sy) % d.n[1]), k = (int)(p % sy);
  const bool in0 = mc_inside(sigma[p], level);
  int m = 0;
  if (i + 1 < d.n[0] && mc_inside(sigma[p + sx], level) != in0) m |= 1;
  if (j + 1 < d.n[1] && mc_inside(sigma[p + sy], level) != in0) m |= 2;
  if (k + 1 < d.n[2] && mc_inside(sigma[p + 1], level) != in0) m |= 4;
  emask[p] = (uint8_t)m;
  vcount[p] = __popc(m);
}

__global__ void mc_totals_kernel(const int* __restrict__ vcount, const long long* __restrict__ voff, long long np,
                                 const int* __restrict__ tcount, const long long* __restrict__ toff, long long nc,
                                 long long* __restrict__ totals) {
  totals[0] = voff[np - 1] + vcount[np - 1];
  totals[1] = toff[nc - 1] + tcount[nc - 1];
}

__global__ void __launch_bounds__(EX_BLOCK)
mc_vert_kernel(const float* __restrict__ sigma, McDims d, FieldGrid g, float level, const uint8_t* __restrict__ emask,
               const long long* __restrict__ voff, float* __restrict__ verts) {
  const long long p = (long long)blockIdx.x * EX_BLOCK + threadIdx.x;
  if (p >= d.points) return;
  const int m = emask[p];
  if (!m) return;
  const long long sx = (long long)d.n[1] * d.n[2], sy = d.n[2];
  const int idx[3] = {(int)(p / sx), (int)((p / sy) % d.n[1]), (int)(p % sy)};
  const long long stride[3] = {sx, sy, 1};
  float base[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) base[a] = __fadd_rn(__fmul_rn((float)idx[a], g.step[a]), g.origin[a]);
  const float v0 = sigma[p];
  long long vid = voff[p];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!(m & (1 << a))) continue;
    const float v1 = sigma[p + stride[a]];
    float t = __fdiv_rn(__fsub_rn(level, v0), __fsub_rn(v1, v0));
    // finite values give t in [0, 1]; with a NaN or an infinite endpoint the vertex goes to the outside endpoint
    if (!(t >= 0.f && t <= 1.f)) t = mc_inside(v0, level) ? 1.f : 0.f;
    const float x1 = __fadd_rn(__fmul_rn((float)(idx[a] + 1), g.step[a]), g.origin[a]);
    float out[3] = {base[0], base[1], base[2]};
    out[a] = __fadd_rn(base[a], __fmul_rn(t, __fsub_rn(x1, base[a])));
    verts[3 * vid] = out[0]; verts[3 * vid + 1] = out[1]; verts[3 * vid + 2] = out[2];
    ++vid;
  }
}

__global__ void __launch_bounds__(EX_BLOCK)
mc_face_kernel(McDims d, const uint8_t* __restrict__ cases, const long long* __restrict__ toff, const uint8_t* __restrict__ emask,
               const long long* __restrict__ voff, int* __restrict__ faces) {
  const long long c = (long long)blockIdx.x * EX_BLOCK + threadIdx.x;
  if (c >= d.cells) return;
  const int cs = cases[c];
  const int nt = c_mc_ntri[cs];
  if (!nt) return;
  const int cy = d.n[1] - 1, cz = d.n[2] - 1;
  const int i = (int)(c / ((long long)cy * cz)), j = (int)((c / cz) % cy), k = (int)(c % cz);
  const long long sx = (long long)d.n[1] * d.n[2], sy = d.n[2];
  const long long b = i * sx + j * sy + k;
  const long long t0 = toff[c];
  for (int t = 0; t < nt; ++t) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const int e = c_mc_edge[c_mc_tri[cs][3 * t + q]];
      const long long p = b + ((e & 1) ? sx : 0) + ((e & 2) ? sy : 0) + ((e & 4) ? 1 : 0);
      const int axis = e >> 3;
      faces[3 * (t0 + t) + q] = (int)(voff[p] + __popc(emask[p] & ((1 << axis) - 1)));
    }
  }
}

namespace {
struct ToI64 {
  __host__ __device__ long long operator()(int x) const { return (long long)x; }
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// scratch layout of one grid: emask[points] u8 | cases[cells] u8 | vcount[points] i32 | tcount[cells] i32 |
// voff[points] i64 | toff[cells] i64 | totals[2] i64 | cub temp storage
struct McScratch {
  uint8_t *emask, *cases;
  int *vcount, *tcount;
  long long *voff, *toff, *totals;
  void* temp;
  size_t temp_bytes, total;
};

McScratch mc_layout(const McDims& d, void* base) {
  McScratch s{};
  size_t tb_p = 0, tb_c = 0;
  cub::TransformInputIterator<long long, ToI64, const int*> it(nullptr, ToI64());
  cub::DeviceScan::ExclusiveSum(nullptr, tb_p, it, (long long*)nullptr, (int)d.points);
  cub::DeviceScan::ExclusiveSum(nullptr, tb_c, it, (long long*)nullptr, (int)d.cells);
  s.temp_bytes = tb_p > tb_c ? tb_p : tb_c;
  uint8_t* p = static_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* q = p ? p + off : nullptr; off += align256(bytes); return q; };
  s.emask = take(d.points);
  s.cases = take(d.cells);
  s.vcount = (int*)take(4 * d.points);
  s.tcount = (int*)take(4 * d.cells);
  s.voff = (long long*)take(8 * d.points);
  s.toff = (long long*)take(8 * d.cells);
  s.totals = (long long*)take(16);
  s.temp = take(s.temp_bytes);
  s.total = off;
  return s;
}

unsigned blocks_of(long long n) { return (unsigned)((n + EX_BLOCK - 1) / EX_BLOCK); }
}  // namespace

// dims >= 2 on every axis, finite origin, finite positive steps, fewer than 2^31 points
bool mc_dims(const stnerf_grid& g, McDims& d, FieldGrid& geo) {
  long long np = 1, nc = 1;
  for (int a = 0; a < 3; ++a) {
    if (g.dims[a] < 2 || !isfinite(g.origin[a]) || !isfinite(g.step[a]) || !(g.step[a] > 0.f)) return false;
    d.n[a] = g.dims[a];
    np *= g.dims[a];
    nc *= g.dims[a] - 1;
    if (np >= (1LL << 31)) return false;
    geo.origin[a] = g.origin[a];
    geo.step[a] = g.step[a];
  }
  d.points = np;
  d.cells = nc;
  return true;
}

size_t mc_scratch_bytes(const McDims& d) { return mc_layout(d, nullptr).total; }

int mc_count(const float* sigma, const McDims& d, float level, void* scratch, long long* totals_host, cudaStream_t st) {
  const McScratch s = mc_layout(d, scratch);
  mc_case_kernel<<<blocks_of(d.cells), EX_BLOCK, 0, st>>>(sigma, d, level, s.cases, s.tcount);
  STNERF_LAUNCH_CHECK();
  mc_edge_kernel<<<blocks_of(d.points), EX_BLOCK, 0, st>>>(sigma, d, level, s.emask, s.vcount);
  STNERF_LAUNCH_CHECK();
  size_t tb = s.temp_bytes;
  cub::TransformInputIterator<long long, ToI64, const int*> vin(s.vcount, ToI64()), tin(s.tcount, ToI64());
  STNERF_CUDA(cub::DeviceScan::ExclusiveSum(s.temp, tb, vin, s.voff, (int)d.points, st));
  tb = s.temp_bytes;
  STNERF_CUDA(cub::DeviceScan::ExclusiveSum(s.temp, tb, tin, s.toff, (int)d.cells, st));
  mc_totals_kernel<<<1, 1, 0, st>>>(s.vcount, s.voff, d.points, s.tcount, s.toff, d.cells, s.totals);
  STNERF_LAUNCH_CHECK();
  STNERF_CUDA(cudaMemcpyAsync(totals_host, s.totals, 16, cudaMemcpyDeviceToHost, st));
  STNERF_CUDA(cudaStreamSynchronize(st));      // the one host sync: the caller sizes verts / faces from the counts
  return STNERF_OK;
}

int mc_fill(const float* sigma, const McDims& d, const FieldGrid& g, float level, void* scratch, float* verts, int* faces,
            cudaStream_t st) {
  const McScratch s = mc_layout(d, scratch);
  mc_vert_kernel<<<blocks_of(d.points), EX_BLOCK, 0, st>>>(sigma, d, g, level, s.emask, s.voff, verts);
  STNERF_LAUNCH_CHECK();
  mc_face_kernel<<<blocks_of(d.cells), EX_BLOCK, 0, st>>>(d, s.cases, s.toff, s.emask, s.voff, faces);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

}  // namespace stnerf

using namespace stnerf;

extern "C" {

size_t stnerf_mc_scratch_bytes(const stnerf_grid* grid_host) {
  McDims d;
  FieldGrid g;
  if (!grid_host || !mc_dims(*grid_host, d, g)) return 0;
  return mc_scratch_bytes(d);
}

int stnerf_mc_count(const float* sigma, const stnerf_grid* grid_host, float level, void* scratch, size_t scratch_bytes,
                    int64_t* n_verts_host, int64_t* n_faces_host, void* stream) {
  McDims d;
  FieldGrid g;
  if (!grid_host || !mc_dims(*grid_host, d, g) || !sigma || !scratch || !n_verts_host || !n_faces_host) return STNERF_EINVAL;
  if (scratch_bytes < mc_scratch_bytes(d)) return STNERF_EINVAL;
  long long tot[2];
  const int rc = mc_count(sigma, d, level, scratch, tot, (cudaStream_t)stream);
  if (rc) return rc;
  *n_verts_host = tot[0];
  *n_faces_host = tot[1];
  return tot[0] > 0x7fffffffLL ? STNERF_EINVAL : STNERF_OK;     // faces hold int32 vertex ids
}

int stnerf_mc_fill(const float* sigma, const stnerf_grid* grid_host, float level, void* scratch, size_t scratch_bytes,
                   float* verts, int32_t* faces, void* stream) {
  McDims d;
  FieldGrid g;
  if (!grid_host || !mc_dims(*grid_host, d, g) || !sigma || !scratch || !verts || !faces) return STNERF_EINVAL;
  if (scratch_bytes < mc_scratch_bytes(d)) return STNERF_EINVAL;
  return mc_fill(sigma, d, g, level, scratch, verts, faces, (cudaStream_t)stream);
}

}  // extern "C"
