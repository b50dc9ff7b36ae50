// C ABI of libstnerf_b200 (include/stnerf.h): context, weight packing, workspace, chunked render orchestration.
//
// The orchestration restates the control flow of modeling/layered_rfrender.py:141-734 (BBOX sampling) as a
// stream-ordered sequence of kernels per chunk of rays -- no host synchronisation, hit counts stay on the device:
//   sample -> [bkgd SpaceNet] -> per performer [MotionNet -> SpaceNet] -> composite+resample
//          -> same nets (fine weights) on n1+n2 depths -> per-layer + merged composite.
#include <algorithm>
#include <new>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "common.cuh"
#include "mlp_tc.cuh"

namespace stnerf {
thread_local char g_cuda_err[512] = "";
std::atomic<unsigned long long> g_launches{0};
}  // namespace stnerf

using namespace stnerf;

namespace {

struct SpaceNetDev {
  float* blob = nullptr;       // SIMT layout (transposed fp32)
  SpaceNetW w{};
  TcNet tc{};                  // tensor-core packing (mlp_tc.cu)
  bool loaded = false;
};
struct MotionNetDev {
  float* blob = nullptr;
  MotionNetW w{};
  TcNet tc{};
  bool loaded = false;
};

}  // namespace

struct stnerf_ctx {
  stnerf_model_desc desc{};
  int l = 0, num_sms = 0, device = 0, precision = 0, chunk_rays = 65536;
  SpaceNetDev space[2][STNERF_MAX_LAYERS];
  MotionNetDev motion[STNERF_MAX_LAYERS];
  stnerf_scene scene{};
  DevScene dscene{};
  bool have_scene = false;
  // workspace (sized for chunk_rays rays, cap_n1 coarse and cap_s2 total samples)
  int cap_n1 = 0, cap_s2 = 0;
  long long last_chunk_rays = 0;       // geometry of the most recent chunk (stnerf_debug_read_depths)
  int last_n1 = 0, last_s2 = 0;
  bool last_reuse = false;             // that chunk's coarse pass wrote z_new / src_map
  float *t_coarse = nullptr, *raw_coarse = nullptr, *t_fine = nullptr, *raw_fine = nullptr, *xyz = nullptr;
  // flow reuse (fine pass): per performer layer the coarse pass' deformed points, the new depths and the origin map of t_fine
  float *xyz_coarse = nullptr, *z_new = nullptr;
  uint8_t* src_map = nullptr;
  bool no_reuse = false;       // STNERF_NO_REUSE=1 at create: the fine pass evaluates the MotionNet on all n1+n2 depths (A/B)
  float* cbuf = nullptr;       // per-slot rgb_net.1 bias of the SpaceNet being evaluated (tensor-core modes)
  uint8_t* mask_ws = nullptr;
  int *hit = nullptr, *counts = nullptr, *lerp_flags = nullptr;
  size_t ws_bytes = 0;
  // staging for stnerf_render_host
  float *h_rays = nullptr, *h_out = nullptr;
  uint8_t* h_mask = nullptr;
  size_t h_rays_bytes = 0, h_out_bytes = 0, h_mask_bytes = 0;
  // staging for stnerf_render_views(_host): rays of one view, two image buffers (double-buffered device->host copies)
  float *v_rays = nullptr, *v_img[2] = {nullptr, nullptr};
  size_t v_rays_bytes = 0, v_img_bytes[2] = {0, 0};
  cudaStream_t copy_in = nullptr, copy_out = nullptr;      // host<->device copies that overlap the kernels of other chunks
  std::vector<cudaEvent_t> ev_pool;                         // timing-disabled events, reused call after call
  float* box_table = nullptr;  // [n_frames][l][2][3] per-frame boxes for rays with their own frame id (stnerf_set_box_table)
  int box_frames = 0;
  bool no_fuse = false;        // STNERF_NO_FUSE=1 in the environment at create: keep the coarse compositing in its own kernel (A/B)
  int* any_frac = nullptr;     // scratch flag for stnerf_motionnet(lerp_mode=-1)
  RayIdMap idmap{0, 0, 0};     // stnerf_set_ray_ids
  // stnerf_set_rotation: per layer STNERF_ROT_*, R (row-major) and the explicit centre
  int rot_mode[STNERF_MAX_LAYERS] = {0};
  float rot_R[STNERF_MAX_LAYERS][9] = {}, rot_c[STNERF_MAX_LAYERS][3] = {};
  // profiling (stnerf_profile_begin / _end): CUDA-event pairs around every launch, on the launching stream
  struct ProfRec { int cls; cudaEvent_t a, b; double points; int count_slot; int S; };
  bool prof_on = false;
  std::vector<ProfRec> prof;
  int* prof_counts = nullptr;  // pinned host copies of the per-chunk hit counts
  int prof_chunks = 0;
};

namespace {
constexpr int PROF_MAX_CHUNKS = 1 << 16;
struct ProfScope {
  stnerf_ctx* c; int idx = -1; cudaStream_t st;
  ProfScope(stnerf_ctx* c_, int cls, double points, int count_slot, int S, cudaStream_t st_) : c(c_), st(st_) {
    if (!c->prof_on) return;
    stnerf_ctx::ProfRec r{cls, nullptr, nullptr, points, count_slot, S};
    if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
    cudaEventRecord(r.a, st);
    c->prof.push_back(r);
    idx = (int)c->prof.size() - 1;
  }
  ~ProfScope() { if (idx >= 0) cudaEventRecord(c->prof[idx].b, st); }
};
}  // namespace

static void free_ws(stnerf_ctx* c) {
  cudaFree(c->t_coarse); cudaFree(c->raw_coarse); cudaFree(c->t_fine); cudaFree(c->raw_fine); cudaFree(c->xyz);
  cudaFree(c->xyz_coarse); cudaFree(c->z_new); cudaFree(c->src_map);
  c->xyz_coarse = c->z_new = nullptr; c->src_map = nullptr;
  cudaFree(c->cbuf); c->cbuf = nullptr;
  cudaFree(c->mask_ws); cudaFree(c->hit); cudaFree(c->counts); cudaFree(c->lerp_flags);
  c->t_coarse = c->raw_coarse = c->t_fine = c->raw_fine = c->xyz = nullptr;
  c->mask_ws = nullptr; c->hit = c->counts = c->lerp_flags = nullptr;
  c->ws_bytes = 0; c->cap_n1 = c->cap_s2 = 0;
}

static int ensure_ws(stnerf_ctx* c, int n1, int s2) {
  if (n1 <= c->cap_n1 && s2 <= c->cap_s2 && c->t_coarse) return STNERF_OK;
  const int cn1 = std::max(n1, c->cap_n1), cs2 = std::max(s2, c->cap_s2);
  free_ws(c);
  const size_t R = (size_t)c->chunk_rays, l = (size_t)c->l;
  size_t tot = 0;
  auto A = [&](void** p, size_t bytes) -> int {
    if (cudaMalloc(p, bytes) != cudaSuccess) { cudaGetLastError(); return STNERF_ENOMEM; }
    tot += bytes;
    return STNERF_OK;
  };
  int rc = 0;
  rc |= A((void**)&c->t_coarse, l * R * cn1 * 4);
  rc |= A((void**)&c->raw_coarse, l * R * cn1 * 16);
  rc |= A((void**)&c->t_fine, l * R * cs2 * 4);
  rc |= A((void**)&c->raw_fine, l * R * cs2 * 16);
  rc |= A((void**)&c->xyz, R * cs2 * 12);
  rc |= A((void**)&c->xyz_coarse, l * R * cn1 * 12);
  rc |= A((void**)&c->z_new, l * R * cs2 * 4);
  rc |= A((void**)&c->src_map, l * R * cs2);
  rc |= A((void**)&c->cbuf, R * 128 * 4);
  rc |= A((void**)&c->mask_ws, l * R);
  rc |= A((void**)&c->hit, l * R * 4);
  rc |= A((void**)&c->counts, STNERF_MAX_LAYERS * 4);
  rc |= A((void**)&c->lerp_flags, STNERF_MAX_LAYERS * 4);
  if (rc) { free_ws(c); return STNERF_ENOMEM; }
  c->cap_n1 = cn1; c->cap_s2 = cs2; c->ws_bytes = tot;
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// weight packing (host): state_dict order blob -> transposed [k][n] fp32 for the SIMT kernels
// ---------------------------------------------------------------------------------------------------------
static void transpose_into(std::vector<float>& dst, const float* W, int N, int K) {   // W (N,K) -> [K][N]
  const size_t base = dst.size();
  dst.resize(base + (size_t)N * K);
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) dst[base + (size_t)k * N + n] = W[(size_t)n * K + k];
}

static int upload(float** dev, const std::vector<float>& host) {
  if (*dev) { cudaFree(*dev); *dev = nullptr; }
  STNERF_CUDA(cudaMalloc((void**)dev, host.size() * sizeof(float)));
  STNERF_CUDA(cudaMemcpy(*dev, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice));
  return STNERF_OK;
}

extern "C" {

const char* stnerf_strerror(int code) {
  switch (code) {
    case STNERF_OK: return "ok";
    case STNERF_EINVAL: return "invalid argument";
    case STNERF_ENODEVICE: return "no usable CUDA device (needs sm_90)";
    case STNERF_ECUDA: return "CUDA runtime error (see stnerf_last_cuda_error)";
    case STNERF_ENOWEIGHTS: return "network weights not loaded";
    case STNERF_ENOMEM: return "out of device memory";
    default: return "unknown error";
  }
}
const char* stnerf_last_cuda_error(void) { return g_cuda_err; }
uint64_t stnerf_launch_count(void) { return g_launches.load(); }

int stnerf_create(stnerf_handle* out, const stnerf_model_desc* d) {
  if (!out || !d || d->n_layers < 2 || d->n_layers > STNERF_MAX_LAYERS) return STNERF_EINVAL;
  if (d->precision < 0 || d->precision > STNERF_PREC_TC_3XF16_CF || d->chunk_rays < 0) return STNERF_EINVAL;
  // the kernels index samples of a chunk with 32-bit integers: chunk_rays * STNERF_MAX_S must stay below 2^31
  if ((long long)d->chunk_rays * STNERF_MAX_S >= (1LL << 31)) return STNERF_EINVAL;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return STNERF_ENODEVICE; }
  int dev = 0;
  STNERF_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  STNERF_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0) return STNERF_ENODEVICE;     // the cubin is sm_90a only
  stnerf_ctx* c = new (std::nothrow) stnerf_ctx();
  if (!c) return STNERF_ENOMEM;
  c->desc = *d;
  c->l = d->n_layers;
  c->device = dev;
  c->num_sms = prop.multiProcessorCount;
  c->precision = d->precision;
  c->chunk_rays = d->chunk_rays > 0 ? d->chunk_rays : 65536;
  if (const char* e = getenv("STNERF_NO_FUSE")) c->no_fuse = (e[0] == '1');
  if (const char* e = getenv("STNERF_NO_REUSE")) c->no_reuse = (e[0] == '1');
  if (cudaMalloc((void**)&c->any_frac, 4) != cudaSuccess) { delete c; return STNERF_ENOMEM; }
  *out = c;
  return STNERF_OK;
}

void stnerf_destroy(stnerf_handle c) {
  if (!c) return;
  cudaDeviceSynchronize();
  free_ws(c);
  for (int f = 0; f < 2; ++f)
    for (int i = 0; i < STNERF_MAX_LAYERS; ++i) { cudaFree(c->space[f][i].blob); tc_free(c->space[f][i].tc); }
  for (int i = 0; i < STNERF_MAX_LAYERS; ++i) { cudaFree(c->motion[i].blob); tc_free(c->motion[i].tc); }
  cudaFree(c->h_rays); cudaFree(c->h_out); cudaFree(c->h_mask); cudaFree(c->any_frac);
  cudaFree(c->v_rays); cudaFree(c->v_img[0]); cudaFree(c->v_img[1]); cudaFree(c->box_table);
  if (c->copy_in) cudaStreamDestroy(c->copy_in);
  if (c->copy_out) cudaStreamDestroy(c->copy_out);
  for (cudaEvent_t e : c->ev_pool) cudaEventDestroy(e);
  if (c->prof_counts) cudaFreeHost(c->prof_counts);
  delete c;
}

int stnerf_set_precision(stnerf_handle c, int precision) {
  if (!c || precision < 0 || precision > STNERF_PREC_TC_3XF16_CF) return STNERF_EINVAL;
  c->precision = precision;
  return STNERF_OK;
}

int stnerf_reserve(stnerf_handle c, int n1, int n2) {
  if (!c || n1 < 3 || n1 > STNERF_MAX_N1 || n2 < 0 || n1 + n2 > STNERF_MAX_S) return STNERF_EINVAL;
  return ensure_ws(c, n1, n1 + n2);
}
size_t stnerf_workspace_bytes(stnerf_handle c) { return c ? c->ws_bytes : 0; }

// fp32 (SIMT) device image of a SpaceNet: [w_i^T | b_i] x 7, w_sigma, w_rgbh^T, b_rgbh, w_rgbo; the scalar biases live in SpaceNetW
static size_t bind_spacenet(SpaceNetDev& N, bool use_time) {
  const int krgb = HID + PE_DIR + (use_time ? PE_TIME : 0);
  const int Ks[7] = {PE_POS, HID, HID, HID, HID + PE_POS, HID, HID};
  size_t cur = 0;
  for (int i = 0; i < 7; ++i) {
    N.w.w[i] = N.blob + cur; cur += (size_t)HID * Ks[i];
    N.w.b[i] = N.blob + cur; cur += HID;
  }
  N.w.w_sigma = N.blob + cur; cur += HID;
  N.w.w_rgbh = N.blob + cur; cur += (size_t)HEAD * krgb;
  N.w.b_rgbh = N.blob + cur; cur += HEAD;
  N.w.w_rgbo = N.blob + cur; cur += 3 * HEAD;
  N.w.use_time = use_time ? 1 : 0;
  return cur;
}
static size_t bind_motionnet(MotionNetDev& N) {
  size_t cur = 0;
  for (int i = 0; i < 5; ++i) {
    const int K = i == 0 ? PE_MOTION : HEAD;
    N.w.w[i] = N.blob + cur; cur += (size_t)HEAD * K;
    N.w.b[i] = N.blob + cur; cur += HEAD;
  }
  N.w.w_out = N.blob + cur; cur += 3 * HEAD;
  return cur;
}

// Install a network's SIMT image and scalar biases on the context.  The caller adds the tensor-core weights, then marks it loaded.
static int install_spacenet(SpaceNetDev& N, const std::vector<float>& simt, bool use_time, float b_sigma, const float* b_rgbo) {
  N.loaded = false;
  const int rc = upload(&N.blob, simt);
  if (rc) return rc;
  if (bind_spacenet(N, use_time) != simt.size()) return STNERF_EINVAL;
  N.w.b_sigma = b_sigma;
  for (int a = 0; a < 3; ++a) N.w.b_rgbo[a] = b_rgbo[a];
  return STNERF_OK;
}
static int install_motionnet(MotionNetDev& N, const std::vector<float>& simt, const float* b_out) {
  N.loaded = false;
  const int rc = upload(&N.blob, simt);
  if (rc) return rc;
  if (bind_motionnet(N) != simt.size()) return STNERF_EINVAL;
  for (int a = 0; a < 3; ++a) N.w.b_out[a] = b_out[a];
  return STNERF_OK;
}

int stnerf_load_spacenet(stnerf_handle c, int layer, int fine, const float* blob, size_t n) {
  if (!c || !blob || layer < 0 || layer >= c->l || (fine != 0 && fine != 1)) return STNERF_EINVAL;
  const bool use_time = (n == (size_t)SPACENET_FLOATS_TIME);
  if (!use_time && n != (size_t)SPACENET_FLOATS_NOTIME) return STNERF_EINVAL;
  if ((c->desc.space_time[layer] != 0) != use_time) return STNERF_EINVAL;
  const int krgb = HID + PE_DIR + (use_time ? PE_TIME : 0);
  // walk the blob in state_dict order
  const float* p = blob;
  std::vector<float> host;
  const int Ks[7] = {PE_POS, HID, HID, HID, HID + PE_POS, HID, HID};
  for (int i = 0; i < 7; ++i) {
    transpose_into(host, p, HID, Ks[i]);
    p += (size_t)HID * Ks[i];
    host.insert(host.end(), p, p + HID);
    p += HID;
  }
  host.insert(host.end(), p, p + HID); p += HID;
  const float b_sigma = *p++;
  transpose_into(host, p, HEAD, krgb); p += (size_t)HEAD * krgb;
  host.insert(host.end(), p, p + HEAD); p += HEAD;
  host.insert(host.end(), p, p + 3 * HEAD); p += 3 * HEAD;
  SpaceNetDev& N = c->space[fine][layer];
  int rc = install_spacenet(N, host, use_time, b_sigma, p);
  if (rc) return rc;
  rc = tc_pack_spacenet(N.tc, blob, use_time);
  if (rc) return rc;
  N.loaded = true;
  return STNERF_OK;
}

int stnerf_load_motionnet(stnerf_handle c, int layer, const float* blob, size_t n) {
  if (!c || !blob || layer < 1 || layer >= c->l || n != (size_t)MOTIONNET_FLOATS) return STNERF_EINVAL;
  const float* p = blob;
  std::vector<float> host;
  for (int i = 0; i < 5; ++i) {
    const int K = i == 0 ? PE_MOTION : HEAD;
    transpose_into(host, p, HEAD, K); p += (size_t)HEAD * K;
    host.insert(host.end(), p, p + HEAD); p += HEAD;
  }
  host.insert(host.end(), p, p + 3 * HEAD); p += 3 * HEAD;
  MotionNetDev& N = c->motion[layer];
  int rc = install_motionnet(N, host, p);
  if (rc) return rc;
  rc = tc_pack_motionnet(N.tc, blob);
  if (rc) return rc;
  N.loaded = true;
  return STNERF_OK;
}

// ---- packed-weight image (SURVEY 8f row 3): every loaded network's device buffers, as they are, behind a small header ----
namespace {
constexpr char PACK_MAGIC[8] = {'S', 'T', 'N', 'B', '2', '0', '0', 'W'};
constexpr uint32_t PACK_VERSION = 4;      // 4: weight stream = (hi, lo) stage per 32-k sub-chunk, each stage stored once
struct PackHeader { char magic[8]; uint32_t version, n_layers, n_records, reserved; };
struct PackRec { uint32_t kind, fine, layer, use_time; uint64_t simt_floats, stream_bytes, aux_floats, tail_floats; float scalars[4]; uint32_t pad[4]; };
static size_t rec_payload(const PackRec& r) { return r.simt_floats * 4 + r.stream_bytes + r.aux_floats * 4 + r.tail_floats * 4; }
static size_t simt_floats_space(bool use_time) { return (size_t)(use_time ? SPACENET_FLOATS_TIME : SPACENET_FLOATS_NOTIME) - 4; }
static size_t simt_floats_motion() { return (size_t)MOTIONNET_FLOATS - 3; }
}  // namespace

int stnerf_weights_export(stnerf_handle c, void* buf, size_t capacity, size_t* bytes_needed) {
  if (!c) return STNERF_EINVAL;
  std::vector<PackRec> recs;
  for (int f = 0; f < 2; ++f)
    for (int i = 0; i < c->l; ++i)
      if (c->space[f][i].loaded) {
        const SpaceNetDev& N = c->space[f][i];
        PackRec r{};
        r.kind = 0; r.fine = (uint32_t)f; r.layer = (uint32_t)i; r.use_time = (uint32_t)N.w.use_time;
        r.simt_floats = simt_floats_space(N.w.use_time != 0); r.stream_bytes = tc_stream_bytes(true);
        r.aux_floats = tc_aux_floats(); r.tail_floats = tc_tail_floats(true);
        r.scalars[0] = N.w.b_sigma; for (int a = 0; a < 3; ++a) r.scalars[1 + a] = N.w.b_rgbo[a];
        recs.push_back(r);
      }
  for (int i = 1; i < c->l; ++i)
    if (c->motion[i].loaded) {
      PackRec r{};
      r.kind = 1; r.layer = (uint32_t)i;
      r.simt_floats = simt_floats_motion(); r.stream_bytes = tc_stream_bytes(false);
      r.aux_floats = tc_aux_floats(); r.tail_floats = 0;
      for (int a = 0; a < 3; ++a) r.scalars[a] = c->motion[i].w.b_out[a];
      recs.push_back(r);
    }
  if (recs.empty()) return STNERF_ENOWEIGHTS;
  size_t need = sizeof(PackHeader);
  for (const PackRec& r : recs) need += sizeof(PackRec) + rec_payload(r);
  if (bytes_needed) *bytes_needed = need;
  if (!buf) return STNERF_OK;                         // size query
  if (capacity < need) return STNERF_EINVAL;
  uint8_t* p = static_cast<uint8_t*>(buf);
  PackHeader h{};
  memcpy(h.magic, PACK_MAGIC, 8); h.version = PACK_VERSION; h.n_layers = (uint32_t)c->l; h.n_records = (uint32_t)recs.size();
  memcpy(p, &h, sizeof(h)); p += sizeof(h);
  for (const PackRec& r : recs) {
    memcpy(p, &r, sizeof(r)); p += sizeof(r);
    float* simt = reinterpret_cast<float*>(p);
    uint8_t* stream = p + r.simt_floats * 4;
    float* aux = reinterpret_cast<float*>(stream + r.stream_bytes);
    float* tail = aux + r.aux_floats;
    const float* dev = r.kind == 0 ? c->space[r.fine][r.layer].blob : c->motion[r.layer].blob;
    const TcNet& tc = r.kind == 0 ? c->space[r.fine][r.layer].tc : c->motion[r.layer].tc;
    STNERF_CUDA(cudaMemcpy(simt, dev, r.simt_floats * 4, cudaMemcpyDeviceToHost));
    const int rc = tc_export(tc, r.kind == 0, stream, aux, tail);
    if (rc) return rc;
    p += rec_payload(r);
  }
  return STNERF_OK;
}

int stnerf_weights_import(stnerf_handle c, const void* buf, size_t bytes) {
  if (!c || !buf || bytes < sizeof(PackHeader)) return STNERF_EINVAL;
  const uint8_t* p = static_cast<const uint8_t*>(buf);
  const uint8_t* end = p + bytes;
  PackHeader h;
  memcpy(&h, p, sizeof(h)); p += sizeof(h);
  if (memcmp(h.magic, PACK_MAGIC, 8) != 0 || h.version != PACK_VERSION || (int)h.n_layers != c->l) return STNERF_EINVAL;
  // validate every record against this context before touching any network
  const uint8_t* q = p;
  for (uint32_t k = 0; k < h.n_records; ++k) {
    if ((size_t)(end - q) < sizeof(PackRec)) return STNERF_EINVAL;
    PackRec r;
    memcpy(&r, q, sizeof(r)); q += sizeof(r);
    if (r.kind > 1 || r.fine > 1 || (int)r.layer >= c->l || r.aux_floats != tc_aux_floats()) return STNERF_EINVAL;
    if (r.kind == 0) {
      if ((c->desc.space_time[r.layer] != 0) != (r.use_time != 0)) return STNERF_EINVAL;
      if (r.simt_floats != simt_floats_space(r.use_time != 0) || r.stream_bytes != tc_stream_bytes(true) ||
          r.tail_floats != tc_tail_floats(true)) return STNERF_EINVAL;
    } else {
      if (r.layer < 1 || r.simt_floats != simt_floats_motion() || r.stream_bytes != tc_stream_bytes(false) || r.tail_floats != 0)
        return STNERF_EINVAL;
    }
    if ((size_t)(end - q) < rec_payload(r)) return STNERF_EINVAL;
    q += rec_payload(r);
  }
  if (q != end) return STNERF_EINVAL;
  for (uint32_t k = 0; k < h.n_records; ++k) {
    PackRec r;
    memcpy(&r, p, sizeof(r)); p += sizeof(r);
    const float* simt = reinterpret_cast<const float*>(p);
    const uint8_t* stream = p + r.simt_floats * 4;
    const float* aux = reinterpret_cast<const float*>(stream + r.stream_bytes);
    const float* tail = aux + r.aux_floats;
    const std::vector<float> host(simt, simt + r.simt_floats);
    if (r.kind == 0) {
      SpaceNetDev& N = c->space[r.fine][r.layer];
      int rc = install_spacenet(N, host, r.use_time != 0, r.scalars[0], r.scalars + 1);
      if (rc) return rc;
      rc = tc_import(N.tc, true, (int)r.use_time, stream, aux, tail);
      if (rc) return rc;
      N.loaded = true;
    } else {
      MotionNetDev& N = c->motion[r.layer];
      int rc = install_motionnet(N, host, r.scalars);
      if (rc) return rc;
      rc = tc_import(N.tc, false, 0, stream, aux, nullptr);
      if (rc) return rc;
      N.loaded = true;
    }
    p += rec_payload(r);
  }
  return STNERF_OK;
}

// the scene constants of `l` layers as the kernels read them
static void dev_scene_from(const stnerf_scene& s, int l, DevScene& d) {
  memset(&d, 0, sizeof(d));
  for (int i = 0; i < l; ++i) {
    for (int a = 0; a < 3; ++a) { d.bmin[i][a] = s.bmin[i][a]; d.bmax[i][a] = s.bmax[i][a]; }
    d.shown[i] = s.shown[i];
  }
  d.near_plane = s.near_plane; d.alpha2 = s.alpha_layer2;
  d.thr_layer = s.density_threshold; d.thr_bkgd = s.bkgd_density_threshold;
  d.boarder = s.boarder_weight; d.apply_thr = s.apply_thresholds; d.n_layers = l;
  d.fid_shared = s.shared_frame_id;
}

int stnerf_set_scene(stnerf_handle c, const stnerf_scene* s) {
  if (!c || !s) return STNERF_EINVAL;
  c->scene = *s;
  dev_scene_from(*s, c->l, c->dscene);
  for (int i = 0; i < c->l; ++i)
    if ((s->scale_coarse_on[i] || s->scale_fine_on[i]) && s->scale[i] == 0.0f) return STNERF_EINVAL;
  c->have_scene = true;
  return STNERF_OK;
}

}  // extern "C"

// Layer i's rotation for the scene in effect, or false.  `sampled`: a render / training path, where a hidden performer is sampled
// unrotated (it draws nothing, and this keeps its samples -- which still take part in the resampling -- those of an unrotated layer).
static bool layer_rot(const stnerf_ctx* c, int i, bool sampled, RayRot& r) {
  const int mode = c->rot_mode[i];
  if (mode == STNERF_ROT_OFF || (sampled && i > 0 && !c->scene.shown[i])) return false;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) r.Rt[3 * a + b] = c->rot_R[i][3 * b + a];
  for (int a = 0; a < 3; ++a)
    r.c[a] = mode == STNERF_ROT_BOX ? (c->scene.bmin[i][a] + c->scene.bmax[i][a]) * 0.5f : c->rot_c[i][a];
  return true;
}

// The rotated layers of a render or training call: their rotations and one (rays, ray_stride) copy each, in stream-ordered
// scratch sized for `cap` rays.  layer_rays() points every other layer at the caller's rays.
struct RotatedRays {
  int n = 0, layer[STNERF_MAX_LAYERS];
  RayRot rot[STNERF_MAX_LAYERS];
  float* buf = nullptr;
  long long cap = 0;
  int stride = 0;
  cudaStream_t st = nullptr;
  int init(const stnerf_ctx* c, long long cap_rays, int ray_stride, cudaStream_t s, int only_layer = -1) {
    st = s; cap = cap_rays; stride = ray_stride;
    for (int i = 0; i < c->l; ++i)
      if ((only_layer < 0 || i == only_layer) && layer_rot(c, i, true, rot[n])) layer[n++] = i;
    if (n > 0 && cap > 0) STNERF_CUDA(cudaMallocAsync((void**)&buf, (size_t)n * cap * stride * sizeof(float), st));
    return STNERF_OK;
  }
  // rotate rays [0, m) (m <= cap) into every copy; lr = where each layer's rays are
  int rotate(const float* rays, long long m, LayerRays& lr) {
    for (int i = 0; i < STNERF_MAX_LAYERS; ++i) lr.p[i] = rays;
    for (int k = 0; k < n; ++k) {
      float* dst = buf + (size_t)k * cap * stride;
      const int rc = launch_rotate_rays(rays, m, stride, rot[k], dst, st);
      if (rc) return rc;
      lr.p[layer[k]] = dst;
    }
    return STNERF_OK;
  }
  ~RotatedRays() { if (buf) cudaFreeAsync(buf, st); }
};

// ---------------------------------------------------------------------------------------------------------
// one pass of the networks over a chunk
// ---------------------------------------------------------------------------------------------------------
// The inverse edit of one layer and pass (common.cuh: inverse_edit) into a PointSrc or a FieldEdit.
template <class E>
static void fill_edit(E& e, const stnerf_scene& sc, int layer, bool fine) {
  e.shift_on = sc.shift_on[layer];
  e.scale_on = fine ? sc.scale_fine_on[layer] : sc.scale_coarse_on[layer];
  for (int a = 0; a < 3; ++a) { e.shift[a] = sc.shift[layer][a]; e.pivot[a] = sc.pivot[a]; }
  e.scale = e.scale_on ? sc.scale[layer] : 1.0f;
}

// n points given one by one: pos (n, pos_stride), dirs (n,3) or null, times (n, time_stride) or null.
static PointSrc explicit_src(const float* pos, int pos_stride, const float* dirs, const float* times, int time_stride, long long n) {
  PointSrc s;
  memset(&s, 0, sizeof(s));
  s.mode = SRC_EXPLICIT; s.pos = pos; s.pos_stride = pos_stride; s.dirs = dirs; s.times = times; s.time_stride = time_stride;
  s.n_slots = n; s.S = 1; s.scale = 1.f;
  return s;
}

// Layer `layer`'s samples at depths t (ray, S) along `rays`, with the inverse edit of the pass; the caller adds which rays
// (hit, count, slots).
static PointSrc march_src(const stnerf_ctx* c, int layer, bool fine, const float* rays, int ray_stride, const float* t, int S) {
  PointSrc s;
  memset(&s, 0, sizeof(s));
  s.mode = SRC_MARCH;
  s.rays = rays; s.ray_stride = ray_stride; s.t = t; s.S = S;
  s.layer = c->scene.shared_frame_id ? 0 : layer;             // frame-id column offset of this layer
  fill_edit(s, c->scene, layer, fine);
  return s;
}

// The context has a scene (unless the call reads none) and is on its own device, where its weights and workspace live.
static int ctx_ready(const stnerf_ctx* c, bool need_scene = true) {
  if (need_scene && !c->have_scene) return STNERF_EINVAL;
  int cur = -1;
  STNERF_CUDA(cudaGetDevice(&cur));
  return cur == c->device ? STNERF_OK : STNERF_EINVAL;
}

// Rays carry o, d and a frame-id column per layer, or one shared column (the reference prints + exit(-1) otherwise, :162-163).
static bool ray_stride_ok(const stnerf_ctx* c, int ray_stride) {
  return ray_stride >= 6 + (c->scene.shared_frame_id ? 1 : c->l);
}

static int run_spacenet(stnerf_ctx* c, const PointSrc& src, SpaceNetDev& net, float* raw, float* rgb, float* sigma,
                        cudaStream_t st, int count_slot = -1, const FuseCoarse* fuse = nullptr, bool fine_pass = false) {
  if (!net.loaded) return STNERF_ENOWEIGHTS;
  ProfScope ps(c, 0, (double)src.n_slots * src.S, count_slot, src.S, st);
  if (c->precision == STNERF_PREC_FP32_SIMT)
    return launch_spacenet_simt(src, net.w, raw, 0, rgb, sigma, c->num_sms, st);
  if (src.mode == SRC_EXPLICIT) {      // unit entry point: one bias row per point, stream-ordered scratch
    float* cb = nullptr;
    STNERF_CUDA(cudaMallocAsync((void**)&cb, (size_t)std::max<long long>(src.n_slots, 1) * 128 * sizeof(float), st));
    const int rc = tc_launch_spacenet(src, net.tc, c->precision, cb, raw, rgb, sigma, c->num_sms, st, nullptr, fine_pass);
    STNERF_CUDA(cudaFreeAsync(cb, st));
    return rc;
  }
  return tc_launch_spacenet(src, net.tc, c->precision, c->cbuf, raw, rgb, sigma, c->num_sms, st, fuse, fine_pass);
}
static int run_motionnet(stnerf_ctx* c, const PointSrc& src, MotionNetDev& net, const int* lerp_flag, int lerp_force,
                         float* xyz_out, float* flow_out, cudaStream_t st, int count_slot = -1) {
  if (!net.loaded) return STNERF_ENOWEIGHTS;
  ProfScope ps(c, 1, (double)src.n_slots * src.S, count_slot, src.S, st);
  if (c->precision == STNERF_PREC_FP32_SIMT)
    return launch_motionnet_simt(src, net.w, lerp_flag, lerp_force, xyz_out, flow_out, c->num_sms, st);
  return tc_launch_motionnet(src, net.tc, c->precision, lerp_flag, lerp_force, xyz_out, flow_out, c->num_sms, st);
}

// `fuse` (coarse pass only): template of the per-layer fusion request (everything but the layer-specific fields), or null.
// `want_raw`: the (rgb, sigma) samples must reach HBM (a later kernel composites them); false only with `fuse`.
// `reuse_n1` > 0 (fine pass): the MotionNet runs on the S - reuse_n1 NEW depths only; the flow of the coarse depths is the coarse
// pass' (xyz_coarse), stitched together through the origin map the merge wrote (z_new / src_map).
static int run_nets(stnerf_ctx* c, const LayerRays& rays, long long n, int ray_stride, bool fine, int S, cudaStream_t st,
                    int chunk_slot, const FuseCoarse* fuse = nullptr, bool want_raw = true, float* coarse_imgs = nullptr,
                    long long plane = 0, int reuse_n1 = 0) {
  const long long R = c->chunk_rays;
  const float* tbuf = fine ? c->t_fine : c->t_coarse;
  float* rawbuf = fine ? c->raw_fine : c->raw_coarse;
  const long long tl = R * (fine ? c->cap_s2 : c->cap_n1);      // layer strides of the workspace arrays
  for (int i = 0; i < c->l; ++i) {
    if (i > 0 && !c->scene.shown[i]) continue;                  // hidden performers: sigma = rgb = 0 (:401, :556)
    PointSrc s = march_src(c, i, fine, rays.p[i], ray_stride, tbuf + i * tl, S);   // a rotated layer marches along its own rays
    float* raw = want_raw ? rawbuf + (size_t)i * tl * 4 : nullptr;
    FuseCoarse f;
    memset(&f, 0, sizeof(f));
    if (fuse) {
      f = *fuse;
      f.on = 1; f.layer = i;
      f.t_fine = c->t_fine + (size_t)i * R * c->cap_s2;
      f.z_new = fuse->z_new ? c->z_new + (size_t)i * R * c->cap_s2 : nullptr;
      f.src_map = fuse->z_new ? c->src_map + (size_t)i * R * c->cap_s2 : nullptr;
      f.u = fuse->u ? fuse->u + (size_t)i * fuse->n_total * fuse->n2 : nullptr;     // [layer][ray of the call][n2], chunk offset applied by the caller
      f.img = coarse_imgs ? coarse_imgs + (size_t)(1 + i) * plane : nullptr;
    }
    int rc;
    if (i == 0) {
      s.hit = nullptr; s.count = nullptr; s.n_slots = n;
      rc = run_spacenet(c, s, c->space[fine ? 1 : 0][0], raw, nullptr, nullptr, st, -1, fuse ? &f : nullptr, fine);
      if (rc) return rc;
      continue;
    }
    s.hit = c->hit + (size_t)i * R;
    s.count = c->counts + i;
    s.n_slots_cap = n;
    // the coarse pass keeps every performer's deformed points (the fine pass may reuse them); the fine pass has one scratch
    float* xyz_out = fine ? c->xyz : c->xyz_coarse + (size_t)i * R * c->cap_n1 * 3;
    // reuse needs the same inverse edit in both passes (a None shift entry skips the fine-pass scale only, layered_rfrender.py:468-469)
    const bool reuse = fine && reuse_n1 > 0 && c->scene.scale_fine_on[i] == c->scene.scale_coarse_on[i];
    if (reuse) {
      PointSrc m = s;                                            // MotionNet on the n2 new depths of every hit ray
      m.t = c->z_new + (size_t)i * R * c->cap_s2;
      m.S = S - reuse_n1;
      rc = run_motionnet(c, m, c->motion[i], c->lerp_flags + i, -1, xyz_out, nullptr, st, chunk_slot >= 0 ? chunk_slot * 8 + i : -1);
      if (rc) return rc;
      s.mode = SRC_XYZ_MAP;
      s.pos = c->xyz_coarse + (size_t)i * R * c->cap_n1 * 3;
      s.pos2 = xyz_out;
      s.src_map = c->src_map + (size_t)i * R * c->cap_s2;
      s.n_first = reuse_n1;
      rc = run_spacenet(c, s, c->space[1][i], raw, nullptr, nullptr, st, chunk_slot >= 0 ? chunk_slot * 8 + i : -1, nullptr, true);
      if (rc) return rc;
      continue;
    }
    rc = run_motionnet(c, s, c->motion[i], c->lerp_flags + i, -1, xyz_out, nullptr, st, chunk_slot >= 0 ? chunk_slot * 8 + i : -1);
    if (rc) return rc;
    s.mode = SRC_XYZ;
    s.pos = xyz_out;
    rc = run_spacenet(c, s, c->space[fine ? 1 : 0][i], raw, nullptr, nullptr, st, chunk_slot >= 0 ? chunk_slot * 8 + i : -1,
                      fuse ? &f : nullptr, fine);
    if (rc) return rc;
  }
  return STNERF_OK;
}

// Where the images of a call go.  `coarse` / `fine`: [l+1 images][5*n_total floats] each (image 0 mixed, 1+i layer i), or null =
// that pass writes no images (the coarse pass then only resamples: its merged composite is skipped altogether).
struct OutSpec {
  float* coarse;
  float* fine;
  int pixels;            // 0: image = rgb (N,3) | depth (N) | acc (N) planes;  1: image = (N,5) pixel-interleaved
};

// Called after the last kernel of a chunk has been enqueued (pipelined host copies hang their events here).
struct ChunkHook {
  int (*fn)(void* user, long long c0, long long n, cudaStream_t st);
  void* user;
};

static int render_core(stnerf_ctx* c, const float* rays, long long n_rays, int ray_stride, int n1, int n2, int only_coarse,
                       const float* jitter, const float* u, uint64_t seed, OutSpec out, uint8_t* ray_mask, cudaStream_t st,
                       const ChunkHook* before_chunk = nullptr, const ChunkHook* after_chunk = nullptr,
                       bool lerp_per_call = true) {
  if (!c || !rays || n_rays < 0) return STNERF_EINVAL;
  int rc = ctx_ready(c);
  if (rc) return rc;
  if (!ray_stride_ok(c, ray_stride)) return STNERF_EINVAL;
  if (n1 < 3 || n1 > STNERF_MAX_N1) return STNERF_EINVAL;
  if (only_coarse) n2 = 0;
  if (n2 < 0 || n1 + n2 > STNERF_MAX_S) return STNERF_EINVAL;
  if (n2 == 0 && !out.coarse) return STNERF_EINVAL;
  if (n2 > 0 && !out.fine) return STNERF_EINVAL;
  rc = ensure_ws(c, n1, n1 + n2);
  if (rc) return rc;
  const int l = c->l, S2 = n1 + n2;
  const long long R = c->chunk_rays, N = n_rays;
  RotatedRays rot;
  rc = rot.init(c, std::min(R, N), ray_stride, st);
  if (rc) return rc;
  // the coarse sampling of rays [c0, c0 + n): depths, masks, hit lists, counts and lerp flags; lr = where each layer's rays are
  LayerRays lr;
  auto sample = [&](long long c0, long long n, uint8_t* mask, long long mask_ls) -> int {
    const float* rch = rays + c0 * ray_stride;
    const int rc = rot.rotate(rch, n, lr);
    if (rc) return rc;
    return launch_sample(rch, n, ray_stride, c->dscene, l, n1, jitter ? jitter + c0 * n1 : nullptr, N * n1, seed, c0, c->idmap,
                         c->t_coarse, R * c->cap_n1, mask, mask_ls, c->hit, R, c->counts, c->lerp_flags, st, c->box_table,
                         c->box_frames, &lr);
  };
  // MotionNet's lerp (motion_net.py:53) is decided once per call, over every hit ray of the call.  With more than one chunk, a
  // sampling pass over all chunks sets the flags first (the chunk loop overwrites its depths, masks and hit lists).  Rays that
  // share their frame-id columns (render_one_view) give every chunk the call's decision, so they skip it.
  STNERF_CUDA(cudaMemsetAsync(c->lerp_flags, 0, STNERF_MAX_LAYERS * 4, st));
  for (long long c0 = 0; lerp_per_call && N > R && c0 < N; c0 += R) {
    const long long n = std::min(R, N - c0);
    if (before_chunk) { rc = before_chunk->fn(before_chunk->user, c0, n, st); if (rc) return rc; }
    STNERF_CUDA(cudaMemsetAsync(c->counts, 0, STNERF_MAX_LAYERS * 4, st));
    rc = sample(c0, n, c->mask_ws, R);
    if (rc) return rc;
  }
  for (long long c0 = 0; c0 < N; c0 += R) {
    const long long n = std::min(R, N - c0);
    if (before_chunk) { rc = before_chunk->fn(before_chunk->user, c0, n, st); if (rc) return rc; }
    c->last_chunk_rays = n; c->last_n1 = n1; c->last_s2 = n2 > 0 ? S2 : 0;
    STNERF_CUDA(cudaMemsetAsync(c->counts, 0, STNERF_MAX_LAYERS * 4, st));
    uint8_t* mask = ray_mask ? ray_mask + c0 : c->mask_ws;
    const long long mask_ls = ray_mask ? N : R;
    int chunk_slot = -1;
    {
      ProfScope ps(c, 2, (double)n, -1, 1, st);
      rc = sample(c0, n, mask, mask_ls);
      if (rc) return rc;
    }
    if (c->prof_on && c->prof_counts && c->prof_chunks < PROF_MAX_CHUNKS) {
      chunk_slot = c->prof_chunks++;
      STNERF_CUDA(cudaMemcpyAsync(c->prof_counts + chunk_slot * 8, c->counts, 32, cudaMemcpyDeviceToHost, st));
    }
    // NOTE: the workspace t arrays are laid out with the *capacity* sample counts as layer stride but the
    // per-ray stride is the live n1 / S2, so a ray's samples stay contiguous.
    // Coarse-pass fusion: with a tensor-core mode and n1 = 64 the SpaceNet kernel composites and resamples every shown layer in
    // its spare warps (mlp_tc.cuh: FuseCoarse).  The stand-alone kernel is then only needed for the merged coarse image (when
    // coarse images are wanted), for the zero pixels of missed rays, and for the resampling of hit-but-hidden layers.
    const bool fuse = n2 > 0 && c->precision != STNERF_PREC_FP32_SIMT && tc_can_fuse_coarse(n1, n2) && !c->no_fuse;
    unsigned fused_layers = 0;
    bool hidden_any = false;
    for (int i = 0; i < l; ++i) {
      if (i == 0 || c->scene.shown[i]) fused_layers |= fuse ? (1u << i) : 0u;
      else hidden_any = true;
    }
    // Flow reuse: the merge (fused or stand-alone register path) also writes the new depths and the origin of every fine depth, so
    // the fine pass runs the MotionNet on the n2 new depths only (same network, same points for the other n1: SURVEY A.6).
    const bool reuse = n2 > 0 && c->precision != STNERF_PREC_FP32_SIMT && n1 <= 128 && n2 <= 256 && S2 <= 256 && !c->no_reuse;
    c->last_reuse = reuse;
    FuseCoarse ft;
    memset(&ft, 0, sizeof(ft));
    if (fuse) {
      ft.z_new = reuse ? c->z_new : nullptr;
      ft.n1 = n1; ft.n2 = n2; ft.u = u ? u + c0 * n2 : nullptr; ft.seed = seed; ft.idmap = c->idmap; ft.ray_base = c0;
      ft.n_total = N; ft.pixels = out.pixels; ft.mask = pass_mask(c->dscene); ft.boarder = c->dscene.boarder;
    }
    rc = run_nets(c, lr, n, ray_stride, false, n1, st, chunk_slot, fuse ? &ft : nullptr, /*want_raw=*/!fuse || out.coarse != nullptr,
                  out.coarse, 5 * N);
    if (rc) return rc;
    CompositeArgs a;
    memset(&a, 0, sizeof(a));
    a.skip_layers = fused_layers;
    a.t = c->t_coarse; a.t_layer_stride = R * c->cap_n1;
    a.raw = c->raw_coarse; a.raw_layer_stride = R * c->cap_n1 * 4;
    a.mask = mask; a.mask_layer_stride = mask_ls;
    a.u = u ? u + c0 * n2 : nullptr; a.u_layer_stride = N * n2;
    a.t_fine = c->t_fine; a.tf_layer_stride = R * c->cap_s2;
    if (reuse) { a.z_new = c->z_new; a.zn_layer_stride = R * c->cap_s2; a.src_map = c->src_map; a.sm_layer_stride = R * c->cap_s2; }
    a.out = out.coarse; a.pixel_layout = out.pixels; a.n_total = N; a.ray_base = c0; a.n = n;
    a.S = n1; a.n2 = n2; a.fine = 0; a.seed = seed; a.idmap = c->idmap;
    if (!fuse || out.coarse != nullptr || hidden_any) {
      ProfScope ps(c, 3, (double)n, -1, 1, st);
      rc = launch_composite_pass(a, c->dscene, l, st);
      if (rc) return rc;
    }
    if (n2 > 0) {
      rc = run_nets(c, lr, n, ray_stride, true, S2, st, chunk_slot, nullptr, true, nullptr, 0, reuse ? n1 : 0);
      if (rc) return rc;
      a.t = c->t_fine; a.t_layer_stride = R * c->cap_s2;
      a.raw = c->raw_fine; a.raw_layer_stride = R * c->cap_s2 * 4;
      a.u = nullptr; a.t_fine = nullptr;
      a.out = out.fine;
      a.S = S2; a.n2 = 0; a.fine = 1; a.skip_layers = 0;
      ProfScope ps(c, 3, (double)n, -1, 1, st);
      rc = launch_composite_pass(a, c->dscene, l, st);
      if (rc) return rc;
    }
    if (after_chunk) { rc = after_chunk->fn(after_chunk->user, c0, n, st); if (rc) return rc; }
  }
  return STNERF_OK;
}

extern "C" {

int stnerf_render(stnerf_handle c, const float* rays, int64_t n_rays, int ray_stride, int n1, int n2, int only_coarse,
                  const float* jitter, const float* u, uint64_t seed, float* out, uint8_t* ray_mask, void* stream) {
  if (!c || !out) return STNERF_EINVAL;
  OutSpec o{out, out + (size_t)(c->l + 1) * 5 * (size_t)n_rays, 0};
  return render_core(c, rays, n_rays, ray_stride, n1, n2, only_coarse, jitter, u, seed, o, ray_mask, (cudaStream_t)stream);
}

static int grow(void** p, size_t* have, size_t want) {
  if (want <= *have) return STNERF_OK;
  if (*p) cudaFree(*p);
  *p = nullptr; *have = 0;
  if (cudaMalloc(p, want) != cudaSuccess) { cudaGetLastError(); return STNERF_ENOMEM; }
  *have = want;
  return STNERF_OK;
}

}  // extern "C"

// ---- host-buffer plumbing: copy streams, an event pool, per-chunk hooks ------------------------------------------------------
static int ensure_copy_streams(stnerf_ctx* c) {
  if (!c->copy_in) STNERF_CUDA(cudaStreamCreateWithFlags(&c->copy_in, cudaStreamNonBlocking));
  if (!c->copy_out) STNERF_CUDA(cudaStreamCreateWithFlags(&c->copy_out, cudaStreamNonBlocking));
  return STNERF_OK;
}
static int ensure_events(stnerf_ctx* c, size_t n) {
  while (c->ev_pool.size() < n) {
    cudaEvent_t e;
    STNERF_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    c->ev_pool.push_back(e);
  }
  return STNERF_OK;
}

namespace {
// stnerf_render_host: rays arrive chunk by chunk on `copy_in` while earlier chunks render; the image slices of a finished chunk
// leave on `copy_out` while later chunks render.
struct HostPipe {
  stnerf_ctx* c;
  long long N;
  int only_coarse;
  float* out_host;
  uint8_t* mask_host;
  size_t ev_in0, ev_out0;      // first event index of the per-chunk "rays landed" / "chunk rendered" events
};
int host_before_chunk(void* user, long long c0, long long, cudaStream_t st) {
  HostPipe* p = static_cast<HostPipe*>(user);
  const size_t k = (size_t)(c0 / p->c->chunk_rays);
  STNERF_CUDA(cudaStreamWaitEvent(st, p->c->ev_pool[p->ev_in0 + k], 0));
  return STNERF_OK;
}
int host_after_chunk(void* user, long long c0, long long n, cudaStream_t st) {
  HostPipe* p = static_cast<HostPipe*>(user);
  stnerf_ctx* c = p->c;
  const size_t k = (size_t)(c0 / c->chunk_rays);
  cudaEvent_t done = c->ev_pool[p->ev_out0 + k];
  STNERF_CUDA(cudaEventRecord(done, st));
  STNERF_CUDA(cudaStreamWaitEvent(c->copy_out, done, 0));
  const size_t N = (size_t)p->N, plane = 5 * N;
  const int n_img = (p->only_coarse ? 1 : 2) * (c->l + 1);
  for (int im = 0; im < n_img; ++im) {      // plane = rgb (N,3) | depth (N) | acc (N): three contiguous slices per chunk
    const float* src = c->h_out + (size_t)im * plane;
    float* dst = p->out_host + (size_t)im * plane;
    STNERF_CUDA(cudaMemcpyAsync(dst + 3 * (size_t)c0, src + 3 * (size_t)c0, (size_t)n * 12, cudaMemcpyDeviceToHost, c->copy_out));
    STNERF_CUDA(cudaMemcpyAsync(dst + 3 * N + c0, src + 3 * N + c0, (size_t)n * 4, cudaMemcpyDeviceToHost, c->copy_out));
    STNERF_CUDA(cudaMemcpyAsync(dst + 4 * N + c0, src + 4 * N + c0, (size_t)n * 4, cudaMemcpyDeviceToHost, c->copy_out));
  }
  if (p->mask_host)
    for (int i = 0; i < c->l; ++i)
      STNERF_CUDA(cudaMemcpyAsync(p->mask_host + (size_t)i * N + c0, c->h_mask + (size_t)i * N + c0, (size_t)n,
                                  cudaMemcpyDeviceToHost, c->copy_out));
  return STNERF_OK;
}
}  // namespace

extern "C" {

int stnerf_reserve_host(stnerf_handle c, int64_t max_rays, int ray_stride) {
  if (!c || max_rays <= 0 || ray_stride < 6) return STNERF_EINVAL;
  const size_t n = (size_t)max_rays;
  int rc = grow((void**)&c->h_rays, &c->h_rays_bytes, n * ray_stride * 4);
  rc |= grow((void**)&c->h_out, &c->h_out_bytes, (size_t)2 * (c->l + 1) * 5 * n * 4);
  rc |= grow((void**)&c->h_mask, &c->h_mask_bytes, (size_t)c->l * n);
  rc |= grow((void**)&c->v_rays, &c->v_rays_bytes, n * (6 + STNERF_MAX_LAYERS) * 4);
  for (int b = 0; b < 2; ++b) rc |= grow((void**)&c->v_img[b], &c->v_img_bytes[b], (size_t)(c->l + 1) * 5 * n * 4);
  if (rc) return STNERF_ENOMEM;
  rc = ensure_copy_streams(c);
  if (rc) return rc;
  return ensure_events(c, 2 * (size_t)((max_rays + c->chunk_rays - 1) / c->chunk_rays) + 8);
}

int stnerf_render_host(stnerf_handle c, const float* rays_host, int64_t n_rays, int ray_stride, int n1, int n2,
                       int only_coarse, uint64_t seed, float* out_host, uint8_t* ray_mask_host, void* stream) {
  if (!c || !rays_host || !out_host || n_rays <= 0) return STNERF_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t rb = (size_t)n_rays * ray_stride * 4, ob = (size_t)2 * (c->l + 1) * 5 * n_rays * 4,
               mb = (size_t)c->l * n_rays;
  if (only_coarse) n2 = 0;
  // staging: sized by stnerf_reserve_host; grown here only when a call exceeds every earlier size
  int rc = grow((void**)&c->h_rays, &c->h_rays_bytes, rb);
  rc |= grow((void**)&c->h_out, &c->h_out_bytes, ob);
  rc |= grow((void**)&c->h_mask, &c->h_mask_bytes, mb);
  if (rc) return STNERF_ENOMEM;
  rc = ensure_copy_streams(c);
  if (rc) return rc;
  const long long R = c->chunk_rays;
  const size_t n_chunks = (size_t)((n_rays + R - 1) / R);
  rc = ensure_events(c, 2 * n_chunks + 1);
  if (rc) return rc;
  // the copy-in stream starts after everything already queued on `st` (the staging buffers may still be read by it)
  cudaEvent_t start = c->ev_pool[2 * n_chunks];
  STNERF_CUDA(cudaEventRecord(start, st));
  STNERF_CUDA(cudaStreamWaitEvent(c->copy_in, start, 0));
  STNERF_CUDA(cudaStreamWaitEvent(c->copy_out, start, 0));
  for (size_t k = 0; k < n_chunks; ++k) {
    const long long c0 = (long long)k * R, n = std::min<long long>(R, n_rays - c0);
    STNERF_CUDA(cudaMemcpyAsync(c->h_rays + (size_t)c0 * ray_stride, rays_host + (size_t)c0 * ray_stride, (size_t)n * ray_stride * 4,
                                cudaMemcpyHostToDevice, c->copy_in));
    STNERF_CUDA(cudaEventRecord(c->ev_pool[k], c->copy_in));
  }
  HostPipe pipe{c, n_rays, n2 == 0 ? 1 : 0, out_host, ray_mask_host, 0, n_chunks};
  ChunkHook before{host_before_chunk, &pipe}, after{host_after_chunk, &pipe};
  OutSpec o{c->h_out, c->h_out + (size_t)(c->l + 1) * 5 * (size_t)n_rays, 0};
  rc = render_core(c, c->h_rays, n_rays, ray_stride, n1, n2, only_coarse, nullptr, nullptr, seed, o, c->h_mask, st, &before, &after);
  // drain both streams even on an error so no copy is left in flight into the caller's buffers
  cudaError_t e1 = cudaStreamSynchronize(c->copy_out), e2 = cudaStreamSynchronize(st), e3 = cudaStreamSynchronize(c->copy_in);
  if (rc) return rc;
  STNERF_CUDA(e1); STNERF_CUDA(e2); STNERF_CUDA(e3);
  return STNERF_OK;
}

// One view of stnerf_render_views: rays of the requested rows generated on the device, scene constants of THIS view, fine images
// written pixel-interleaved to `images` ([l+1][n_rows*W][5]).  Enqueue only.
static int render_one_view(stnerf_ctx* c, const stnerf_view* v, int H, int W, int row0, int row_step, int n_rows, int n1, int n2,
                           float* images, float* coarse_images, cudaStream_t st) {
  const long long n = (long long)n_rows * W;
  const int stride = 6 + c->l;
  int rc = stnerf_set_scene(c, &v->scene);
  if (rc) return rc;
  if (c->scene.shared_frame_id) return STNERF_EINVAL;          // views carry one frame id per layer (retiming rays)
  rc = launch_raygen(v->Kinv, v->T, H, W, row0, row_step, n_rows, v->frame_ids, c->l, c->v_rays, stride, st);
  if (rc) return rc;
  const RayIdMap keep = c->idmap;
  c->idmap = RayIdMap{(long long)row0 * W, (long long)row_step * W, W};       // every pixel keeps the draws of an unsharded render
  OutSpec o{coarse_images, images, 1};
  rc = render_core(c, c->v_rays, n, stride, n1, n2, 0, nullptr, nullptr, v->seed, o, nullptr, st, nullptr, nullptr,
                   /*lerp_per_call=*/false);
  c->idmap = keep;
  return rc;
}

int stnerf_render_views(stnerf_handle c, const stnerf_view* views_host, int n_views, int H, int W, int row0, int row_step,
                        int n_rows, int n1, int n2, float* images, float* coarse_images, int64_t view_stride, void* stream) {
  if (!c || !views_host || !images || n_views < 1 || H < 1 || W < 1 || row0 < 0 || row_step < 1 || n_rows < 1 || n2 < 1)
    return STNERF_EINVAL;
  if (row0 >= H || row0 + (long long)(n_rows - 1) * row_step >= H + row_step) return STNERF_EINVAL;   // at most one padding row
  const size_t n = (size_t)n_rows * W;
  if (view_stride < (int64_t)((size_t)(c->l + 1) * 5 * n)) return STNERF_EINVAL;
  if (grow((void**)&c->v_rays, &c->v_rays_bytes, n * (6 + c->l) * 4)) return STNERF_ENOMEM;
  for (int v = 0; v < n_views; ++v) {
    const int rc = render_one_view(c, views_host + v, H, W, row0, row_step, n_rows, n1, n2, images + (size_t)v * view_stride,
                                   coarse_images ? coarse_images + (size_t)v * view_stride : nullptr, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return STNERF_OK;
}

int stnerf_render_views_host(stnerf_handle c, const stnerf_view* views_host, int n_views, int H, int W, int n1, int n2,
                             float* images_host, void* stream) {
  if (!c || !views_host || !images_host || n_views < 1 || H < 1 || W < 1 || n2 < 1) return STNERF_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)H * W, img_floats = (size_t)(c->l + 1) * 5 * n;
  int rc = grow((void**)&c->v_rays, &c->v_rays_bytes, n * (6 + c->l) * 4);
  for (int b = 0; b < 2; ++b) rc |= grow((void**)&c->v_img[b], &c->v_img_bytes[b], img_floats * 4);
  if (rc) return STNERF_ENOMEM;
  rc = ensure_copy_streams(c);
  if (rc) return rc;
  rc = ensure_events(c, 4);
  if (rc) return rc;
  // events 0/1: "view rendered into buffer b";  2/3: "buffer b copied out"
  for (int v = 0; v < n_views && rc == STNERF_OK; ++v) {
    const int b = v & 1;
    if (v >= 2) STNERF_CUDA(cudaStreamWaitEvent(st, c->ev_pool[2 + b], 0));       // buffer b is free again
    rc = render_one_view(c, views_host + v, H, W, 0, 1, H, n1, n2, c->v_img[b], nullptr, st);
    if (rc) break;
    STNERF_CUDA(cudaEventRecord(c->ev_pool[b], st));
    STNERF_CUDA(cudaStreamWaitEvent(c->copy_out, c->ev_pool[b], 0));
    STNERF_CUDA(cudaMemcpyAsync(images_host + (size_t)v * img_floats, c->v_img[b], img_floats * 4, cudaMemcpyDeviceToHost, c->copy_out));
    STNERF_CUDA(cudaEventRecord(c->ev_pool[2 + b], c->copy_out));
  }
  cudaError_t e1 = cudaStreamSynchronize(c->copy_out), e2 = cudaStreamSynchronize(st);
  if (rc) return rc;
  STNERF_CUDA(e1); STNERF_CUDA(e2);
  return STNERF_OK;
}

int stnerf_debug_read_depths(stnerf_handle c, int what, int layer, void* dst, int64_t n_rays, int S, void* stream) {
  if (!c || !dst || layer < 0 || layer >= c->l || n_rays < 0 || what < 0 || what > 3) return STNERF_EINVAL;
  if (!c->t_coarse || n_rays > c->last_chunk_rays) return STNERF_EINVAL;
  if (what >= 2 && !c->last_reuse) return STNERF_EINVAL;
  const int n2 = c->last_s2 - c->last_n1;
  if (S != (what == 0 ? c->last_n1 : what == 2 ? n2 : c->last_s2)) return STNERF_EINVAL;
  const size_t R = (size_t)c->chunk_rays, fine_row = (size_t)layer * R * c->cap_s2;
  const void* src = what == 0   ? (const void*)(c->t_coarse + (size_t)layer * R * c->cap_n1)
                    : what == 1 ? (const void*)(c->t_fine + fine_row)
                    : what == 2 ? (const void*)(c->z_new + fine_row)
                                : (const void*)(c->src_map + fine_row);
  const size_t elem = what == 3 ? sizeof(uint8_t) : sizeof(float);
  STNERF_CUDA(cudaMemcpyAsync(dst, src, (size_t)n_rays * S * elem, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return STNERF_OK;
}

int stnerf_set_box_table(stnerf_handle c, const float* table_host, int n_frames) {
  if (!c || n_frames < 0 || (n_frames > 0 && !table_host)) return STNERF_EINVAL;
  STNERF_CUDA(cudaDeviceSynchronize());                  // a previous table may still be read by queued kernels
  cudaFree(c->box_table);
  c->box_table = nullptr; c->box_frames = 0;
  if (n_frames == 0) return STNERF_OK;
  const size_t bytes = (size_t)n_frames * c->l * 6 * sizeof(float);
  if (cudaMalloc((void**)&c->box_table, bytes) != cudaSuccess) { cudaGetLastError(); return STNERF_ENOMEM; }
  STNERF_CUDA(cudaMemcpy(c->box_table, table_host, bytes, cudaMemcpyHostToDevice));
  c->box_frames = n_frames;
  return STNERF_OK;
}

int stnerf_set_ray_ids(stnerf_handle c, int64_t base, int32_t width, int64_t row_stride) {
  if (!c || width < 0) return STNERF_EINVAL;
  c->idmap.base = base; c->idmap.width = width; c->idmap.row_stride = row_stride;
  return STNERF_OK;
}

int stnerf_set_rotation(stnerf_handle c, const int32_t* on_host, const float* R_host, const float* centre_host) {
  if (!c) return STNERF_EINVAL;
  int mode[STNERF_MAX_LAYERS] = {0};
  float R[STNERF_MAX_LAYERS][9] = {}, cen[STNERF_MAX_LAYERS][3] = {};
  if (on_host) {                                       // validate everything before changing anything
    for (int i = 0; i < c->l; ++i) {
      mode[i] = on_host[i];
      if (mode[i] < STNERF_ROT_OFF || mode[i] > STNERF_ROT_BOX) return STNERF_EINVAL;
      if (mode[i] == STNERF_ROT_OFF) continue;
      if (!R_host || (mode[i] == STNERF_ROT_CENTRE && !centre_host)) return STNERF_EINVAL;
      for (int k = 0; k < 9; ++k) {
        R[i][k] = R_host[9 * i + k];
        if (!isfinite(R[i][k])) return STNERF_EINVAL;
      }
      if (mode[i] == STNERF_ROT_CENTRE)
        for (int a = 0; a < 3; ++a) {
          cen[i][a] = centre_host[3 * i + a];
          if (!isfinite(cen[i][a])) return STNERF_EINVAL;
        }
    }
  }
  memcpy(c->rot_mode, mode, sizeof(mode));
  memcpy(c->rot_R, R, sizeof(R));
  memcpy(c->rot_c, cen, sizeof(cen));
  return STNERF_OK;
}

int stnerf_rotate_rays(const float* rays, int64_t n, int ray_stride, const float* R_host, const float* centre_host, float* out,
                       void* stream) {
  if (n < 0 || ray_stride < 6 || !R_host || !centre_host) return STNERF_EINVAL;
  if (n == 0) return STNERF_OK;
  if (!rays || !out) return STNERF_EINVAL;
  RayRot r;
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) r.Rt[3 * a + b] = R_host[3 * b + a];
    r.c[a] = centre_host[a];
  }
  return launch_rotate_rays(rays, n, ray_stride, r, out, (cudaStream_t)stream);
}

int stnerf_selftest_umma(float* max_err_host) {
  if (!max_err_host) return STNERF_EINVAL;
  return tc_selftest(max_err_host);
}

int stnerf_selftest_umma_accum(int reps, float* max_err_host, float* mean_signed_rel_err_host) {
  if (!max_err_host || !mean_signed_rel_err_host || reps < 1 || reps > 4096) return STNERF_EINVAL;
  return tc_selftest_accum(reps, max_err_host, mean_signed_rel_err_host);
}

int stnerf_profile_begin(stnerf_handle c) {
  if (!c) return STNERF_EINVAL;
  if (!c->prof_counts) STNERF_CUDA(cudaHostAlloc((void**)&c->prof_counts, (size_t)PROF_MAX_CHUNKS * 32, cudaHostAllocDefault));
  for (auto& r : c->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  c->prof.clear();
  c->prof_chunks = 0;
  c->prof_on = true;
  return STNERF_OK;
}

int stnerf_profile_end(stnerf_handle c, stnerf_profile* out) {
  if (!c || !out) return STNERF_EINVAL;
  c->prof_on = false;
  STNERF_CUDA(cudaDeviceSynchronize());
  memset(out, 0, sizeof(*out));
  for (auto& r : c->prof) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) out->ms[r.cls] += ms;
    out->launches[r.cls] += 1;
    out->points[r.cls] += r.count_slot >= 0 ? (double)c->prof_counts[r.count_slot] * r.S : r.points;
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  c->prof.clear();
  return STNERF_OK;
}

int stnerf_raygen(const float* Kinv_host, const float* T_host, int H, int W, int row0, int row_step, int n_rows,
                  const float* frame_ids_host, int n_frame_ids, float* rays, int ray_stride, void* stream) {
  if (!Kinv_host || !T_host || !rays || row_step < 1 || row0 < 0 || (n_frame_ids > 0 && !frame_ids_host))
    return STNERF_EINVAL;
  return launch_raygen(Kinv_host, T_host, H, W, row0, row_step, n_rows, frame_ids_host, n_frame_ids, rays, ray_stride,
                       (cudaStream_t)stream);
}

int stnerf_intersect_sample(const float* rays, int64_t n, int ray_stride, const float* bmin_host, const float* bmax_host,
                            int is_bkgd, int n1, const float* jitter, float* t, float* xyz, uint8_t* mask,
                            float* tfar_tnear, void* stream) {
  if (!rays || !bmin_host || !bmax_host || !jitter || n1 < 1 || ray_stride < 6) return STNERF_EINVAL;
  return launch_intersect_sample(rays, n, ray_stride, bmin_host, bmax_host, is_bkgd, n1, jitter, t, xyz, mask,
                                 tfar_tnear, (cudaStream_t)stream);
}

int stnerf_composite(const float* t, const float* rgb, const float* sigma, int64_t n, int S, float boarder, float* color,
                     float* depth, float* acc, float* w, void* stream) {
  if (!t || !rgb || !sigma || !color || !depth || !acc || S < 1) return STNERF_EINVAL;
  return launch_composite_simple(t, rgb, sigma, n, S, boarder, color, depth, acc, w, (cudaStream_t)stream);
}

int stnerf_composite_pass(const stnerf_scene* scene_host, int n_layers, int fine, const float* t, const float* raw,
                          const uint8_t* mask, const float* u, uint64_t seed, int64_t n, int S, int n2, int pixel_layout,
                          float* images, float* t_fine, float* z_new, uint8_t* src_map, void* stream) {
  if (!scene_host || !t || !raw || n < 0 || n_layers < 1 || n_layers > STNERF_MAX_LAYERS) return STNERF_EINVAL;
  if ((n_layers > 1 && !mask) || (pixel_layout != 0 && pixel_layout != 1) || (fine != 0 && fine != 1)) return STNERF_EINVAL;
  if (fine ? (S < 1 || S > STNERF_MAX_S || n2 != 0) : (S < 3 || S > STNERF_MAX_N1 || n2 < 0 || S + n2 > STNERF_MAX_S))
    return STNERF_EINVAL;
  if (n2 > 0 ? !t_fine : (!images || t_fine)) return STNERF_EINVAL;
  // STNERF_PASS_GENERIC=1: a coarse pass takes the shared-memory path whatever its sample counts (A/B of the two paths)
  const char* e = getenv("STNERF_PASS_GENERIC");
  const bool generic = e && e[0] == '1';
  if ((z_new == nullptr) != (src_map == nullptr)) return STNERF_EINVAL;
  // the origin map is one byte per fine depth and only the register-resident resampling writes it
  if (z_new && (n2 == 0 || generic || !composite_pass_in_registers(S, n2, fine) || S + n2 > 256)) return STNERF_EINVAL;
  DevScene d;
  dev_scene_from(*scene_host, n_layers, d);
  CompositeArgs a;
  memset(&a, 0, sizeof(a));
  a.t = t; a.t_layer_stride = n * S;
  a.raw = raw; a.raw_layer_stride = n * S * 4;
  a.mask = mask; a.mask_layer_stride = n;
  a.u = u; a.u_layer_stride = n * n2;
  a.t_fine = t_fine; a.tf_layer_stride = n * (S + n2);
  a.z_new = z_new; a.zn_layer_stride = n * n2;
  a.src_map = src_map; a.sm_layer_stride = n * (S + n2);
  a.out = images; a.pixel_layout = pixel_layout; a.n_total = n; a.ray_base = 0; a.n = n;
  a.S = S; a.n2 = n2; a.fine = fine; a.seed = seed; a.idmap = RayIdMap{0, 0, 0};
  return launch_composite_pass(a, d, n_layers, (cudaStream_t)stream, generic);
}

int stnerf_sample_pdf(const float* t, const float* w, const float* u, int64_t n, int n1, int n2, float* z, float* t_fine,
                      void* stream) {
  if (!t || !w || !u || (!z && !t_fine) || n1 > STNERF_MAX_N1 * 4 || n1 + n2 > 4096) return STNERF_EINVAL;
  return launch_sample_pdf(t, w, u, n, n1, n2, z, t_fine, (cudaStream_t)stream);
}

int stnerf_positional_encoding(const float* x, int64_t P, int dim, int n_freq, float* out, void* stream) {
  if (!x || !out || dim < 1 || n_freq < 0 || n_freq > 16) return STNERF_EINVAL;
  return launch_posenc(x, P, dim, n_freq, out, (cudaStream_t)stream);
}

// One SpaceNet on explicit points; `render_schedule`: the weight-stage schedule the render's pass of these weights uses.
static int spacenet_explicit(stnerf_ctx* c, int layer, int fine, const float* pos, const float* dirs, const float* times,
                             int64_t P, float* rgb, float* sigma, cudaStream_t st, bool render_schedule) {
  if (!c || P < 0 || layer < 0 || layer >= c->l || (fine != 0 && fine != 1)) return STNERF_EINVAL;
  SpaceNetDev& net = c->space[fine][layer];
  if (!net.loaded) return STNERF_ENOWEIGHTS;
  if (P == 0) return STNERF_OK;        // an empty batch has no buffers (an empty torch tensor's data pointer is null)
  if (!pos || !dirs || !rgb || !sigma || (net.w.use_time && !times)) return STNERF_EINVAL;
  return run_spacenet(c, explicit_src(pos, 3, dirs, times, 1, P), net, nullptr, rgb, sigma, st, -1, nullptr,
                      render_schedule && fine != 0);
}

int stnerf_spacenet(stnerf_handle c, int layer, int fine, const float* pos, const float* dirs, const float* times,
                    int64_t P, float* rgb, float* sigma, void* stream) {
  return spacenet_explicit(c, layer, fine, pos, dirs, times, P, rgb, sigma, (cudaStream_t)stream, false);
}

int stnerf_spacenet_pass(stnerf_handle c, int layer, int fine, const float* pos, const float* dirs, const float* times,
                         int64_t P, float* rgb, float* sigma, void* stream) {
  return spacenet_explicit(c, layer, fine, pos, dirs, times, P, rgb, sigma, (cudaStream_t)stream, true);
}

}  // extern "C"

__global__ void any_fraction_kernel(const float* __restrict__ xyzt, long long P, int* __restrict__ flag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P) {
    const float t = xyzt[4 * i + 3];
    if (floorf(t) != t) atomicOr(flag, 1);
  }
}

// *flag = 1 when any of the P points (x, y, z, t) has a fractional t: MotionNet's lerp decision for a batch (motion_net.py:53)
static int launch_any_fraction(const float* xyzt, long long P, int* flag, cudaStream_t st) {
  STNERF_CUDA(cudaMemsetAsync(flag, 0, 4, st));
  any_fraction_kernel<<<(int)((P + 255) / 256), 256, 0, st>>>(xyzt, P, flag);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

extern "C" int stnerf_motionnet(stnerf_handle c, int layer, const float* xyzt, int64_t P, int lerp_mode, float* flow,
                                void* stream) {
  if (!c || P < 0 || layer < 1 || layer >= c->l || lerp_mode < -1 || lerp_mode > 1) return STNERF_EINVAL;
  MotionNetDev& net = c->motion[layer];
  if (!net.loaded) return STNERF_ENOWEIGHTS;
  if (P == 0) return STNERF_OK;        // see stnerf_spacenet
  if (!xyzt || !flow) return STNERF_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (lerp_mode < 0) {
    const int rc = launch_any_fraction(xyzt, P, c->any_frac, st);
    if (rc) return rc;
  }
  return run_motionnet(c, explicit_src(xyzt, 4, nullptr, xyzt + 3, 4, P), net, c->any_frac, lerp_mode, nullptr, flow, st);
}

// ---- a layer's field at one frame (extract.cu builds the points; the networks are the render's) ------------------------------
static constexpr long long FIELD_CHUNK = 1LL << 20;

static int field_check(stnerf_ctx* c, int layer, int fine, float frame_id) {
  if (!c || layer < 0 || layer >= c->l || (fine != 0 && fine != 1) || !isfinite(frame_id)) return STNERF_EINVAL;
  if (!c->space[fine][layer].loaded || (layer > 0 && !c->motion[layer].loaded)) return STNERF_ENOWEIGHTS;
  return ctx_ready(c);
}

// Points [0, P) of `xyz` (or of grid `g` when xyz == null) through the edit, the MotionNet and the SpaceNet, chunk by chunk.
static int field_run(stnerf_ctx* c, int layer, int fine, float frame_id, const float* xyz, const FieldGrid& g, long long P,
                     const float* dirs, float* rgb, float* sigma, cudaStream_t st) {
  FieldEdit e;
  memset(&e, 0, sizeof(e));
  fill_edit(e, c->scene, layer, fine != 0);
  e.rot_on = layer_rot(c, layer, false, e.rot) ? 1 : 0;
  const bool rot_dirs = e.rot_on && dirs;                             // the SpaceNet looks along R^T dir
  const int lerp = floorf(frame_id) != frame_id ? 1 : 0;              // motion_net.py:53 for a batch of one frame
  const long long chunk = std::min(P, FIELD_CHUNK);
  // stream-ordered scratch: xyzt (chunk,4), deformed points (chunk,3), zero directions (chunk,3) when none are given,
  // rotated directions (chunk,3) for a rotated layer
  float* buf = nullptr;
  STNERF_CUDA(cudaMallocAsync((void**)&buf, (size_t)chunk * (rot_dirs ? 13 : 10) * sizeof(float), st));
  float *xyzt = buf, *def = buf + 4 * chunk, *zdirs = buf + 7 * chunk, *rdirs = buf + 10 * chunk;
  int rc = STNERF_OK;
  if (!dirs && cudaMemsetAsync(zdirs, 0, (size_t)chunk * 3 * sizeof(float), st) != cudaSuccess) rc = STNERF_ECUDA;
  for (long long p0 = 0; p0 < P && !rc; p0 += chunk) {
    const long long n = std::min(chunk, P - p0);
    rc = launch_field_points(xyz, g, p0, n, e, frame_id, xyzt, dirs, rdirs, st);
    if (!rc && layer > 0)                                              // :340-356 / :495-510: xyz += MotionNet(xyz, t)
      rc = run_motionnet(c, explicit_src(xyzt, 4, nullptr, xyzt + 3, 4, n), c->motion[layer], nullptr, lerp, def, nullptr, st);
    if (rc) break;
    const PointSrc s = explicit_src(layer > 0 ? def : xyzt, layer > 0 ? 3 : 4, rot_dirs ? rdirs : dirs ? dirs + 3 * p0 : zdirs,
                                    xyzt + 3, 4, n);
    rc = run_spacenet(c, s, c->space[fine][layer], nullptr, rgb ? rgb + 3 * p0 : nullptr, sigma + p0, st);
  }
  if (cudaFreeAsync(buf, st) != cudaSuccess && !rc) rc = STNERF_ECUDA;
  return rc;
}

extern "C" int stnerf_layer_field(stnerf_handle c, int layer, int fine, float frame_id, const float* xyz, const float* dirs,
                                  int64_t P, float* rgb, float* sigma, void* stream) {
  int rc = field_check(c, layer, fine, frame_id);
  if (rc) return rc;
  if (P < 0) return STNERF_EINVAL;
  if (P == 0) return STNERF_OK;
  if (!xyz || !sigma || (rgb && !dirs)) return STNERF_EINVAL;
  FieldGrid g;
  memset(&g, 0, sizeof(g));
  return field_run(c, layer, fine, frame_id, xyz, g, P, dirs, rgb, sigma, (cudaStream_t)stream);
}

extern "C" int stnerf_layer_grid(stnerf_handle c, int layer, int fine, float frame_id, const stnerf_grid* grid_host, float* sigma,
                                 void* stream) {
  int rc = field_check(c, layer, fine, frame_id);
  if (rc) return rc;
  if (!grid_host || !sigma) return STNERF_EINVAL;
  FieldGrid g;
  long long P = 1;
  for (int a = 0; a < 3; ++a) {
    if (grid_host->dims[a] < 2 || !isfinite(grid_host->origin[a]) || !isfinite(grid_host->step[a])) return STNERF_EINVAL;
    g.origin[a] = grid_host->origin[a]; g.step[a] = grid_host->step[a]; g.dims[a] = grid_host->dims[a];
    P *= grid_host->dims[a];
  }
  return field_run(c, layer, fine, frame_id, nullptr, g, P, nullptr, nullptr, sigma, (cudaStream_t)stream);
}

// ---- training: forward with saved activations, and the backward (mlp_train.cu, mlp_train_tc.cu) -----------------------------
static bool train_prec_ok(int prec) { return prec == STNERF_TRAIN_FP32 || prec == STNERF_TRAIN_TC_3XTF32; }

extern "C" {

size_t stnerf_train_saved_floats(int kind, int use_time, int64_t P) {
  if ((kind != 0 && kind != 1) || P < 0) return 0;
  return train_saved_floats(kind, use_time != 0) * (size_t)P;
}

size_t stnerf_train_scratch_bytes_prec(int kind, int use_time, int64_t P, int precision) {
  if ((kind != 0 && kind != 1) || P < 0 || !train_prec_ok(precision)) return 0;
  return train_scratch_bytes(kind, use_time != 0, P);     // both precisions chunk the weight-gradient sums alike
}

size_t stnerf_train_scratch_bytes(int kind, int use_time, int64_t P) {
  return stnerf_train_scratch_bytes_prec(kind, use_time, P, STNERF_TRAIN_FP32);
}

int stnerf_spacenet_train_forward_prec(const float* weights, int use_time, const float* pos, const float* dirs, const float* times,
                                       int64_t P, float* rgb, float* sigma, float* saved, int precision, void* stream) {
  if (P < 0 || !train_prec_ok(precision)) return STNERF_EINVAL;
  if (P == 0) return STNERF_OK;
  if (!weights || !pos || !dirs || !rgb || !sigma || !saved || (use_time && !times)) return STNERF_EINVAL;
  return launch_spacenet_train_forward(weights, use_time != 0, pos, dirs, times, P, rgb, sigma, saved, (cudaStream_t)stream,
                                       precision);
}

int stnerf_spacenet_train_forward(const float* weights, int use_time, const float* pos, const float* dirs, const float* times,
                                  int64_t P, float* rgb, float* sigma, float* saved, void* stream) {
  return stnerf_spacenet_train_forward_prec(weights, use_time, pos, dirs, times, P, rgb, sigma, saved, STNERF_TRAIN_FP32, stream);
}

int stnerf_spacenet_backward_prec(const float* weights, int use_time, int64_t P, const float* saved, const float* d_rgb,
                                  const float* d_sigma, float* d_weights, float* d_pos, void* scratch, size_t scratch_bytes,
                                  int precision, void* stream) {
  if (P < 0 || !d_weights || !train_prec_ok(precision)) return STNERF_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (P == 0) {                        // an empty batch contributes nothing to the gradient
    STNERF_CUDA(cudaMemsetAsync(d_weights, 0, (use_time ? SPACENET_FLOATS_TIME : SPACENET_FLOATS_NOTIME) * sizeof(float), st));
    return STNERF_OK;
  }
  if (!weights || !saved || !d_rgb || !d_sigma || !scratch ||
      scratch_bytes < stnerf_train_scratch_bytes_prec(0, use_time, P, precision))
    return STNERF_EINVAL;
  return launch_spacenet_backward(weights, use_time != 0, P, saved, d_rgb, d_sigma, d_weights, d_pos, scratch, st, precision);
}

int stnerf_spacenet_backward(const float* weights, int use_time, int64_t P, const float* saved, const float* d_rgb,
                             const float* d_sigma, float* d_weights, float* d_pos, void* scratch, size_t scratch_bytes,
                             void* stream) {
  return stnerf_spacenet_backward_prec(weights, use_time, P, saved, d_rgb, d_sigma, d_weights, d_pos, scratch, scratch_bytes,
                                       STNERF_TRAIN_FP32, stream);
}

int stnerf_motionnet_train_forward_prec(const float* weights, const float* xyzt, int64_t P, int lerp_mode, float* flow,
                                        float* saved, void* scratch, size_t scratch_bytes, int precision, void* stream) {
  if (P < 0 || lerp_mode < -1 || lerp_mode > 1 || !train_prec_ok(precision)) return STNERF_EINVAL;
  if (P == 0) return STNERF_OK;
  if (!weights || !xyzt || !flow || !saved || !scratch || scratch_bytes < stnerf_train_scratch_bytes_prec(1, 0, P, precision))
    return STNERF_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  int* flag = (int*)scratch;
  if (lerp_mode < 0) {
    const int rc = launch_any_fraction(xyzt, P, flag, st);
    if (rc) return rc;
  }
  return launch_motionnet_train_forward(weights, xyzt, P, flag, lerp_mode, flow, saved, st, precision);
}

int stnerf_motionnet_train_forward(const float* weights, const float* xyzt, int64_t P, int lerp_mode, float* flow, float* saved,
                                   void* scratch, size_t scratch_bytes, void* stream) {
  return stnerf_motionnet_train_forward_prec(weights, xyzt, P, lerp_mode, flow, saved, scratch, scratch_bytes, STNERF_TRAIN_FP32,
                                             stream);
}

int stnerf_motionnet_backward_prec(const float* weights, int64_t P, const float* saved, const float* d_flow, float* d_weights,
                                   void* scratch, size_t scratch_bytes, int precision, void* stream) {
  if (P < 0 || !d_weights || !train_prec_ok(precision)) return STNERF_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (P == 0) {
    STNERF_CUDA(cudaMemsetAsync(d_weights, 0, MOTIONNET_FLOATS * sizeof(float), st));
    return STNERF_OK;
  }
  if (!weights || !saved || !d_flow || !scratch || scratch_bytes < stnerf_train_scratch_bytes_prec(1, 0, P, precision))
    return STNERF_EINVAL;
  return launch_motionnet_backward(weights, P, saved, d_flow, d_weights, scratch, st, precision);
}

int stnerf_motionnet_backward(const float* weights, int64_t P, const float* saved, const float* d_flow, float* d_weights,
                              void* scratch, size_t scratch_bytes, void* stream) {
  return stnerf_motionnet_backward_prec(weights, P, saved, d_flow, d_weights, scratch, scratch_bytes, STNERF_TRAIN_FP32, stream);
}

int stnerf_composite_backward(const float* t, const float* rgb, const float* sigma, int64_t n, int S, float boarder,
                              const float* d_color, const float* d_depth, const float* d_acc, const float* d_w, float* d_rgb,
                              float* d_sigma, void* stream) {
  if (n < 0 || S < 1) return STNERF_EINVAL;
  if (n == 0) return STNERF_OK;
  if (!t || !rgb || !sigma || !d_rgb || !d_sigma) return STNERF_EINVAL;
  return launch_composite_backward(t, rgb, sigma, n, S, boarder, d_color, d_depth, d_acc, d_w, d_rgb, d_sigma,
                                   (cudaStream_t)stream);
}

// ---- training: the per-sample work around the networks (train_march.cu) ------------------------------------------------------
int stnerf_train_sample(stnerf_handle c, const float* rays, int64_t n, int ray_stride, int n1, const float* jitter, uint64_t seed,
                        float* t, uint8_t* mask, int32_t* hit, int32_t* hit_counts_host, int32_t* any_frac_host, void* stream) {
  if (!c || n < 0 || n1 < 3 || n1 > STNERF_MAX_N1 || !hit_counts_host || !any_frac_host) return STNERF_EINVAL;
  if ((long long)n * STNERF_MAX_S >= (1LL << 31)) return STNERF_EINVAL;      // 32-bit sample indices, as for a render chunk
  int rc = ctx_ready(c);
  if (rc) return rc;
  if (!ray_stride_ok(c, ray_stride)) return STNERF_EINVAL;
  hit_counts_host[0] = (int32_t)n;
  any_frac_host[0] = 0;
  for (int i = 1; i < c->l; ++i) hit_counts_host[i] = any_frac_host[i] = 0;
  if (n == 0) return STNERF_OK;
  if (!rays || !t || !mask || !hit) return STNERF_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t ints = 2 * STNERF_MAX_LAYERS + train_hits_scratch_ints(n, c->l);
  int* scratch = nullptr;
  STNERF_CUDA(cudaMallocAsync((void**)&scratch, ints * sizeof(int), st));
  int* counts = scratch;                              // sample_kernel's own (unordered) counters, then the ordered totals
  int* lerp = scratch + STNERF_MAX_LAYERS;
  STNERF_CUDA(cudaMemsetAsync(scratch, 0, 2 * STNERF_MAX_LAYERS * sizeof(int), st));
  // sampling as in render_core (rotated layers along their own rays); its block-ordered hit lists land in `hit` and are
  // overwritten in ray order below
  LayerRays lr;
  {
    RotatedRays rot;
    rc = rot.init(c, n, ray_stride, st);
    if (!rc) rc = rot.rotate(rays, n, lr);
    if (!rc)
      rc = launch_sample(rays, n, ray_stride, c->dscene, c->l, n1, jitter, n * n1, seed, 0, c->idmap, t, n * n1, mask, n, hit, n,
                         counts, lerp, st, c->box_table, c->box_frames, &lr);
  }
  if (!rc) rc = launch_train_hits(mask, n, c->l, rays, ray_stride, c->scene.shared_frame_id, hit,
                                  scratch + 2 * STNERF_MAX_LAYERS, counts, st);
  int host[2 * STNERF_MAX_LAYERS];
  if (!rc && cudaMemcpyAsync(host, counts, sizeof(host), cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = STNERF_ECUDA;
  if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = STNERF_ECUDA;     // the one host sync: sizes the saved activations
  cudaFreeAsync(scratch, st);
  if (rc) return rc;
  for (int i = 1; i < c->l; ++i) { hit_counts_host[i] = host[i]; any_frac_host[i] = host[STNERF_MAX_LAYERS + i]; }
  return STNERF_OK;
}

int stnerf_train_points(stnerf_handle c, int layer, int fine, const float* rays, int64_t n, int ray_stride, const float* t, int S,
                        const int32_t* hit, int64_t m, float* pos, float* dirs, float* times, float* xyzt, void* stream) {
  if (!c || layer < 0 || layer >= c->l || (fine != 0 && fine != 1) || n < 0 || m < 0 || S < 1 || S > STNERF_MAX_S) return STNERF_EINVAL;
  if ((layer == 0) != (hit == nullptr) || m > n || (layer == 0 && m != n)) return STNERF_EINVAL;
  int rc = ctx_ready(c);
  if (rc) return rc;
  if (!ray_stride_ok(c, ray_stride)) return STNERF_EINVAL;
  if (m == 0) return STNERF_OK;
  if (!rays || !t || (!pos && !dirs && !times && !xyzt)) return STNERF_EINVAL;
  // a rotated layer: the points and directions of its own rays, as render_core marches them
  RotatedRays rot;
  rc = rot.init(c, n, ray_stride, (cudaStream_t)stream, layer);
  LayerRays lr;
  if (!rc) rc = rot.rotate(rays, n, lr);
  if (rc) return rc;
  PointSrc s = march_src(c, layer, fine != 0, lr.p[layer], ray_stride, t, S);
  s.hit = hit; s.n_slots = m;
  return launch_train_points(s, (long long)m * S, pos, dirs, times, xyzt, (cudaStream_t)stream);
}

int stnerf_train_scatter(stnerf_handle c, int layer, int fine, const float* t, int64_t n, int S, const int32_t* hit, int64_t m,
                         const float* rgb_c, const float* sigma_c, float* rgb, float* sigma, float* factor, void* stream) {
  if (!c || layer < 0 || layer >= c->l || (fine != 0 && fine != 1) || n < 0 || m < 0 || m > n || S < 1) return STNERF_EINVAL;
  if ((layer == 0) != (hit == nullptr) || (layer == 0 && m != n)) return STNERF_EINVAL;
  const int rc = ctx_ready(c);
  if (rc) return rc;
  if (n == 0) return STNERF_OK;
  if (!t || !rgb || !sigma || (m > 0 && (!rgb_c || !sigma_c || !factor))) return STNERF_EINVAL;
  return launch_train_scatter(c->dscene, layer, fine, t, n, S, hit, m * S, rgb_c, sigma_c, rgb, sigma, factor, (cudaStream_t)stream);
}

int stnerf_train_gather(stnerf_handle c, int S, const int32_t* hit, int64_t m, const float* factor, const float* d_rgb,
                        const float* d_sigma, float* d_rgb_c, float* d_sigma_c, void* stream) {
  if (!c || m < 0 || S < 1) return STNERF_EINVAL;
  const int rc = ctx_ready(c, /*need_scene=*/false);
  if (rc) return rc;
  if (m == 0) return STNERF_OK;
  if (!factor || !d_rgb_c || !d_sigma_c) return STNERF_EINVAL;
  return launch_train_gather(S, hit, m * S, factor, d_rgb, d_sigma, d_rgb_c, d_sigma_c, (cudaStream_t)stream);
}

int stnerf_train_uniforms(stnerf_handle c, int64_t n, int n2, uint64_t seed, float* u, void* stream) {
  if (!c || n < 0 || n2 < 0) return STNERF_EINVAL;
  if (n == 0 || n2 == 0) return STNERF_OK;
  if (!u) return STNERF_EINVAL;
  return launch_train_uniforms(n, n2, c->l, seed, c->idmap, u, (cudaStream_t)stream);
}

}  // extern "C"
