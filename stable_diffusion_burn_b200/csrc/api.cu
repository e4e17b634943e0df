// api.cu — extern "C" boundary (include/sdb200.h). No exception crosses it.
#include "../../include/sdb200.h"

#include <dlfcn.h>

#include <cstdlib>
#include <cstring>
#include <mutex>

#include "attention.cuh"
#include "kernels.cuh"
#include "model.cuh"
#include "runtime.cuh"

using namespace sdb;

struct sdb_ctx {
  Ctx c;
};

static thread_local std::string g_err;

#define API_BEGIN(ctxp)                      \
  if (!(ctxp)) {                             \
    g_err = "null context";                  \
    return 1;                                \
  }                                          \
  Ctx& c = (ctxp)->c;                        \
  try {                                      \
    SDB_CUDA(cudaSetDevice(c.device));

#define API_END                              \
  }                                          \
  catch (const std::exception& e) {          \
    c.err = e.what();                        \
    g_err = c.err;                           \
    return 1;                                \
  }                                          \
  return 0;

// one teardown for sdb_destroy and for a failed sdb_create (a context holds ~35 GB of device memory)
static void ctx_teardown(sdb_ctx* h) {
  if (!h) return;
  cudaSetDevice(h->c.device);
  cudaDeviceSynchronize();
  model_destroy(h->c);
  h->c.io_destroy();
  h->c.master.destroy();
  h->c.packed.destroy();
  h->c.work.destroy();
  if (h->c.stream) cudaStreamDestroy(h->c.stream);
  h->c.stream = nullptr;
  delete h;
}

// ------------------------------------------------------------------------------ NCCL, resolved at run time
// The library has no link-time dependency on NCCL: libnccl.so.2 is dlopen'ed by the first multi-GPU call (inside a torch
// process this binds to the copy torch already loaded, same SONAME). Only the four entry points used are declared.
namespace {
struct NcclApi {
  typedef struct { char internal[128]; } UniqueId;
  int (*GetUniqueId)(UniqueId*) = nullptr;
  int (*CommInitRank)(void** comm, int nranks, UniqueId id, int rank) = nullptr;
  int (*Broadcast)(const void* send, void* recv, size_t count, int dtype, int root, void* comm, cudaStream_t st) = nullptr;
  int (*CommDestroy)(void* comm) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};
NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return;
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
    api.Broadcast = (decltype(api.Broadcast))dlsym(h, "ncclBroadcast");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
    api.ok = api.GetUniqueId && api.CommInitRank && api.Broadcast && api.CommDestroy;
  });
  return api;
}
void nccl_check(int rc, const char* what) {
  if (rc != 0) {
    NcclApi& a = nccl();
    throw Error(std::string(what) + " failed: " + (a.GetErrorString ? a.GetErrorString(rc) : "nccl error " + std::to_string(rc)));
  }
}
}  // namespace

extern "C" {

const char* sdb_version(void) { return "sdb200 0.2.0 sm_90a"; }

static int create(int device, int unet_cin, sdb_ctx** out) {
  if (!out) {
    g_err = "null out pointer";
    return 1;
  }
  *out = nullptr;
  sdb_ctx* h = nullptr;
  try {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
      throw Error(std::string("no CUDA device available (") + cudaGetErrorString(e) +
                  "); this library has no CPU fallback");
    if (device < 0 || device >= ndev) throw Error("device index out of range");
    SDB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    SDB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
      throw Error(std::string("device is sm_") + std::to_string(prop.major) + std::to_string(prop.minor) +
                  "; kernels are built for sm_90a only");
    g_num_sms = prop.multiProcessorCount;
    h = new sdb_ctx();
    h->c.device = device;
    h->c.unet_cin = unet_cin;
    h->c.debug_sync = getenv("SDB_DEBUG_SYNC") && atoi(getenv("SDB_DEBUG_SYNC")) != 0;
    if (getenv("SDB_PDL")) g_pdl_enabled = atoi(getenv("SDB_PDL")) != 0;
    SDB_CUDA(cudaStreamCreateWithFlags(&h->c.stream, cudaStreamNonBlocking));
    model_create(h->c);
    *out = h;
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    ctx_teardown(h);  // arenas, stream, model, tickets: nothing of a half-built context may leak
    return 1;
  }
}

int sdb_create(int device, sdb_ctx** out) { return create(device, 4, out); }

int sdb_create_inpaint(int device, sdb_ctx** out) { return create(device, 9, out); }

int sdb_create_pix2pix(int device, sdb_ctx** out) { return create(device, 8, out); }

int sdb_destroy(sdb_ctx* ctx) {
  ctx_teardown(ctx);
  return 0;
}

const char* sdb_last_error(sdb_ctx* ctx) { return ctx ? ctx->c.err.c_str() : g_err.c_str(); }

// ------------------------------------------------------------------------------ weights
int sdb_tensor_count(sdb_ctx* ctx) { return ctx ? (int)ctx->c.tensors.size() : -1; }

int sdb_tensor_info(sdb_ctx* ctx, int index, const char** name, int64_t dims[4], int* ndim) {
  API_BEGIN(ctx)
  SDB_CHECK(index >= 0 && index < (int)c.tensors.size(), "tensor index");
  const TensorInfo& t = c.tensors[index];
  if (name) *name = t.name.c_str();
  if (dims)
    for (int i = 0; i < 4; ++i) dims[i] = t.dims[i];
  if (ndim) *ndim = t.ndim;
  API_END
}

int sdb_set_tensor(sdb_ctx* ctx, const char* name, const float* host, const int64_t* dims, int ndim) {
  API_BEGIN(ctx)
  SDB_CHECK(name && host && dims, "null argument");
  const TensorInfo& t = c.info(name);
  if (t.name == "unet/input_blocks/conv/weight") check_conv_in_shape(c, "set_tensor", ndim, dims);
  SDB_CHECK(ndim == t.ndim, std::string("rank mismatch for ") + name);
  for (int i = 0; i < ndim; ++i) SDB_CHECK(dims[i] == t.dims[i], std::string("shape mismatch for ") + name);
  SDB_CUDA(cudaMemcpyAsync(c.master_ptr(name), host, t.count * sizeof(float), cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  c.finalized = false;
  API_END
}

int sdb_get_tensor(sdb_ctx* ctx, const char* name, float* host, int64_t count) {
  API_BEGIN(ctx)
  const TensorInfo& t = c.info(name);
  SDB_CHECK(count == t.count, "element count mismatch");
  SDB_CUDA(cudaMemcpyAsync(host, c.master_ptr(name), t.count * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  API_END
}

int sdb_load_dump_dir(sdb_ctx* ctx, const char* path) {
  API_BEGIN(ctx)
  model_load_dump_dir(c, path);
  API_END
}

int64_t sdb_read_dump_tensor(const char* file, int ndim, int64_t* dims, float* data, int64_t capacity) {
  try {
    SDB_CHECK(file && dims && ndim >= 1 && ndim <= 4, "bad argument");
    std::vector<float> payload;
    int64_t d[4];
    const long long count = dump_tensor_read(file, ndim, d, payload);
    for (int i = 0; i < ndim; ++i) dims[i] = d[i];
    if (data) {
      SDB_CHECK(capacity >= count, "buffer too small");
      std::memcpy(data, payload.data() + ndim, (size_t)count * sizeof(float));
    }
    return count;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

int sdb_load_safetensors(sdb_ctx* ctx, const char* path) {
  API_BEGIN(ctx)
  model_load_safetensors(c, path);
  API_END
}

int sdb_probe_safetensors(const char* path, int* kind, int* conv_in_width) {
  try {
    safetensors_probe(path, kind, conv_in_width);
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

int sdb_init_synthetic(sdb_ctx* ctx, uint32_t seed) {
  API_BEGIN(ctx)
  c.norm_eps.clear();
  model_init_synthetic(c, seed);
  c.finalized = false;
  API_END
}

int sdb_weight_arena(sdb_ctx* ctx, void** dev_ptr, size_t* bytes) {
  API_BEGIN(ctx)
  if (dev_ptr) *dev_ptr = c.master.base;
  if (bytes) *bytes = c.master.off;
  API_END
}

int sdb_nccl_unique_id(void* id128) {
  try {
    SDB_CHECK(id128, "null argument");
    SDB_CHECK(nccl().ok, "libnccl.so.2 not found: multi-GPU weight broadcast unavailable");
    NcclApi::UniqueId id;
    nccl_check(nccl().GetUniqueId(&id), "ncclGetUniqueId");
    std::memcpy(id128, &id, sizeof(id));
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

int sdb_broadcast_weights(sdb_ctx* ctx, const void* id128, int rank, int world) {
  API_BEGIN(ctx)
  SDB_CHECK(id128 && world >= 1 && rank >= 0 && rank < world, "broadcast_weights arguments");
  if (world > 1) {
    SDB_CHECK(nccl().ok, "libnccl.so.2 not found: multi-GPU weight broadcast unavailable");
    NcclApi::UniqueId id;
    std::memcpy(&id, id128, sizeof(id));
    void* comm = nullptr;
    nccl_check(nccl().CommInitRank(&comm, world, id, rank), "ncclCommInitRank");
    try {
      // (1) the fp32 master arena: every tensor of the registry in one contiguous block (dtype 7 = ncclFloat32)
      nccl_check(nccl().Broadcast(c.master.base, c.master.base, c.master.off / sizeof(float), 7, 0, comm, c.stream), "ncclBroadcast(arena)");
      // (2) the per-norm eps table a dump-dir carries beside the tensors (host map on rank 0): one float per registry tensor
      // (0 = default), so ranks that did not read the directory normalise with the same eps
      const size_t nt = c.tensors.size();
      std::vector<float> eps(nt, 0.f);
      if (rank == 0)
        for (size_t i = 0; i < nt; ++i)
          if (c.tensors[i].kind == K_NORM_G) {
            const std::string& nm = c.tensors[i].name;
            auto it = c.norm_eps.find(nm.substr(0, nm.rfind('/')));
            if (it != c.norm_eps.end()) eps[i] = it->second;
          }
      float* d_eps = (float*)c.io(5, nt * sizeof(float));
      SDB_CUDA(cudaMemcpyAsync(d_eps, eps.data(), nt * sizeof(float), cudaMemcpyHostToDevice, c.stream));
      nccl_check(nccl().Broadcast(d_eps, d_eps, nt, 7, 0, comm, c.stream), "ncclBroadcast(eps)");
      SDB_CUDA(cudaMemcpyAsync(eps.data(), d_eps, nt * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
      SDB_CUDA(cudaStreamSynchronize(c.stream));
      if (rank != 0) {
        c.norm_eps.clear();
        for (size_t i = 0; i < nt; ++i)
          if (eps[i] > 0.f) {
            const std::string& nm = c.tensors[i].name;
            c.norm_eps[nm.substr(0, nm.rfind('/'))] = eps[i];
          }
      }
    } catch (...) {
      nccl().CommDestroy(comm);
      throw;
    }
    nccl_check(nccl().CommDestroy(comm), "ncclCommDestroy");
  }
  c.finalized = false;
  API_END
}

int sdb_finalize_weights(sdb_ctx* ctx) {
  API_BEGIN(ctx)
  model_finalize(c);
  c.finalized = true;
  API_END
}

// ------------------------------------------------------------------------------ hot path
static void need_final(Ctx& c) {
  SDB_CHECK(c.finalized, "call sdb_finalize_weights first");
  SDB_CHECK(!model_lora_pending(c), "LoRA adapter changes are pending: call sdb_lora_apply first");
}

int sdb_unet_forward(sdb_ctx* ctx, const float* x, int32_t timestep, const float* context, int n, int H, int W, int L,
                     float* out) {
  API_BEGIN(ctx)
  need_final(c);
  model_unet_forward_host(c, x, timestep, context, n, H, W, L, out);
  API_END
}

int sdb_unet_forward_at(sdb_ctx* ctx, const float* x, double t, const float* context, int n, int H, int W, int L, float* out) {
  API_BEGIN(ctx)
  need_final(c);
  model_unet_forward_at_host(c, x, t, context, n, H, W, L, out);
  API_END
}

int sdb_unet_forward_dev(sdb_ctx* ctx, const float* d_x, int32_t timestep, const float* d_context, int n, int H, int W,
                         int L, float* d_out, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  model_unet_forward_dev(c, d_x, timestep, d_context, n, H, W, L, d_out, (cudaStream_t)stream);
  API_END
}

int sdb_decode_latent(sdb_ctx* ctx, const float* latent, int n, int H, int W, float* img) {
  API_BEGIN(ctx)
  need_final(c);
  model_decode_host(c, latent, n, H, W, img);
  API_END
}

int sdb_decode_latent_dev(sdb_ctx* ctx, const float* d_latent, int n, int H, int W, float* d_img, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  model_decode_dev(c, d_latent, n, H, W, d_img, (cudaStream_t)stream);
  API_END
}

// the request of a single-prompt sampling entry: n prompts of L rows, one negative of Lu rows broadcast over them, one scale
static SampleRequest uniform_request(int kind, const float* context, int n, int L, const float* uncond, int Lu, double scale,
                                     int n_steps, int H, int W) {
  SampleRequest r;
  r.kind = kind, r.context = context, r.n = n, r.L = L, r.uncond = uncond, r.Lu = Lu, r.scale = scale;
  r.n_steps = n_steps, r.H = H, r.W = W;
  return r;
}

static SampleRequest batch_request(int kind, const sdb_batch* batch, int n_steps, int H, int W) {
  SampleRequest r;
  r.kind = kind, r.batched = true, r.batch = batch, r.n_steps = n_steps, r.H = H, r.W = W;
  return r;
}

int sdb_sample_latent(sdb_ctx* ctx, const float* context, int n, int L, const float* uncond, int Lu,
                      double guidance_scale, int n_steps, const float* init_latent, uint64_t seed, int H, int W,
                      float* latent_out) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = uniform_request(SAMPLE_TXT2IMG, context, n, L, uncond, Lu, guidance_scale, n_steps, H, W);
  r.start = init_latent, r.seed = seed, r.latent_out = latent_out;
  model_sample_host(c, r);
  API_END
}

int sdb_latent_to_image(sdb_ctx* ctx, const float* latent, int n, int H, int W, uint8_t* rgb) {
  API_BEGIN(ctx)
  need_final(c);
  model_latent_to_image_host(c, latent, n, H, W, rgb);
  API_END
}

int sdb_sample_image(sdb_ctx* ctx, const float* context, int n, int L, const float* uncond, int Lu, double guidance_scale,
                     int n_steps, const float* init_latent, uint64_t seed, int H, int W, uint8_t* rgb) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = uniform_request(SAMPLE_TXT2IMG, context, n, L, uncond, Lu, guidance_scale, n_steps, H, W);
  r.start = init_latent, r.seed = seed, r.rgb = rgb;
  model_sample_host(c, r);
  API_END
}

int sdb_sample_image_dev(sdb_ctx* ctx, const float* d_context, int n, int L, const float* d_uncond, int Lu,
                         double guidance_scale, int n_steps, const float* d_init_latent, int H, int W, uint8_t* d_rgb,
                         void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = uniform_request(SAMPLE_TXT2IMG, d_context, n, L, d_uncond, Lu, guidance_scale, n_steps, H, W);
  r.start = d_init_latent, r.rgb = d_rgb;
  model_sample_dev(c, r, (cudaStream_t)stream);
  API_END
}

int sdb_img2img(sdb_ctx* ctx, const uint8_t* image, const uint8_t* mask, double strength, const float* context, int n, int L,
                const float* uncond, int Lu, double guidance_scale, int n_steps, const float* noise, uint64_t seed, int H, int W,
                float* latent_out, uint8_t* rgb_out) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = uniform_request(SAMPLE_IMG2IMG, context, n, L, uncond, Lu, guidance_scale, n_steps, H, W);
  r.image = image, r.mask = mask, r.strength = strength, r.start = noise, r.seed = seed, r.latent_out = latent_out, r.rgb = rgb_out;
  model_sample_host(c, r);
  API_END
}

int sdb_img2img_dev(sdb_ctx* ctx, const uint8_t* d_image, const uint8_t* d_mask, double strength, const float* d_context, int n,
                    int L, const float* d_uncond, int Lu, double guidance_scale, int n_steps, const float* d_noise, int H, int W,
                    float* d_latent_out, uint8_t* d_rgb_out, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = uniform_request(SAMPLE_IMG2IMG, d_context, n, L, d_uncond, Lu, guidance_scale, n_steps, H, W);
  r.image = d_image, r.mask = d_mask, r.strength = strength, r.start = d_noise, r.latent_out = d_latent_out, r.rgb = d_rgb_out;
  model_sample_dev(c, r, (cudaStream_t)stream);
  API_END
}

int sdb_edit_image(sdb_ctx* ctx, const uint8_t* image, const float* context, int n, int L, const float* uncond, int Lu,
                   double text_scale, double image_scale, int n_steps, const float* init_latent, uint64_t seed, int H, int W,
                   float* latent_out, uint8_t* rgb_out) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = uniform_request(SAMPLE_EDIT, context, n, L, uncond, Lu, text_scale, n_steps, H, W);
  r.image = image, r.image_scale = image_scale, r.start = init_latent, r.seed = seed, r.latent_out = latent_out, r.rgb = rgb_out;
  model_sample_host(c, r);
  API_END
}

int sdb_edit_image_dev(sdb_ctx* ctx, const uint8_t* d_image, const float* d_context, int n, int L, const float* d_uncond, int Lu,
                       double text_scale, double image_scale, int n_steps, const float* d_init_latent, int H, int W,
                       float* d_latent_out, uint8_t* d_rgb_out, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = uniform_request(SAMPLE_EDIT, d_context, n, L, d_uncond, Lu, text_scale, n_steps, H, W);
  r.image = d_image, r.image_scale = image_scale, r.start = d_init_latent, r.latent_out = d_latent_out, r.rgb = d_rgb_out;
  model_sample_dev(c, r, (cudaStream_t)stream);
  API_END
}

int sdb_sample_batch(sdb_ctx* ctx, const sdb_batch* batch, int n_steps, const float* init_latent, int H, int W, float* latent_out,
                     uint8_t* rgb_out) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = batch_request(SAMPLE_TXT2IMG, batch, n_steps, H, W);
  r.start = init_latent, r.latent_out = latent_out, r.rgb = rgb_out;
  model_sample_host(c, r);
  API_END
}

int sdb_sample_batch_dev(sdb_ctx* ctx, const sdb_batch* batch, int n_steps, const float* d_init_latent, int H, int W,
                         float* d_latent_out, uint8_t* d_rgb_out, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = batch_request(SAMPLE_TXT2IMG, batch, n_steps, H, W);
  r.start = d_init_latent, r.latent_out = d_latent_out, r.rgb = d_rgb_out;
  model_sample_dev(c, r, (cudaStream_t)stream);
  API_END
}

int sdb_img2img_batch(sdb_ctx* ctx, const sdb_batch* batch, const uint8_t* image, const uint8_t* mask, double strength,
                      int n_steps, const float* noise, int H, int W, float* latent_out, uint8_t* rgb_out) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = batch_request(SAMPLE_IMG2IMG, batch, n_steps, H, W);
  r.image = image, r.mask = mask, r.strength = strength, r.start = noise, r.latent_out = latent_out, r.rgb = rgb_out;
  model_sample_host(c, r);
  API_END
}

int sdb_img2img_batch_dev(sdb_ctx* ctx, const sdb_batch* batch, const uint8_t* d_image, const uint8_t* d_mask, double strength,
                          int n_steps, const float* d_noise, int H, int W, float* d_latent_out, uint8_t* d_rgb_out, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  SampleRequest r = batch_request(SAMPLE_IMG2IMG, batch, n_steps, H, W);
  r.image = d_image, r.mask = d_mask, r.strength = strength, r.start = d_noise, r.latent_out = d_latent_out, r.rgb = d_rgb_out;
  model_sample_dev(c, r, (cudaStream_t)stream);
  API_END
}

int sdb_forward_diffuser(sdb_ctx* ctx, const float* latent, int32_t timestep, const float* context, int n, int L,
                         const float* uncond, int Lu, double guidance_scale, int H, int W, float* pred, float* out_uncond,
                         float* out_cond) {
  API_BEGIN(ctx)
  need_final(c);
  SDB_CHECK(latent && context && uncond, "null argument");
  model_forward_diffuser_host(c, latent, timestep, context, n, L, uncond, Lu, guidance_scale, H, W, pred, out_uncond, out_cond);
  API_END
}

int sdb_forward_diffuser_dev(sdb_ctx* ctx, const float* d_latent, int32_t timestep, const float* d_context, int n, int L,
                             const float* d_uncond, int Lu, double guidance_scale, int H, int W, float* d_pred, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  model_forward_diffuser_dev(c, d_latent, timestep, d_context, n, L, d_uncond, Lu, guidance_scale, H, W, d_pred, nullptr, nullptr,
                             (cudaStream_t)stream);
  API_END
}

int sdb_encode_image(sdb_ctx* ctx, const float* img, int n, int H, int W, float* latent) {
  API_BEGIN(ctx)
  need_final(c);
  SDB_CHECK(img && latent, "null argument");
  model_encode_host(c, img, n, H, W, latent);
  API_END
}

int sdb_encode_image_dev(sdb_ctx* ctx, const float* d_img, int n, int H, int W, float* d_latent, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  model_encode_dev(c, d_img, n, H, W, d_latent, (cudaStream_t)stream);
  API_END
}

int sdb_clip_forward(sdb_ctx* ctx, const int32_t* tokens, int n, int L, float* out) {
  API_BEGIN(ctx)
  need_final(c);
  SDB_CHECK(tokens && out, "null argument");
  model_clip_forward_host(c, tokens, n, L, out);
  API_END
}

int sdb_clip_forward_dev(sdb_ctx* ctx, const int32_t* d_tokens, int n, int L, float* d_out, void* stream) {
  API_BEGIN(ctx)
  need_final(c);
  model_clip_forward_dev(c, d_tokens, n, L, d_out, (cudaStream_t)stream);
  API_END
}

// ------------------------------------------------------------------------------ sampler (DESIGN.md §7 f6)
int sdb_set_sampler(sdb_ctx* ctx, int kind, double eta, uint64_t noise_seed) {
  API_BEGIN(ctx)
  char msg[160];
  snprintf(msg, sizeof(msg), "sampler: unknown kind %d (SDB_SAMPLER_DDIM = 0, SDB_SAMPLER_DPMPP_2M = 1)", kind);
  SDB_CHECK(kind == SDB_SAMPLER_DDIM || kind == SDB_SAMPLER_DPMPP_2M, msg);
  snprintf(msg, sizeof(msg), "sampler: eta %.17g must be finite and in [0, 1]", eta);
  SDB_CHECK(std::isfinite(eta) && eta >= 0.0 && eta <= 1.0, msg);
  snprintf(msg, sizeof(msg), "sampler: DPM-Solver++(2M) is deterministic; eta %.17g must be 0", eta);
  SDB_CHECK(kind != SDB_SAMPLER_DPMPP_2M || eta == 0.0, msg);
  c.sampler_kind = kind, c.sampler_eta = eta, c.sampler_noise_seed = noise_seed;
  API_END
}

// ------------------------------------------------------------------------------ schedule (DESIGN.md §7 f15)
int sdb_set_schedule(sdb_ctx* ctx, int kind) {
  API_BEGIN(ctx)
  char msg[160];
  snprintf(msg, sizeof(msg), "schedule: unknown kind %d (SDB_SCHEDULE_DDIM = 0, SDB_SCHEDULE_KARRAS = 1)", kind);
  SDB_CHECK(kind == SDB_SCHEDULE_DDIM || kind == SDB_SCHEDULE_KARRAS, msg);
  c.sampler_schedule = kind;
  API_END
}

// ------------------------------------------------------------------------------ LoRA adapters (DESIGN.md §7 f8)
int sdb_lora_add(sdb_ctx* ctx, int adapter, const char* tensor, int rank, const float* down, const float* up, double alpha) {
  API_BEGIN(ctx)
  model_lora_add(c, adapter, tensor, rank, down, up, alpha);
  API_END
}

int sdb_lora_scale(sdb_ctx* ctx, int adapter, double multiplier) {
  API_BEGIN(ctx)
  model_lora_scale(c, adapter, multiplier);
  API_END
}

int sdb_lora_remove(sdb_ctx* ctx, int adapter) {
  API_BEGIN(ctx)
  model_lora_remove(c, adapter);
  API_END
}

int sdb_lora_apply(sdb_ctx* ctx) {
  API_BEGIN(ctx)
  model_lora_apply(c);
  API_END
}

int sdb_get_merged_tensor(sdb_ctx* ctx, const char* tensor, float* host, int64_t count) {
  API_BEGIN(ctx)
  model_get_merged_tensor(c, tensor, host, count);
  API_END
}

// ------------------------------------------------------------------------------ options / profiling
int sdb_set_option(sdb_ctx* ctx, const char* key, int value) {
  API_BEGIN(ctx)
  const std::string k = key ? key : "";
  if (k == "precision")
    c.opt_precision = value;
  else if (k == "graphs")
    c.opt_graphs = value;
  else if (k == "splitk")
    c.opt_splitk = value;
  else if (k == "raw16")
    c.opt_raw16 = value;
  else if (k == "attn_split")
    c.opt_attn_split = value;
  else if (k == "emb_hoist")
    c.opt_emb_hoist = value;
  else if (k == "gn_epilogue")
    c.opt_gn_epilogue = value;
  else if (k == "skip_merge")
    c.opt_skip_merge = value;
  else
    throw Error("unknown option: " + k);
  model_invalidate_graphs(c);
  API_END
}

int sdb_profile_enable(sdb_ctx* ctx, int on) {
  API_BEGIN(ctx)
  profile_collect(c);
  c.profiling = on != 0;
  API_END
}
int sdb_profile_reset(sdb_ctx* ctx) {
  API_BEGIN(ctx)
  profile_collect(c);
  c.launches = 0;
  for (int i = 0; i < KC_COUNT; ++i) c.cls_ms[i] = c.cls_flops[i] = c.cls_bytes[i] = c.cls_issued[i] = 0, c.cls_launches[i] = 0;
  API_END
}
int sdb_profile_class_count(sdb_ctx*) { return KC_COUNT; }
int sdb_profile_get(sdb_ctx* ctx, int cls, const char** name, int64_t* launches, double* ms, double* flops, double* bytes) {
  API_BEGIN(ctx)
  SDB_CHECK(cls >= 0 && cls < KC_COUNT, "class index");
  profile_collect(c);
  if (name) *name = kernel_class_name(cls);
  if (launches) *launches = c.cls_launches[cls];
  if (ms) *ms = c.cls_ms[cls];
  if (flops) *flops = c.cls_flops[cls];
  if (bytes) *bytes = c.cls_bytes[cls];
  API_END
}
int sdb_profile_get_issued(sdb_ctx* ctx, int cls, double* issued_flops) {
  API_BEGIN(ctx)
  SDB_CHECK(cls >= 0 && cls < KC_COUNT && issued_flops, "class index");
  *issued_flops = c.cls_issued[cls];
  API_END
}
int64_t sdb_launch_count(sdb_ctx* ctx) { return ctx ? ctx->c.launches : -1; }

// ------------------------------------------------------------------------------ single-kernel test entries
// (host pointers; each call stages through the context's work arena)

int sdb_test_gemm_ex(sdb_ctx* ctx, const float* a, const float* w, const float* bias, const float* residual, int M, int K, int N,
                     int passes, int flags, const float* xa, const float* xw, int XK, float* out, int32_t* trace) {
  API_BEGIN(ctx)
  c.work.reset();
  model_test_gemm_ex(c, a, w, bias, residual, M, K, N, passes, flags, xa, xw, XK, out, trace);
  API_END
}

int sdb_test_conv2d(sdb_ctx* ctx, const float* x, const float* w, const float* bias, int n, int cin, int H, int W,
                    int cout, int ksize, int stride, int upsample, int passes, float* y, int32_t* trace) {
  API_BEGIN(ctx)
  c.work.reset();
  model_test_conv2d(c, x, w, bias, n, cin, H, W, cout, ksize, stride, upsample, passes, y, trace);
  API_END
}

int sdb_test_ln_fold(sdb_ctx* ctx, const float* a, const float* a2, const float* w0, const float* b0, const float* gamma,
                     const float* beta, const float* w1, const float* b1, int M, int K0, int C, int N, int passes, int geglu,
                     float* out, int32_t* trace) {
  API_BEGIN(ctx)
  c.work.reset();
  model_test_ln_fold(c, a, a2, w0, b0, gamma, beta, w1, b1, M, K0, C, N, passes, geglu, out, trace);
  API_END
}

int sdb_test_conv_groupnorm(sdb_ctx* ctx, const float* x, const float* w, const float* bias, const float* gamma, const float* beta,
                            int n, int cin, int H, int W, int cout, int ksize, int stride, int upsample, int passes, int silu,
                            float* y, int* used_epilogue_stats, int32_t* trace) {
  API_BEGIN(ctx)
  c.work.reset();
  model_test_conv_groupnorm(c, x, w, bias, gamma, beta, n, cin, H, W, cout, ksize, stride, upsample, passes, silu, y,
                            used_epilogue_stats, trace);
  API_END
}

int sdb_test_layernorm(sdb_ctx* ctx, const float* x, const float* gamma, const float* beta, int rows, int ch, float* y) {
  API_BEGIN(ctx)
  c.work.reset();
  const size_t cnt = (size_t)rows * ch;
  float* d_x = upload(c, x, cnt);
  float* d_y = c.work.get<float>(cnt);
  float* d_g = upload(c, gamma, ch);
  float* d_b = upload(c, beta, ch);
  layernorm_launch(d_x, rows, ch, d_g, d_b, 1e-5f, Half2Ptr{}, d_y, c.stream);
  SDB_CUDA(cudaMemcpyAsync(y, d_y, sizeof(float) * cnt, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  API_END
}

int sdb_test_attention(sdb_ctx* ctx, const float* q, const float* k, const float* v, int n, int Nq, int Nk, int C,
                       int heads, const int32_t* kvlen, int flags, float* out) {
  API_BEGIN(ctx)
  c.work.reset();
  model_test_attention(c, q, k, v, n, Nq, Nk, C, heads, kvlen, flags, out);
  API_END
}

int sdb_test_resblock(sdb_ctx* ctx, const float* x0, const float* x1, int n, int c0, int c1, int H, int W, int cout,
                      const float* norm1_g, const float* norm1_b, const float* conv1_w, const float* conv1_b, const float* norm2_g,
                      const float* norm2_b, const float* conv2_w, const float* conv2_b, const float* skip_w, const float* skip_b,
                      const float* emb_bias, int passes, int flags, float* out, float* out16, float* out_norm, int32_t* trace) {
  API_BEGIN(ctx)
  c.work.reset();
  model_test_resblock(c, x0, x1, n, c0, c1, H, W, cout, norm1_g, norm1_b, conv1_w, conv1_b, norm2_g, norm2_b, conv2_w, conv2_b,
                      skip_w, skip_b, emb_bias, passes, flags, out, out16, out_norm, trace);
  API_END
}

int sdb_test_groupnorm_cat(sdb_ctx* ctx, const float* x0, const float* x1, int n, int c0, int c1, int H, int W, const float* gamma,
                           const float* beta, int silu, int mode, float* y, int32_t* trace) {
  API_BEGIN(ctx)
  c.work.reset();
  model_test_groupnorm_cat(c, x0, x1, n, c0, c1, H, W, gamma, beta, silu, mode, y, trace);
  API_END
}

int sdb_test_spatial_transformer(sdb_ctx* ctx, int index, const float* x, int n, int ch, int H, int W, const float* context,
                                 int lmax, const int32_t* lens, int flags, float* out, float* out16, float* out_norm, float* taps_y,
                                 float* taps_ln, int32_t* trace) {
  API_BEGIN(ctx)
  need_final(c);
  c.work.reset();
  model_test_spatial_transformer(c, index, x, n, ch, H, W, context, lmax, lens, flags, out, out16, out_norm, taps_y, taps_ln, trace);
  API_END
}

int sdb_test_vae_stage(sdb_ctx* ctx, int stage, const float* x, const float* cond, int n, int ch, int H, int W, float scale, int flags,
                       float* out, float* out16, float* tap, float* out_norm, int32_t* trace) {
  API_BEGIN(ctx)
  need_final(c);
  c.work.reset();
  model_test_vae_stage(c, stage, x, cond, n, ch, H, W, scale, flags, out, out16, tap, out_norm, trace);
  API_END
}

int sdb_test_clip_block(sdb_ctx* ctx, int index, const float* x, int n, int L, int flags, float* out, float* taps, int32_t* trace) {
  API_BEGIN(ctx)
  need_final(c);
  c.work.reset();
  model_test_clip_block(c, index, x, n, L, flags, out, taps, trace);
  API_END
}

int sdb_test_step_noise(sdb_ctx* ctx, uint64_t noise_seed, int t, int64_t count, float* out) {
  API_BEGIN(ctx)
  SDB_CHECK(out && count >= 1, "step_noise: null output or count < 1");
  SDB_CHECK(t >= 0 && t < 1000, "step_noise: timestep must be in [0, 1000)");
  float* d = (float*)c.io(0, (size_t)count * 4);
  step_noise_launch(d, (long long)count, noise_seed, t, c.stream);
  SDB_CUDA(cudaMemcpyAsync(out, d, (size_t)count * 4, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  API_END
}

}  // extern "C"
