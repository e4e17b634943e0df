// model.cuh — the SD-v1.4 sampling graph on top of the kernels (UNet, VAE decoder, DDIM sampler).
#pragma once
#include "../../include/sdb200.h"
#include "runtime.cuh"

namespace sdb {

void model_create(Ctx& c);   // builds the tensor registry, allocates arenas
// rejects a unet/input_blocks/conv/weight of [320,C,3,3] with C != c.unet_cin (4, 8 or 9), naming both shapes and the create
// entry to use
void check_conv_in_shape(const Ctx& c, const std::string& what, int ndim, const int64_t* dims);
void model_destroy(Ctx& c);
void model_init_synthetic(Ctx& c, uint32_t seed);
void model_finalize(Ctx& c);  // packs weights into kernel layouts
void model_invalidate_graphs(Ctx& c);
// LoRA adapters (DESIGN §7 f8; include/sdb200.h: sdb_lora_*)
void model_lora_add(Ctx& c, int adapter, const char* tensor, int rank, const float* down, const float* up, double alpha);
void model_lora_scale(Ctx& c, int adapter, double multiplier);
void model_lora_remove(Ctx& c, int adapter);  // -1 = all
void model_lora_apply(Ctx& c);
bool model_lora_pending(Ctx& c);
void model_get_merged_tensor(Ctx& c, const char* tensor, float* host, int64_t count);

void model_unet_forward_host(Ctx& c, const float* x, int t, const float* context, int n, int H, int W, int L, float* out);
void model_unet_forward_at_host(Ctx& c, const float* x, double t, const float* context, int n, int H, int W, int L, float* out);
void model_unet_forward_dev(Ctx& c, const float* d_x, int t, const float* d_context, int n, int H, int W, int L,
                            float* d_out, cudaStream_t caller);
void model_decode_host(Ctx& c, const float* latent, int n, int H, int W, float* img);
void model_decode_dev(Ctx& c, const float* d_latent, int n, int H, int W, float* d_img, cudaStream_t caller);
void model_encode_host(Ctx& c, const float* img, int n, int H, int W, float* latent);
void model_encode_dev(Ctx& c, const float* d_img, int n, int H, int W, float* d_latent, cudaStream_t caller);
void model_latent_to_image_host(Ctx& c, const float* latent, int n, int H, int W, uint8_t* rgb);
// One sampling call of any kind: text-to-image, image-to-image / masked inpainting / 9-channel inpainting (DESIGN §7 f5, f9),
// batches of different requests (f7) and InstructPix2Pix edits (f10). The sdb_* sampling entries fill it from their arguments;
// pointers are host pointers for model_sample_host and device pointers for model_sample_dev.
enum : int { SAMPLE_TXT2IMG = 0, SAMPLE_IMG2IMG = 1, SAMPLE_EDIT = 2 };
struct SampleRequest {
  int kind = SAMPLE_TXT2IMG;  // SAMPLE_IMG2IMG: plain, masked or 9-channel inpainting, as the context's UNet and the mask select
  // the prompts: a batch entry's descriptor (batched; may be null, which the checks reject), or n prompts of L rows [n][L][768],
  // one negative of Lu rows [Lu][768] broadcast over the batch and one guidance scale (an edit's text scale)
  bool batched = false;
  const sdb_batch* batch = nullptr;
  const float* context = nullptr;
  const float* uncond = nullptr;
  int n = 0, L = 0, Lu = 0;
  double scale = 0.0;
  const uint8_t* image = nullptr;  // img2img, edit: u8 [n,8H,8W,3]
  const uint8_t* mask = nullptr;   // img2img: u8 [n,8H,8W] or null
  double strength = 1.0;           // img2img
  double image_scale = 0.0;        // edit
  // [n,4,H,W]: the init latent (txt2img, edit) or the noise (img2img). Null: drawn from seed (host entries) or a batch's seeds
  const float* start = nullptr;
  uint64_t seed = 0;
  int n_steps = 0, H = 0, W = 0;   // latent height and width
  float* latent_out = nullptr;     // [n,4,H,W] or null
  uint8_t* rgb = nullptr;          // u8 [n,8H,8W,3] or null
};
void model_sample_dev(Ctx& c, const SampleRequest& r, cudaStream_t caller);
void model_sample_host(Ctx& c, const SampleRequest& r);
void model_forward_diffuser_dev(Ctx& c, const float* d_latent, int t, const float* d_context, int n, int L, const float* d_uncond,
                                int Lu, double scale, int H, int W, float* d_pred, float* d_u, float* d_c, cudaStream_t caller);
void model_forward_diffuser_host(Ctx& c, const float* latent, int t, const float* context, int n, int L, const float* uncond,
                                 int Lu, double scale, int H, int W, float* pred, float* out_u, float* out_c);
void model_clip_forward_dev(Ctx& c, const int* d_tokens, int n, int L, float* d_out, cudaStream_t caller);
void model_clip_forward_host(Ctx& c, const int* tokens, int n, int L, float* out);
// dump-dir reader (dumpdir.cu)
bool npy_read_f32(const std::string& file, std::vector<float>& out);
long long dump_tensor_read(const std::string& file, int ndim, int64_t* dims, std::vector<float>& payload);
void model_load_dump_dir(Ctx& c, const char* root);
// SD-1.x single-file .safetensors checkpoints (safetensors.cu)
void model_load_safetensors(Ctx& c, const char* path);
void safetensors_probe(const char* path, int* kind, int* conv_in_width);

// ---- test entries (host pointers; each call stages through the context's work arena)
// Records every traced launch while it lives, when `out` (SDB_TRACE_INTS ints, sdb200.h) is not null; write() fills `out` and
// fails the call if the records do not fit.
struct TraceScope {
  Ctx& c;
  int32_t* out;
  TraceScope(Ctx& c, int32_t* out) : c(c), out(out) {
    c.trace.clear();
    c.trace_on = out != nullptr;
  }
  ~TraceScope() { c.trace_on = false; }
  void write() const;
};
// `count` host values copied to a new work-arena buffer on the context's stream (null host: null)
template <class T>
T* upload(Ctx& c, const T* host, size_t count) {
  if (!host) return nullptr;
  T* d = c.work.get<T>(count);
  SDB_CUDA(cudaMemcpyAsync(d, host, count * sizeof(T), cudaMemcpyHostToDevice, c.stream));
  return d;
}
// `count` fp16 hi + lo pairs read back as fp32 (a null half reads as 0): out[i] = hi[i] + lo[i], or with planes hi to
// out[0, count) and lo to out[count, 2 count)
void fetch_pair(Ctx& c, Half2Ptr p, size_t count, float* out, bool planes = false);
// fetch_pair of an NHWC [n][H][W][C] tensor, written NCHW
void fetch_half2(Ctx& c, Half2Ptr p, int n, int C, int H, int W, float* out);

void model_test_gemm_ex(Ctx& c, const float* a, const float* w, const float* bias, const float* residual, int M, int K, int N,
                        int passes, int flags, const float* xa, const float* xw, int XK, float* out, int32_t* trace);
void model_test_conv2d(Ctx& c, const float* x, const float* w, const float* bias, int n, int cin, int H, int W, int cout, int k,
                       int stride, int upsample, int passes, float* y, int32_t* trace);
void model_test_conv_groupnorm(Ctx& c, const float* x, const float* w, const float* bias, const float* gamma, const float* beta,
                               int n, int cin, int H, int W, int cout, int k, int stride, int upsample, int passes, int silu,
                               float* y, int* slots, int32_t* trace);
void model_test_ln_fold(Ctx& c, const float* a, const float* a2, const float* w0, const float* b0, const float* gamma,
                        const float* beta, const float* w1, const float* b1, int M, int K0, int C, int N, int passes, int geglu,
                        float* out, int32_t* trace);
void model_test_attention(Ctx& c, const float* q, const float* k, const float* v, int n, int Nq, int Nk, int C, int heads,
                          const int32_t* kvlen, int flags, float* out);
void model_test_resblock(Ctx& c, const float* x0, const float* x1, int n, int C0, int C1, int H, int W, int Cout,
                         const float* n1g, const float* n1b, const float* w1, const float* b1, const float* n2g, const float* n2b,
                         const float* w2, const float* b2, const float* wsk, const float* bsk, const float* emb_bias, int passes,
                         int flags, float* out, float* out16, float* outn, int32_t* trace);
void model_test_groupnorm_cat(Ctx& c, const float* x0, const float* x1, int n, int C0, int C1, int H, int W, const float* gamma,
                              const float* beta, int silu, int mode, float* y, int32_t* trace);
void model_test_spatial_transformer(Ctx& c, int index, const float* x, int n, int C, int H, int W, const float* context, int Lmax,
                                    const int32_t* lens, int flags, float* out, float* out16, float* out_norm, float* taps_y,
                                    float* taps_ln, int32_t* trace);
void model_test_vae_stage(Ctx& c, int stage, const float* x, const float* cond, int n, int C, int H, int W, float scale, int flags,
                          float* out, float* out16, float* tap, float* out_norm, int32_t* trace);
void model_test_clip_block(Ctx& c, int index, const float* x, int n, int L, int flags, float* out, float* taps, int32_t* trace);

}  // namespace sdb
