// kernels.cuh — launchers of the non-GEMM kernels (normalisation, operand staging, small convs,
// sampler elementwise ops, weight packing, synthetic weights).
#pragma once
#include "common.cuh"

namespace sdb {

// fp16 operand tensor [n][P][H][W][C] (hi part + optional lo residual part)
struct Half2Ptr {
  __half* hi = nullptr;
  __half* lo = nullptr;
};

// ---- GroupNorm (reference src/model/groupnorm/mod.rs:53-82), NHWC fp32
// sums: [n][32][2] doubles (sum, sum of squares) of one tensor. Deterministic: per-CTA partials (scratch `partials`,
// gn_stats_partial_floats(n,HW) floats) folded in fixed order by the last CTA; `tickets` [n] must be zero.
size_t gn_stats_partial_floats(int n, int HW);
void gn_stats_launch(const float* x, int C, int n, int HW, double* sums, float* partials, unsigned int* tickets, cudaStream_t st);
// One-launch GroupNorm(+SiLU) -> fp16 hi(/lo) operand: statistics and apply fused through an in-kernel grid wait.
// tickets: [n] zeroed counters; partials: gn_fused_partial_floats(n,HW) floats of scratch.
size_t gn_fused_partial_floats(int n, int HW);
void gn_fused_launch(const float* x0, int C0, const float* x1, int C1, int n, int H, int W, int silu, const float* gamma,
                     const float* beta, float eps, Half2Ptr out, float* partials, unsigned int* tickets, cudaStream_t st);
// GroupNorm(+SiLU) -> fp16 hi(/lo) operand from statistics the producing GEMM left beside the tensor (gemm_tc.cuh: gn_part):
// one read of x, no statistics pass, no rendezvous. part = [n][cap][C / bucket][2] floats, `slots` of the cap written.
struct GnSrc {
  const float* x = nullptr;
  int C = 0;
  const float* part = nullptr;
  int cap = 0, slots = 0;
};
// folds groups of 64 partial slots: out [n][gn_fold_slots(slots)][nbk][2]
int gn_fold_slots(int slots);
void gn_fold_launch(const float* part, int cap, int slots, int nbk, int n, float* out, cudaStream_t st);
// group sums [n][32][2] of one tensor from its producer-side partials (cap / slots as in GnSrc)
void gn_sums_from_partials_launch(const float* part, int cap, int slots, int nbk, int C, int bucket, int n, double* sums,
                                  cudaStream_t st);
void gn_apply_launch(const GnSrc& s0, const GnSrc& s1, int bucket, int n, int H, int W, int silu, const float* gamma,
                     const float* beta, float eps, Half2Ptr out, cudaStream_t st);
// Stages a conv/GEMM A operand without normalisation: cat(x0, x1) -> fp16 hi(/lo), [n][H][W][C], or with phase2 split into the
// four stride-2 phase planes [n][4][H/2][W/2][C] (the stride-2 conv input)
void prep_operand_launch(const float* x0, int C0, const float* x1, int C1, int n, int H, int W, bool phase2, Half2Ptr out,
                         cudaStream_t st);

// ---- LayerNorm (burn nn::LayerNorm; call sites unet/mod.rs:523-525): rows x C fp32 -> fp16 hi(/lo) or fp32
void layernorm_launch(const float* x, int rows, int C, const float* gamma, const float* beta, float eps,
                      Half2Ptr out, float* out_f32, cudaStream_t st);

// ---- plain fp32 -> fp16 hi(/lo) conversion (context tokens, test inputs)
void convert_f16_launch(const float* x, long long count, Half2Ptr out, cudaStream_t st);

// ---- layout conversion at the boundary
void nchw_to_nhwc_launch(const float* x, int n, int C, int H, int W, float* y, cudaStream_t st);
void nhwc_to_nchw_launch(const float* x, int n, int C, int H, int W, float* y, cudaStream_t st);

// ---- small convolutions on CUDA cores (fp32 exact)
// 3x3 pad 1, Cin = 4 (NCHW fp32 input [n,4,H,W]) -> NHWC fp32 [n,H,W,Cout]; weights OIHW fp32.
// pre: optional 1x1 4->4 conv (post_quant_conv) with scalar input scale applied to the input first.
void conv3x3_cin4_launch(const float* x_nchw, int n, int H, int W, const float* w, const float* b, int Cout,
                         const float* pre_w, const float* pre_b, float pre_scale, float* y, Half2Ptr y16, cudaStream_t st);
// conv_in of a conditioned UNet, cin 9 (inpainting, DESIGN §7 f9) or 8 (InstructPix2Pix, f10): channels 0-3 from x (sample
// stride x_stride), 4..cin-1 from cond (sample stride cond_stride, sample index modulo cond_mod); kConvCinCondPix output pixels
// per CTA
constexpr int kConvCinCondPix = 32;
void conv3x3_cin_cond_launch(int cin, const float* x, long long x_stride, const float* cond, long long cond_stride, int cond_mod,
                             int n, int H, int W, const float* w, const float* b, int Cout, float* y, Half2Ptr y16, cudaStream_t st);
// 3x3 pad 1, Cout <= 4, input NHWC fp32 with fused GroupNorm+SiLU; output NCHW fp32 [n,Cout,H,W];
// weights repacked [Cout][9][C] fp32. Returns the variant it launched: rows per CTA tile, channels per round, channel groups.
struct SmallCoutVariant {
  int th, ck, ks;
};
SmallCoutVariant conv3x3_small_cout_launch(const float* x, int n, int H, int W, int C, const double* sums, const float* gamma,
                                           const float* beta, float eps, const float* w_packed, const float* b, int Cout,
                                           float* y_nchw, cudaStream_t st);

// ---- time embedding (reference unet/mod.rs:19-30, 115-118, 718-722)
// emb = lin2(silu(lin1([cos|sin](t*f)))) ; then for every ResBlock r: e_r = lin_embed_r(silu(emb))
void time_embed_launch(const int* t_dev, const float* w1, const float* b1, const float* w2, const float* b2, float* hidden,
                       float* emb_silu, cudaStream_t st);
// the same at a real timestep (DESIGN §7 f15): at an integer t, the int overload's rows bit for bit
void time_embed_launch(const float* t_dev, const float* w1, const float* b1, const float* w2, const float* b2, float* hidden,
                       float* emb_silu, cudaStream_t st);
// the same for `rows` timesteps at once (t_dev[rows]); emb_all[t][n_all] is indexed by the timestep value. Bit-identical rows.
void time_embed_rows_launch(const int* t_dev, int rows, const float* w1, const float* b1, const float* w2, const float* b2,
                            const float* w_all, const float* b_all, int n_all, float* hidden, float* emb_silu, float* emb_all,
                            cudaStream_t st);
// real timesteps t_dev[rows] (the Karras grid): the rows of t_dev[j] go to emb_all[row_of[j]], bit-identical to time_embed_launch
// at t_dev[j]
void time_embed_rows_launch(const float* t_dev, const int* row_of, int rows, const float* w1, const float* b1, const float* w2,
                            const float* b2, const float* w_all, const float* b_all, int n_all, float* hidden, float* emb_silu,
                            float* emb_all, cudaStream_t st);
void emb_select_launch(const float* emb_all, const int* t_dev, int N, float* out, cudaStream_t st);
// y[N] = x[K] @ W[K][N] + b  (tiny GEMV, W fp32 [in,out])
void gemv_launch(const float* x, const float* W, const float* b, int K, int N, float* y, cudaStream_t st);

// ---- CLIP embedding lookup: x [n][Lp][D] = E[tok] + Pos, rows l >= L zero (reference clip/mod.rs:62-68)
void embed_tokens_launch(const int* tok, const float* E, const float* Pos, int n, int L, int Lp, int D, int vocab, float* x,
                         cudaStream_t st);

// ---- the sampler's fused guidance + update step (reference stablediffusion/mod.rs:152-156, 190-191; DESIGN §7 f5, f6, f7, f10)
// pred = u + (c-u)*scale ; x0 = (lat - pred*sqrt(1-a_t))/sqrt(a_t) ; lat' = x0*sqrt(a_prev) + pred*sqrt(1-a_prev) (STEP_DDIM)
enum : int { STEP_DDIM = 0, STEP_DDIM_ETA = 1, STEP_DPMPP_2M = 2 };
struct SamplerStep {   // per-step scalars, computed on the host in double and passed as f32
  float* hist = nullptr;      // STEP_DPMPP_2M: x0 of the previous step [count]; read when `second`, always overwritten
  float cx = 0.f, cd = 0.f;   // STEP_DPMPP_2M: x' = cx x + cd D
  float c1 = 0.f, c2 = 0.f;   // STEP_DPMPP_2M, second order: D = c1 x0 - c2 x0_prev
  int second = 0;
  float s = 0.f;              // STEP_DDIM_ETA: x' = sqrt(a_prev) x0 + dir_coef pred + s z
  uint32_t k0 = 0, k1 = 0;    // STEP_DDIM_ETA: key of z (step_noise_keys)
  float ka = 0.f, kb = 0.f;   // blend of the kinds other than STEP_DDIM: known = ka z0 + kb eps0 (sqrt(a_prev), sqrt(1 - a_prev))
  // per-sample inputs of a batch of different requests (DESIGN §7 f7). scales != null selects the per-sample instantiations:
  // sample s = i / (4 plane) takes scales[s] instead of `scale`, and STEP_DDIM_ETA draws z at the index within the sample,
  // keyed by step_noise_keys(noise_seeds[s], t) instead of (k0, k1). Any kind, STEP_DDIM included, may run per sample.
  const float* scales = nullptr;         // device [n]
  const uint64_t* noise_seeds = nullptr;  // device [n]
  int t = 0;  // the step's noise key (step_noise_keys): the timestep value (DDIM grid) or the index in the Karras grid
};
// One launch per step. groups = 2: eu / ec [count] the unconditional / prompt predictions, the update goes to both halves of
// lat [2][count]. groups = 3 (InstructPix2Pix): eu = eps [3][count] holds e_U | e_I | e_T (ec unused),
// pred = e_U + scale (e_T - e_I) + scale_i (e_I - e_U), and the update goes to all three copies in lat [3][count].
// w != null (masked img2img, two groups): lat' = w lat' + (1 - w) (sqrt(a_prev) z0 + sqrt(1 - a_prev) e0), w [n][plane].
struct CfgStepArgs {
  const float* eu = nullptr;
  const float* ec = nullptr;
  float* lat = nullptr;
  long long count = 0;
  float scale = 0.f;
  float sqrt_1m_at = 0.f, sqrt_at = 0.f, sqrt_aprev = 0.f, dir_coef = 0.f;
  const float* z0 = nullptr;
  const float* e0 = nullptr;
  const float* w = nullptr;
  int plane = 0;        // H * W of the latent
  SamplerStep s;
  float scale_i = 0.f;  // groups = 3: the image guidance scale
  int kind = STEP_DDIM;
  int groups = 2;
};
void cfg_step_launch(const CfgStepArgs& a, cudaStream_t st);
// ---- img2img staging: u8 HWC RGB [nb][Hp][Wp][3] -> encoder input [nb][4][Hp][Wp], v / 127.5 - 1, fourth plane zero
void u8_to_enc_input_launch(const uint8_t* rgb, int nb, int Hp, int Wp, float* out, cudaStream_t st);
// 9-channel inpainting: the masked image's encoder input [nb,4,Hp,Wp] and the latent mask into channel 0 of cond [nb,5,Hp/8,Wp/8]
void inpaint_prep_launch(const uint8_t* rgb, const uint8_t* mask, int nb, int Hp, int Wp, float* enc_in, float* cond,
                         cudaStream_t st);
// z0 [count] *= 0.18215 in place; xb[0..count) = xb[count..2count) = sa z0 + sb eps; mask (optional, u8 [n][8H][8W]) ->
// w [n][H][W] = 8x8 block sum / 16320
void img2img_prep_launch(float* z0, const float* eps, float* xb, long long count, float sa, float sb, const uint8_t* mask, float* w,
                         int H, int W, cudaStream_t st);
// pred = u + (c - u) * scale alone (forward_diffuser without the DDIM update)
void cfg_combine_launch(const float* eps_u, const float* eps_c, long long count, float scale, float* pred, cudaStream_t st);
// u8 = trunc(clamp((img+1)/2*255, 0, 255)), NCHW fp32 -> NHWC u8 (reference stablediffusion/mod.rs:79-97)
void to_rgb8_launch(const float* img_nchw, int n, int H, int W, uint8_t* rgb, cudaStream_t st);
void quant_conv_slice_launch(const float* x, const float* w, const float* b, int n, int HW, float* y, cudaStream_t st);
// the same, writing fl(y * scale) at sample stride y_stride (the inpainting conditioning tensor)
void quant_conv_slice_scaled_launch(const float* x, const float* w, const float* b, int n, int HW, long long y_stride, float scale,
                                    float* y, cudaStream_t st);
void add_vec_launch(const float* a, const float* b, int n, float* y, cudaStream_t st);
// N(0,1) latents from a Philox-like counter hash (used only when the caller passes no init latent)
void randn_launch(float* x, long long count, uint64_t seed, cudaStream_t st);
// Stochastic DDIM's per-step noise: the same generator keyed by (noise_seed, timestep value), element i of the call's latent
// (numpy mirror: synth.step_noise). step_noise_launch writes the stream the fused step draws in registers.
__host__ __device__ void step_noise_keys(uint64_t seed, int t, uint32_t* k0, uint32_t* k1);
void step_noise_launch(float* x, long long count, uint64_t seed, int t, cudaStream_t st);
// One seed per sample (DESIGN §7 f7): x [n][per], sample s is the stream randn_launch(seeds[s]) draws at n = 1, element j < per
// at index j. seeds: device [n]. At n = 1 it is randn_launch bit for bit.
void randn_seeds_launch(float* x, int n, long long per, const uint64_t* seeds, cudaStream_t st);
// The CFG context of a sampling call: out [2n][Lpad][768], samples [0, n) the unconditional rows, [n, 2n) the prompt rows.
// Row r of out sample b is copied when r < lens[b] (device [2n]: uncond lengths, then cond lengths) and zero otherwise, so the
// caller's pad rows are never read. cond [n][L][768]; uncond [n][Lu][768] with ustride = Lu * 768, or [Lu][768] with ustride 0
// (one negative broadcast over the batch). groups = 3 (InstructPix2Pix, DESIGN §7 f10): out [3n][Lpad][768], samples [0, 2n) the
// negative, [2n, 3n) the prompt rows; ustride must be 0 then.
void stage_cfg_context_launch(const float* cond, int L, const float* uncond, long long ustride, const int* lens, int n, int Lpad,
                              float* out, cudaStream_t st, int groups = 2);

// ---- row softmax for the 1-head VAE attention: P = softmax(S*scale) rows -> fp16 hi(/lo); cols <= kSoftmaxRowsMax. Returns the
// values per thread (PER) of the instance it launched.
constexpr int kSoftmaxRowsMax = 9216;
int softmax_rows_launch(const float* S, long long rows, int cols, float scale, Half2Ptr out, cudaStream_t st);

// ---- weight packing (master fp32 -> kernel layouts)
// conv OIHW [Cout][Cin][k][k] -> [Cout][k*k*Cin] with K index = tap*Cin + c ; fp16 hi (+lo)
void pack_conv_launch(const float* w, int Cout, int Cin, int ksize, Half2Ptr out, cudaStream_t st);
// nearest-2x-upsample folded 3x3 conv: 4 output phases x 2x2 taps, [4][Cout][4*Cin]
void pack_conv_up2_launch(const float* w, int Cout, int Cin, Half2Ptr out, cudaStream_t st);
// Linear [in][out] -> [out_row_offset + out][in] inside a packed matrix of row length ld (=in)
// ldw/col0 select a column slice [col0, col0+out) of a source matrix with row stride ldw (0 -> out)
// in_scale (optional, [in]): multiplies input feature i — a LayerNorm gamma folded into the consuming GEMM's weights
void pack_linear_launch(const float* w, int in, int out, Half2Ptr dst, int row_offset, cudaStream_t st, int ldw = 0,
                        int col0 = 0, const float* in_scale = nullptr);
// per-row sums of a packed fp16 matrix [rows][K]: s_hi = sum hi, s_full = sum (hi + lo); either output may be null
void rowsum_f16_launch(Half2Ptr m, int rows, int K, float* s_hi, float* s_full, cudaStream_t st);
// GEGLU proj [in][2*H4] -> rows interleaved per 2*half-tile: tile j holds x rows j*half.. then gate rows
void pack_geglu_launch(const float* w, const float* b, int in, int h4, int half_tile, Half2Ptr dst, float* bias_packed,
                       cudaStream_t st, const float* in_scale = nullptr);
// conv OIHW (Cout<=4, 3x3) -> fp32 [Cout][9][Cin]
void pack_small_cout_launch(const float* w, int Cout, int Cin, float* out, cudaStream_t st);

// ---- synthetic weights (bit-identical to stable_diffusion_burn_b200/synth.py)
void synth_fill_launch(float* dst, long long count, uint32_t key, float bound, float offset, cudaStream_t st);
struct SynthDesc {
  long long offset, count, chunk0;  // float offset in the arena, element count, index of the tensor's first 64K-element chunk
  uint32_t key;
  float bound, shift;
};
void synth_fill_table_launch(float* base, const SynthDesc* d_desc, int ntensors, long long nchunks, cudaStream_t st);

// ---- LoRA merge (DESIGN §7 f8): W_eff = W + sum_t s_t (up_t . down_t), every changed tensor in ONE launch.
// A tensor is stored [rows][cols]: a conv OIHW weight is [out][fan-in] (transposed = 0), a Linear weight of the registry is
// [in][out] (transposed = 1). up_t [out][r_t], down_t [r_t][fan-in]. Per element: d = fmaf(up[o][k], down[k][f], d) with k
// ascending from d = 0, tot = fmaf(s_t, d, tot) over the tensor's terms in table order from tot = 0, W_eff = W + tot (one rounding).
struct LoraTensorDesc {
  const float* base;
  float* out;
  int rows, cols, transposed;
  int term0, nterms;  // the tensor's terms: [term0, term0 + nterms) of the term table
  int tiles_c;        // 64-wide tiles along cols
  long long tile0;    // index of the tensor's first 64 x 64 tile (prefix sums over the table)
};
struct LoraTermDesc {
  const float* down;
  const float* up;
  int r;
  float s;
};
void lora_merge_launch(const LoraTensorDesc* d_tensors, int ntensors, const LoraTermDesc* d_terms, long long ntiles, cudaStream_t st);

}  // namespace sdb
