/*
 * sdb200.h — C ABI of the H100-native Stable Diffusion v1.4 sampling path.
 *
 * Drop-in boundary for the hot path of Gadersd/stable-diffusion-burn (reference @ 893fb095):
 * these entry points are what a Rust FFI shim binds in place of the Burn tensor graph in
 * src/backend.rs and src/model/{unet,attention,groupnorm,autoencoder}. Each function cites the
 * reference interface it replaces. The reference-side binding is shown in INTEGRATION.md and
 * rust/sdb200_ffi.rs.
 *
 * Conventions
 *  - every call returns int: 0 = ok, non-zero = error (text via sdb_last_error); nothing
 *    unwinds across the boundary (the reference panics / exit(1)s: src/bin/sample/main.rs:45-52).
 *  - tensors are contiguous row-major fp32, NCHW / [n, seq, C], exactly the reference's
 *    Tensor<B,4> / Tensor<B,3> contents. Caller owns every buffer; the library owns the context.
 *  - host-pointer calls are synchronous on return. *_dev variants take device pointers and a
 *    cudaStream_t (passed as void*) and are asynchronous on that stream.
 *  - a context is bound to one CUDA device and is not re-entrant (one in-flight call per ctx).
 *  - there is NO CPU fallback: every compute entry fails if the device path is unavailable.
 */
#ifndef SDB200_H
#define SDB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sdb_ctx sdb_ctx;

/* ---- lifetime ------------------------------------------------------------------------- */
/* Replaces device selection + StableDiffusionConfig::init (src/bin/sample/main.rs:59-83,
 * src/model/stablediffusion/mod.rs:22-39). */
int sdb_create(int device, sdb_ctx** out);
/* A context for an inpainting checkpoint (SD-1.5-inpainting and the like; DESIGN.md §7 f9). Its registry is sdb_create's except
 * unet/input_blocks/conv/weight, [320,9,3,3] (and its n_channels_in 9): the UNet reads cat(latent, latent mask, masked-image
 * latent). On such a context sdb_img2img[_dev] and sdb_img2img_batch[_dev] need the mask and condition the UNet on it with no
 * blend; sdb_unet_forward[_dev] and sdb_forward_diffuser[_dev] take x / latent [n,9,H,W] and return [n,4,H,W]; the text-to-image
 * entries fail (use sdb_img2img with an all-255 mask at strength 1). Loading a conv_in of another width fails. */
int sdb_create_inpaint(int device, sdb_ctx** out);
/* A context for an InstructPix2Pix checkpoint (timbrooks/instruct-pix2pix; DESIGN.md §7 f10). Its registry is sdb_create's except
 * unet/input_blocks/conv/weight, [320,8,3,3] (and its n_channels_in 8): the UNet reads cat(latent, image latent). Such a context
 * edits images with sdb_edit_image[_dev]; sdb_unet_forward[_dev] takes x [n,8,H,W] and returns [n,4,H,W]. The text-to-image
 * entries, sdb_img2img[_dev], the sdb_*_batch entries and sdb_forward_diffuser[_dev] (two-way guidance) fail, naming
 * sdb_edit_image. Loading a conv_in of another width fails. */
int sdb_create_pix2pix(int device, sdb_ctx** out);
int sdb_destroy(sdb_ctx* ctx);
/* ctx may be NULL: returns the last error of the calling thread (e.g. a failed sdb_create). */
const char* sdb_last_error(sdb_ctx* ctx);
/* "sdb200 <version> sm_90a" */
const char* sdb_version(void);

/* ---- weights -------------------------------------------------------------------------- */
/* Tensor registry. Names are the reference's dump-dir paths (src/model/unet/load.rs:213-306,
 * src/model/autoencoder/load.rs:16-198), e.g. "unet/input_blocks/rt1/res/conv_in/weight";
 * Linear weights are [in,out] and conv weights OIHW as in src/model/load.rs:65-160. The extra
 * tensor "alpha_cumulative_products" [1000] is the sampler's schedule Param
 * (src/model/stablediffusion/mod.rs:44). */
int sdb_tensor_count(sdb_ctx* ctx);
int sdb_tensor_info(sdb_ctx* ctx, int index, const char** name, int64_t dims[4], int* ndim);
/* Replaces load_tensor -> Param::from_tensor (src/model/load.rs:30-47). host: fp32, dims must match. */
int sdb_set_tensor(sdb_ctx* ctx, const char* name, const float* host, const int64_t* dims, int ndim);
/* Reads back the fp32 master copy (tests / checkpoint round trips). */
int sdb_get_tensor(sdb_ctx* ctx, const char* name, float* host, int64_t count);
/* load_stable_diffusion (src/model/stablediffusion/load.rs:16-33) for the part of the model on this path: reads every
 * registry tensor from the reference's dump-dir tree (1-D f32 .npy = [dims..., values...], python/save.py:10-15 <->
 * src/model/load.rs:17-47; <path>/<tensor name>.npy, the schedule from <path>/alphas_cumprod.npy). Optional files follow
 * the reference (missing Linear/Conv bias = none, missing GroupNorm weight/bias = ones/zeros); the configuration scalars
 * the reference reads (eps, n_group, stride, padding, n_head, n_layer, n_steps ...) are validated against the compiled
 * SD-v1.4 topology and each norm's eps is honoured. Encoder / quant_conv files are not read (not on the path). */
int sdb_load_dump_dir(sdb_ctx* ctx, const char* path);
/* load_tensor::<B, D> (src/model/load.rs:30-47) for one file, no context needed: splits the leading `ndim` shape values
 * from the data. Returns the element count (data may be NULL to probe), or -1 (text via sdb_last_error(NULL)). */
int64_t sdb_read_dump_tensor(const char* file, int ndim, int64_t* dims, float* data, int64_t capacity);
/* SD-1.x single-file .safetensors checkpoints in the original LDM layout (DESIGN.md §7 f13): v1-4, v1-5, the inpainting and
 * InstructPix2Pix releases and their fine-tunes. The key map is the one the reference's converter applies (load_state_dict into
 * python/dump.py:565-570's StableDiffusion, then python/stablediffusion.py:8-14's savers): model.diffusion_model.* -> unet/...,
 * first_stage_model.* -> autoencoder/..., cond_stage_model.transformer.text_model.* (or the older spelling without text_model.)
 * -> clip/..., alphas_cumprod -> alpha_cumulative_products (absent: the SD-1 scaled-linear schedule). Linear weights are
 * transposed to the registry's [in,out] (python/save.py:17-21), everything else is copied; F32, F16 and BF16 (mixed within a
 * file) are widened exactly to fp32. Keys outside the model prefixes (model_ema.*, betas, ...), first_stage_model.loss.* and
 * the CLIP position_ids are not read.
 * A full checkpoint must hold every registry tensor; a VAE-only file (the standalone SD VAE releases: encoder.*, decoder.*,
 * quant_conv.*, post_quant_conv.*) replaces exactly the autoencoder/... tensors, on any kind of context. The whole file (header,
 * keys, shapes, dtypes, byte ranges, a conv_in width that fits the context) is validated before the first weight is written,
 * so a rejected file leaves the context as it was. Afterwards, as after sdb_load_dump_dir: call sdb_finalize_weights; every
 * loaded norm uses the default eps; LoRA adapters are kept and merged onto the new weights by that finalize. */
int sdb_load_safetensors(sdb_ctx* ctx, const char* path);
#define SDB_CKPT_FULL 0
#define SDB_CKPT_VAE 1
/* The validation of sdb_load_safetensors without a context or a device, reading no tensor data: kind = SDB_CKPT_FULL or
 * SDB_CKPT_VAE, conv_in_width = 4, 8 or 9 (the context to create: sdb_create, sdb_create_pix2pix, sdb_create_inpaint), 0 for a
 * VAE-only file. Either pointer may be NULL. Errors via sdb_last_error(NULL). */
int sdb_probe_safetensors(const char* path, int* kind, int* conv_in_width);
/* Fills every tensor with the deterministic synthetic stream documented in
 * stable_diffusion_burn_b200/synth.py (bit-identical to the numpy generator). */
int sdb_init_synthetic(sdb_ctx* ctx, uint32_t seed);
/* fp32 master arena (device pointer, bytes): one contiguous block holding every tensor, for the
 * single init-time ncclBroadcast from rank 0 (SURVEY §8e). */
int sdb_weight_arena(sdb_ctx* ctx, void** dev_ptr, size_t* bytes);
/* Multi-GPU init (SURVEY §8b(2), §8e): the ONE collective of the path. Rank 0 obtains an id with sdb_nccl_unique_id (128 bytes,
 * = ncclUniqueId) and hands it to every rank by its own means (file, socket, MPI, torch store); then every rank calls
 * sdb_broadcast_weights(ctx, id, rank, world): ncclCommInitRank + ncclBroadcast of the fp32 master arena (and of the per-norm
 * eps table a dump-dir carries) from rank 0 over NVLink, then the communicator is destroyed — no collective on the sampling
 * path. NCCL is resolved with dlopen("libnccl.so.2") at the first call: single-GPU hosts need no NCCL. world == 1 is a no-op.
 * Call sdb_finalize_weights afterwards on every rank. */
int sdb_nccl_unique_id(void* id128);
int sdb_broadcast_weights(sdb_ctx* ctx, const void* id128, int rank, int world);
/* Packs the master weights into kernel layouts (fp16 K-major tiles, fused QKV/GEGLU orders).
 * Must be called after the last sdb_set_tensor / broadcast and before any compute call. */
int sdb_finalize_weights(sdb_ctx* ctx);

/* ---- hot path, host buffers -------------------------------------------------------------- */
/* UNet::forward (src/model/unet/mod.rs:109-142): x [n,4,H,W], one timestep for the batch,
 * context [n,L,768] -> out [n,4,H,W]. */
int sdb_unet_forward(sdb_ctx* ctx, const float* x, int32_t timestep, const float* context,
                     int n, int H, int W, int L, float* out);
/* sdb_unet_forward at a real timestep t (DESIGN.md §7 f15), for callers that drive their own sampler on a grid of fractional
 * timesteps: t finite and in [0, 999], rounded once to f32 for the sinusoidal embedding. At an integer t the output equals
 * sdb_unet_forward's bit for bit. */
int sdb_unet_forward_at(sdb_ctx* ctx, const float* x, double t, const float* context, int n, int H, int W, int L, float* out);
/* Autoencoder::decode_latent (src/model/autoencoder/mod.rs:68-71): latent [n,4,H,W] -> img [n,3,8H,8W]. */
int sdb_decode_latent(sdb_ctx* ctx, const float* latent, int n, int H, int W, float* img);
/* StableDiffusion::sample_latent (src/model/stablediffusion/mod.rs:102-160), DDIM eta=0 (the default sampler; see
 * sdb_set_sampler) with classifier-free guidance (forward_diffuser :162-192). context [n,L,768]; uncond [Lu,768] is
 * broadcast over the batch. init_latent [n,4,H,W] (the reference draws it from an unseeded RNG,
 * :115-121); if NULL an internal Philox N(0,1) stream keyed by `seed` is used. */
int sdb_sample_latent(sdb_ctx* ctx, const float* context, int n, int L, const float* uncond, int Lu,
                      double guidance_scale, int n_steps, const float* init_latent, uint64_t seed,
                      int H, int W, float* latent_out);
/* StableDiffusion::forward_diffuser (src/model/stablediffusion/mod.rs:162-192): classifier-free guidance at one timestep,
 * pred = u + (c - u) * scale with u = UNet(latent, t, uncond broadcast over the batch), c = UNet(latent, t, context) — evaluated
 * as ONE batch-2n UNet pass (the pass sample_latent replays per step). latent [n,4,H,W]; pred / out_uncond / out_cond [n,4,H,W],
 * each may be NULL (out_uncond / out_cond expose the two UNet outputs before the combine, for per-step parity checks). */
int sdb_forward_diffuser(sdb_ctx* ctx, const float* latent, int32_t timestep, const float* context, int n, int L,
                         const float* uncond, int Lu, double guidance_scale, int H, int W, float* pred,
                         float* out_uncond, float* out_cond);
/* StableDiffusion::latent_to_image (src/model/stablediffusion/mod.rs:69-100): decode(latent/0.18215),
 * (x+1)/2*255, NHWC, clamp to [0,255], truncate to u8. rgb [n,8H,8W,3]. */
int sdb_latent_to_image(sdb_ctx* ctx, const float* latent, int n, int H, int W, uint8_t* rgb);
/* StableDiffusion::sample_image (src/model/stablediffusion/mod.rs:51-67) = sample_latent + latent_to_image. */
int sdb_sample_image(sdb_ctx* ctx, const float* context, int n, int L, const float* uncond, int Lu,
                     double guidance_scale, int n_steps, const float* init_latent, uint64_t seed,
                     int H, int W, uint8_t* rgb);

/* ---- text encoder (SURVEY §8f row f1: the first "next" row after the hot path) ------------------ */
/* CLIP::forward (src/model/clip/mod.rs:56-75): token ids [n,L] (L <= 77, NOT padded — the reference does not pad,
 * src/model/stablediffusion/mod.rs:198-211) -> context [n,L,768]. The ids come from SimpleTokenizer::encode
 * (src/tokenizer.rs:175-195), mirrored host-side in stable_diffusion_burn_b200/tokenizer.py. */
int sdb_clip_forward(sdb_ctx* ctx, const int32_t* tokens, int n, int L, float* out);
/* device-pointer variant: ids outside [0,49408) are clamped (the host variant rejects them). */
int sdb_clip_forward_dev(sdb_ctx* ctx, const int32_t* d_tokens, int n, int L, float* d_out, void* stream);

/* ---- VAE encoder (SURVEY §8f row f4) ---------------------------------------------------------------- */
/* Autoencoder::encode_image (src/model/autoencoder/mod.rs:60-66): img [n,3,H,W] -> latent [n,4,H/8,W/8] = the first four
 * channels of quant_conv(encoder(img)). H, W multiples of 8 (>= 64). Only img2img needs it; the reference CLI never calls it. */
int sdb_encode_image(sdb_ctx* ctx, const float* img, int n, int H, int W, float* latent);
int sdb_encode_image_dev(sdb_ctx* ctx, const float* d_img, int n, int H, int W, float* d_latent, void* stream);

/* ---- image-to-image / masked inpainting (DESIGN.md §7 f5) -------------------------------------------------------------- */
/* The reference has no img2img; this is built from its own parts: encode_image (src/model/autoencoder/mod.rs:60-66), the latent
 * scale 0.18215 of latent_to_image (src/model/stablediffusion/mod.rs:71) and the schedule and DDIM step of sample_latent (:111,
 * :123-156). image u8 [n,8H,8W,3] HWC RGB (the format sdb_sample_image returns) -> x = v/127.5 - 1 -> z0 = 0.18215 *
 * encode_image(x). Of the N timesteps (0..1000).rev().step_by(1000/n_steps), the last k = floor(strength * N) run, from
 * t0 = ts[N-k], on the start latent sqrt(abar[t0]) z0 + sqrt(1 - abar[t0]) noise. strength must be finite, in (0, 1], and give
 * k >= 1 (strength >= 1/N). mask (optional) u8 [n,8H,8W]: 255 = regenerate, 0 = keep, in between blends; it is reduced to one
 * weight per latent cell, w = (sum of the 8x8 block) / (64*255), and after every step x = w x + (1-w) (sqrt(a_prev) z0 +
 * sqrt(1 - a_prev) noise), so the kept region ends as exactly z0. noise [n,4,H,W]; NULL = the N(0,1) stream keyed by `seed`
 * that sdb_sample_image starts from. Outputs: latent_out [n,4,H,W] and / or rgb_out [n,8H,8W,3]; at least one must be set.
 * H, W are latent sizes with the constraints of sampling (multiples of 8, (H/8)*(W/8) a multiple of 8).
 * On a 9-channel context (sdb_create_inpaint; DESIGN.md §7 f9) the mask is required and binary, m = (mask >= 128); the masked
 * image x_m = m ? 0 : x gives z_m = 0.18215 * encode_image(x_m), the latent mask is the nearest pick m[8h][8w], and both CFG
 * halves of every UNet pass read cat(x_t, latent mask, z_m). The start latent and the strength rule are the above, z0 from the
 * unmasked image; each step is the sampler's update with no blend. */
int sdb_img2img(sdb_ctx* ctx, const uint8_t* image, const uint8_t* mask, double strength, const float* context, int n, int L,
                const float* uncond, int Lu, double guidance_scale, int n_steps, const float* noise, uint64_t seed, int H, int W,
                float* latent_out, uint8_t* rgb_out);
/* device-pointer variant: d_noise is required (as d_init_latent is for sdb_sample_image_dev). */
int sdb_img2img_dev(sdb_ctx* ctx, const uint8_t* d_image, const uint8_t* d_mask, double strength, const float* d_context, int n,
                    int L, const float* d_uncond, int Lu, double guidance_scale, int n_steps, const float* d_noise, int H, int W,
                    float* d_latent_out, uint8_t* d_rgb_out, void* stream);

/* ---- InstructPix2Pix image editing (DESIGN.md §7 f10) ------------------------------------------------------------------ */
/* Edits n images by instruction on an 8-channel context (sdb_create_pix2pix), as the original edit_cli.py and diffusers'
 * StableDiffusionInstructPix2PixPipeline do. image u8 [n,8H,8W,3] HWC RGB -> x = v/127.5 - 1 -> the image latent
 * c_I = encode_image(x), UNSCALED (the posterior mode; no 0.18215). Sampling runs the full schedule from t = 999 (no strength)
 * on init_latent [n,4,H,W]; NULL = the N(0,1) stream keyed by `seed` that sdb_sample_image starts from. Each step is one
 * batch-3n UNet pass over the groups, in this order,
 *   e_U = UNet(cat(x_t, 0), t, uncond)   e_I = UNet(cat(x_t, c_I), t, uncond)   e_T = UNet(cat(x_t, c_I), t, context)
 * combined as pred = e_U + text_scale (e_T - e_I) + image_scale (e_I - e_U) (both finite; all three passes always run), then
 * the context's sampler (sdb_set_sampler) updates the latent with no blend. context [n,L,768]; uncond [Lu,768], one negative
 * broadcast over the batch. Outputs: latent_out [n,4,H,W] and / or rgb_out [n,8H,8W,3]; at least one must be set. H, W are
 * latent sizes with the constraints of sampling. Fails on a 4- or 9-channel context, naming sdb_create_pix2pix. */
int sdb_edit_image(sdb_ctx* ctx, const uint8_t* image, const float* context, int n, int L, const float* uncond, int Lu,
                   double text_scale, double image_scale, int n_steps, const float* init_latent, uint64_t seed, int H, int W,
                   float* latent_out, uint8_t* rgb_out);
/* device-pointer variant: d_init_latent is required; runs ordered after, and before the rest of, `stream`. */
int sdb_edit_image_dev(sdb_ctx* ctx, const uint8_t* d_image, const float* d_context, int n, int L, const float* d_uncond, int Lu,
                       double text_scale, double image_scale, int n_steps, const float* d_init_latent, int H, int W,
                       float* d_latent_out, uint8_t* d_rgb_out, void* stream);

/* ---- sampler (DESIGN.md §7 f6) ------------------------------------------------------------------------------------------ */
/* The reference samples with DDIM at eta = 0 only (src/model/stablediffusion/mod.rs:119, sigma = 0). The sampler is context
 * state, read by sdb_sample_latent, sdb_sample_image, sdb_sample_image_dev, sdb_img2img[_dev] and sdb_edit_image[_dev] (not by
 * sdb_forward_diffuser or sdb_unet_forward); the schedule, the UNet step and the decode are the same for every sampler.
 * SDB_SAMPLER_DDIM with eta in [0, 1] (finite): DDIM (Song et al. 2021, eq. 16), s = eta sqrt((1-a')/(1-a)) sqrt(1 - a/a'),
 *   x' = sqrt(a') x0 + sqrt(1 - a' - s^2) eps + s z. eta = 0 (the default) is the reference's sampler, unchanged to the bit.
 *   z is N(0,1) keyed by (noise_seed, timestep value, element index in the call's [n,4,H,W] latent): a batch member's noise
 *   depends on its position in the call (the sdb_*_batch entries key it per sample instead).
 * SDB_SAMPLER_DPMPP_2M (eta must be 0): DPM-Solver++(2M) (Lu et al. 2022), data prediction, second order from the second step
 *   a call runs; the final step returns x0. A context starts with (SDB_SAMPLER_DDIM, 0.0, 0). Invalid arguments are an error
 *   and leave the setting unchanged. */
#define SDB_SAMPLER_DDIM 0
#define SDB_SAMPLER_DPMPP_2M 1
int sdb_set_sampler(sdb_ctx* ctx, int kind, double eta, uint64_t noise_seed);
/* The grid the sampler walks (DESIGN.md §7 f15), context state read by exactly the entries that read sdb_set_sampler. N = n_steps.
 * SDB_SCHEDULE_DDIM (the default): the reference's timesteps (0..1000).rev().step_by(1000/n_steps), abar = alpha_cumulative_products[t].
 * SDB_SCHEDULE_KARRAS: the sigma grid of Karras et al. 2022 (rho = 7; k-diffusion's get_sigmas_karras) between sigma_max =
 *   sigma_999 and sigma_min = sigma_0 of the table sigma_j = sqrt((1 - abar_j) / abar_j): sigma_i = (sigma_max^(1/7) + i/(N-1)
 *   (sigma_min^(1/7) - sigma_max^(1/7)))^7, i < N, then sigma_N = 0. Step i evaluates the UNet at the real timestep
 *   t_i = sigma_to_t(sigma_i) (k-diffusion's: linear in log sigma between table neighbours, rounded once to f32) and runs the
 *   sampler's update from abar_i = 1/(1 + sigma_i^2) to abar_{i+1} (1 after the last step). In k-diffusion's terms: DDIM eta = 0
 *   is sample_euler, DDIM eta is sample_euler_ancestral(eta), DPM-Solver++(2M) is sample_dpmpp_2m. The latent is the library's
 *   x = sqrt(abar) x0 + sqrt(1 - abar) eps throughout: the start latent is used as is (diffusers' init_noise_sigma
 *   convention). img2img runs the last floor(strength * N) steps; eta noise is keyed by the step's index i in the grid instead of
 *   the timestep value. Every call checks that alpha_cumulative_products is finite, in (0, 1) and strictly decreasing.
 * An unknown kind is an error and leaves the setting unchanged. No cached graph is invalidated. */
#define SDB_SCHEDULE_DDIM 0
#define SDB_SCHEDULE_KARRAS 1
int sdb_set_schedule(sdb_ctx* ctx, int kind);

/* ---- LoRA adapters (DESIGN.md §7 f8) ------------------------------------------------------------------------------------- */
/* An adapter (id >= 0) is a set of terms; a term targets one registry weight with down [r][fan-in] (fan-in = in for a Linear,
 * in*k*k in OIHW order for a conv), up [out][r] and alpha (kohya lora_down / lora_up, PEFT lora_A / lora_B). The weights the
 * packers read are W_eff = W + sum over adapters (ascending id) and their terms (in the order added) of s (up . down), with
 * s = (float)(multiplier * alpha / r) computed in double; for a Linear the registry holds [in][out], so the delta is added
 * transposed. Per element, each term's dot product runs in fp32 FMAs with k ascending, terms accumulate as tot = fmaf(s, d, tot)
 * from 0, and W_eff = W + tot rounded once: with dyadic factors and power-of-two scales every step is exact.
 * Targets: UNet ResBlock conv_in / conv_out / skip_connection / lin_embed, the down- and upsample convs, SpatialTransformer
 * proj_in / proj_out, attn1 / attn2 query / key / value / out, mlp/geglu/proj and mlp/lin, and CLIP attn/{query,key,value,out}
 * and mlp/fc1 / fc2. Norms, biases, embeddings, the VAE, unet/input_blocks/conv, unet/lin{1,2}_time_embed and unet/conv_out
 * are rejected. The master arena stays the base (sdb_get_tensor returns base weights); adapters are per context (the weight
 * broadcast carries the base only) and survive sdb_set_tensor, sdb_load_dump_dir, sdb_broadcast_weights and
 * sdb_finalize_weights, which packs base + active adapters. Every change is pending until sdb_lora_apply (or a finalize); a
 * compute call with pending changes fails. A malformed argument is rejected, naming the field and value, before any state
 * changes. All adapters of a context apply to every sample of a batch. */
/* Copies the factors of one term to the device. Rejects an unknown or non-target tensor, rank < 1, a NULL factor, a non-finite
 * or non-positive alpha and a second term for the same (adapter, tensor). A new adapter starts at multiplier 1. */
int sdb_lora_add(sdb_ctx* ctx, int adapter, const char* tensor, int rank, const float* down, const float* up, double alpha);
/* multiplier (finite) of an existing adapter; 0 disables it without freeing its factors */
int sdb_lora_scale(sdb_ctx* ctx, int adapter, double multiplier);
/* removes one adapter (-1 = all) and frees its device factors */
int sdb_lora_remove(sdb_ctx* ctx, int adapter);
/* Synchronous. One merge launch writes W_eff of every weight whose active terms changed since the last apply or finalize; the
 * packing unit of each (a ResBlock, a SpatialTransformer with its LayerNorm folds, a resample conv, the time-embedding table,
 * a CLIP block with its folded out-projection bias) is re-packed into its own packed addresses and nothing else is touched.
 * Cached step graphs stay valid. With no active term a weight packs from the base tensor itself, so removing every adapter and
 * applying restores the base packing bit for bit. */
int sdb_lora_apply(sdb_ctx* ctx);
/* W_eff of a registry tensor as the packers read it after the last apply or finalize (the base tensor when no active term
 * targets it); host buffer of count elements. */
int sdb_get_merged_tensor(sdb_ctx* ctx, const char* tensor, float* host, int64_t count);

/* ---- batches of different requests (DESIGN.md §7 f7) --------------------------------------------------------------------- */
/* One call samples n requests that differ in prompt length, negative prompt, guidance scale and seed, as one batch-2n UNet pass
 * per step (the weights stream from HBM once per step for all of them). Sample i gives what request i gives as a call of its
 * own at n = 1: its own context_len[i] prompt rows and uncond_len[i] negative rows (rows past a length are never read, so the
 * caller's pad rows may hold anything), its own scale (cast to float), the init latent / img2img noise sdb_sample_image draws
 * for seed[i] at n = 1, and stochastic-DDIM noise keyed by (noise_seed[i], timestep, element index within the sample). It
 * matches that single call to rounding: split-K choices of the UNet's GEMMs depend on the batch size. The sampler
 * (sdb_set_sampler), n_steps, strength, H and W hold for the whole call. The context is padded to the longest length any
 * sample reads, rounded up to 32, whatever the strides L and Lu: a generous stride costs nothing.
 * Errors (the field, the sample index and the value are named; nothing is changed): n < 1, L or Lu < 1, a length outside
 * [1, stride], a non-finite scale, a NULL context / uncond / guidance_scale, a NULL seed when no init latent / noise is given. */
typedef struct sdb_batch {
  int n;
  int L;                           /* row stride of context */
  const float* context;            /* [n][L][768] */
  const int32_t* context_len;      /* [n]: sample i reads rows [0, context_len[i]); NULL = L for every sample */
  int Lu;                          /* row stride of uncond */
  const float* uncond;             /* [n][Lu][768]: one negative / unconditional context per sample */
  const int32_t* uncond_len;       /* [n]; NULL = Lu for every sample */
  const double* guidance_scale;    /* [n], finite */
  const uint64_t* seed;            /* [n]: init latent (txt2img) / noise (img2img) of sample i; unused with an explicit one */
  const uint64_t* noise_seed;      /* [n]: stochastic-DDIM step noise of sample i; NULL = the sdb_set_sampler noise_seed */
} sdb_batch;
/* sdb_sample_latent / sdb_sample_image over a batch. init_latent [n,4,H,W] or NULL (= from the seeds). latent_out [n,4,H,W]
 * and / or rgb_out [n,8H,8W,3]; at least one must be set. */
int sdb_sample_batch(sdb_ctx* ctx, const sdb_batch* batch, int n_steps, const float* init_latent, int H, int W,
                     float* latent_out, uint8_t* rgb_out);
/* sdb_img2img over a batch: image u8 [n,8H,8W,3], mask u8 [n,8H,8W] or NULL, noise [n,4,H,W] or NULL (= from the seeds). */
int sdb_img2img_batch(sdb_ctx* ctx, const sdb_batch* batch, const uint8_t* image, const uint8_t* mask, double strength,
                      int n_steps, const float* noise, int H, int W, float* latent_out, uint8_t* rgb_out);
/* device-pointer variants: context, uncond, image, mask, init latent / noise and the outputs are device buffers; the lengths,
 * scales and seeds stay host arrays. Asynchronous on `stream`. */
int sdb_sample_batch_dev(sdb_ctx* ctx, const sdb_batch* batch, int n_steps, const float* d_init_latent, int H, int W,
                         float* d_latent_out, uint8_t* d_rgb_out, void* stream);
int sdb_img2img_batch_dev(sdb_ctx* ctx, const sdb_batch* batch, const uint8_t* d_image, const uint8_t* d_mask, double strength,
                          int n_steps, const float* d_noise, int H, int W, float* d_latent_out, uint8_t* d_rgb_out, void* stream);

/* ---- hot path, device buffers (zero-copy callers) ------------------------------------------ */
int sdb_unet_forward_dev(sdb_ctx* ctx, const float* d_x, int32_t timestep, const float* d_context,
                         int n, int H, int W, int L, float* d_out, void* stream);
int sdb_decode_latent_dev(sdb_ctx* ctx, const float* d_latent, int n, int H, int W, float* d_img, void* stream);
int sdb_forward_diffuser_dev(sdb_ctx* ctx, const float* d_latent, int32_t timestep, const float* d_context, int n, int L,
                             const float* d_uncond, int Lu, double guidance_scale, int H, int W, float* d_pred, void* stream);
int sdb_sample_image_dev(sdb_ctx* ctx, const float* d_context, int n, int L, const float* d_uncond, int Lu,
                         double guidance_scale, int n_steps, const float* d_init_latent,
                         int H, int W, uint8_t* d_rgb, void* stream);

/* ---- configuration / instrumentation ------------------------------------------------------- */
/* Run configurations: "precision" = 1|2|3 tensor-core passes per product (0 = the per-layer policy, DESIGN.md), "graphs" = 0|1
 * (CUDA-graph replay of the UNet step), "splitk" = 0|1, "emb_hoist" = 0|1 (0: per-step time-embedding GEMVs, as sdb_unet_forward
 * runs them). Test hooks (default 1; 0 selects a path production takes elsewhere): "raw16" (prep_operand staging, as for the
 * stride-2 convs), "skip_merge" (the 1x1 skip conv as its own GEMM, as in the VAE encoder), "gn_epilogue" (the fused GroupNorm,
 * as behind the Cin = 4 convs), "attn_split" (fp16 q / k at d = 40 / 80; no production call takes it). Unknown keys: error. */
int sdb_set_option(sdb_ctx* ctx, const char* key, int value);
/* Per-kernel-class timing: when enabled, every launch is bracketed by CUDA events on the
 * context's stream (graphs are bypassed). */
int sdb_profile_enable(sdb_ctx* ctx, int on);
int sdb_profile_reset(sdb_ctx* ctx);
int sdb_profile_class_count(sdb_ctx* ctx);
/* launches, total device milliseconds, algorithmic FLOPs and bytes of one kernel class. */
int sdb_profile_get(sdb_ctx* ctx, int cls, const char** name, int64_t* launches, double* ms,
                    double* flops, double* bytes);
/* tensor-core FLOPs actually issued by a class (x2 / x3 of the algorithmic count where the split-fp16 product runs). */
int sdb_profile_get_issued(sdb_ctx* ctx, int cls, double* issued_flops);
/* Number of kernel launches issued by this context since creation (sdb_profile_reset zeroes it). */
int64_t sdb_launch_count(sdb_ctx* ctx);

/* ---- unit-test entry points for single kernels (host pointers) ------------------------------- */
/* The test entries that take a trailing `trace` accept NULL, or SDB_TRACE_INTS ints that receive a record of every launch of
 * the call whose choice a test asserts, in launch order: [0] the record count, then 16 ints per record from [1], a kind tag and
 * its fields, zero-padded. A call whose records do not fit fails with an error naming the count; nothing is truncated. Kinds:
 *   1 GEMM: kind (0 Linear, 1 1x1 conv, 2 3x3 conv, 3 stride 2, 4 folded nearest-2x, 5 stride 2 padded bottom/right), N, BN,
 *     split-K, TN, TH, TW, extra-K channels, GroupNorm slots written, second-source channels, passes, epilogue roles (1
 *     LayerNorm statistics, 2 LayerNorm-consuming, 4 GEGLU, 8 fp16-pair residual, 16 fp32 residual, 32 GroupNorm partials),
 *     activation (1 QuickGELU), pipeline stages of the kernel instance
 *   2 fused attention: dpad, Nq, Nk, split q / k (hi + lo), per-sample lengths, causal
 *   3 GroupNorm staging: its path (1 fused statistics + apply, 2 apply from producer partials, 3 apply after the 64:1 pre-fold;
 *     sums for the fused GroupNorm + small-Cout conv: 4 by the statistics kernel, 5 from producer partials, 6 after the pre-fold)
 *   4 fused GroupNorm + small-Cout conv: rows per tile, channels per round, channel groups
 *   5 autoencoder attention row softmax: values per thread
 *   6 conditioned UNet conv_in: m, sample s reads the conditioning of sample s % m */
#define SDB_TRACE_INTS 1024
/* The GEMM as the Linear layers use it, and its other epilogues and K-loop forms, each reachable in isolation: out = A[M,K]
 * (fp32, rounded to the operand format) x W[K,N] (fp32 [in,out]) (+ bias) (+ residual[M,N]) (+ XA[M,XK] x XW[XK,N], the
 * "extra K" operands the ResBlock skip conv rides on). flags: 0 = the plain Linear product, fp32 out; 1 = GEGLU (W = [K][x |
 * gate], out [M, N/2] = (x + b_x) * gelu_erf(gate + b_g), unet/mod.rs:578-592); 4 = read the result back from the fp16 hi + lo
 * outputs;
 * 8 (with 4) = return the two fp16 planes separately: out = [2][M][N (or N/2)], hi then lo, each value converted to float.
 * Split-K is chosen by the library's own policy (small M x N grid, long K). */
int sdb_test_gemm_ex(sdb_ctx* ctx, const float* a, const float* w, const float* bias, const float* residual, int M, int K,
                     int N, int passes, int flags, const float* xa, const float* xw, int XK, float* out, int32_t* trace);
/* conv2d NCHW fp32 in/out through the implicit-GEMM path as the model runs it (its operand staging, weight packing and GEMM
 * kinds): 1x1, 3x3 pad 1, 3x3 stride 2 (ksize 3: the UNet downsample), or upsample = 1 (ksize 3): nearest 2x upsample folded
 * into the weights. cin a multiple of 64, cout of 32; any other stride / upsample combination is an error. */
int sdb_test_conv2d(sdb_ctx* ctx, const float* x, const float* w, const float* bias, int n, int cin, int H,
                    int W, int cout, int ksize, int stride, int upsample, int passes, float* y, int32_t* trace);
/* The LayerNorm-free TransformerBlock chain in isolation (unet/mod.rs:521-527): y = a w0 + b0 (+ a2 w0 + b0 accumulated in place
 * on the fp16 hi/lo residual pair; a2 may be NULL) with row statistics from the producing epilogue, then
 * out = LayerNorm(y; gamma, beta) w1 + b1 with the LayerNorm folded into the consuming GEMM (gamma in the weights, rank-1
 * correction in the epilogue); geglu = 1: w1 = [C][x | gate], out [M, N/2] = x * gelu(gate). C a multiple of 160. */
int sdb_test_ln_fold(sdb_ctx* ctx, const float* a, const float* a2, const float* w0, const float* b0, const float* gamma,
                     const float* beta, const float* w1, const float* b1, int M, int K0, int C, int N, int passes, int geglu,
                     float* out, int32_t* trace);
/* The conv of sdb_test_conv2d whose epilogue also leaves the GroupNorm statistics of its output, in the partial buffer the
 * model gives an activation of that width, followed by the apply-only GroupNorm(+SiLU) that consumes them (the ResBlock's
 * conv_in -> norm_out -> SiLU chain, unet/mod.rs:716-725). NCHW fp32 in/out; *slots = partial-statistics slots per image the
 * GEMM wrote. With the gn_epilogue option at 0 the model leaves no statistics, and the call fails with "the GEMM did not
 * produce GroupNorm statistics for this shape" (*slots = 0). */
int sdb_test_conv_groupnorm(sdb_ctx* ctx, const float* x, const float* w, const float* bias, const float* gamma,
                            const float* beta, int n, int cin, int H, int W, int cout, int ksize, int stride, int upsample,
                            int passes, int silu, float* y, int* slots, int32_t* trace);
/* LayerNorm over the last dim, [rows, c]. */
int sdb_test_layernorm(sdb_ctx* ctx, const float* x, const float* gamma, const float* beta, int rows, int c,
                       float* y);
/* qkv_attention (src/model/attention.rs:5-45): q [n,Nq,C], k,v [n,Nk,C], heads -> out [n,Nq,C].
 * kvlen: host array [n], sample s attends to its first kvlen[s] keys (each in [1, Nk], else an error); NULL = Nk for all.
 * flags: 1 = causal mask (key j visible to query i only if j <= i; Nk <= 128), 2 = V transposed, staged as the CLIP encoder
 * stages it (q / k as single fp16 values in one matrix, V^T; needs Nq == Nk and C / heads a multiple of 16). */
int sdb_test_attention(sdb_ctx* ctx, const float* q, const float* k, const float* v, int n, int Nq, int Nk,
                       int C, int heads, const int32_t* kvlen, int flags, float* out);
/* One UNet ResBlock (unet/mod.rs:712-734) or, with emb_bias = NULL, VAE ResnetBlock (autoencoder/mod.rs:513-528) on
 * cat([x0, x1]) (x1 NULL when c1 = 0), through the model's own staging, packing and launch choices. Host NCHW fp32 tensors;
 * weights OIHW; skip_w [cout][c0 + c1][1][1] or NULL (then x0 is added and c0 must equal cout); emb_bias [cout] replaces conv1's
 * bias (the model passes conv_in.bias + lin_embed(silu(emb))). flags: 1 / 2 = x0 / x1 are written by a producer that leaves
 * GroupNorm statistics (a 3-pass identity conv: the block then sees hi + lo of the input, 22 bits); otherwise an fp32 tensor
 * with an fp16 copy and no statistics. Outputs [n][cout][H][W]: out, out16 = its fp16 hi + lo copy (zero without the raw16
 * option), out_norm = SiLU(GroupNorm(out; norm2)) staged from the statistics conv2 left. trace: NULL or SDB_TRACE_INTS ints (see
 * above). */
int sdb_test_resblock(sdb_ctx* ctx, const float* x0, const float* x1, int n, int c0, int c1, int H, int W, int cout,
                      const float* norm1_g, const float* norm1_b, const float* conv1_w, const float* conv1_b, const float* norm2_g,
                      const float* norm2_b, const float* conv2_w, const float* conv2_b, const float* skip_w, const float* skip_b,
                      const float* emb_bias, int passes, int flags, float* out, float* out16, float* out_norm, int32_t* trace);
/* GroupNorm(32 groups)(+SiLU) of cat([x0, x1]) (x1 NULL when c1 = 0) as an fp16 hi + lo operand, returned NCHW as hi + lo.
 * mode 1: the fused statistics + apply kernel; 2: apply from the partials the producers left (3-pass identity convs, which
 * pass hi + lo of the inputs), with the 64:1 pre-fold above 128 slots per image. Any other mode is an error.
 * trace: NULL or SDB_TRACE_INTS ints (see above). */
int sdb_test_groupnorm_cat(sdb_ctx* ctx, const float* x0, const float* x1, int n, int c0, int c1, int H, int W,
                           const float* gamma, const float* beta, int silu, int mode, float* y, int32_t* trace);
/* One of the UNet's 16 SpatialTransformers (unet/mod.rs:461-481), index = its position in execution order (0..5 input blocks,
 * 6 middle block, 7..15 output blocks), run on the weights sdb_finalize_weights packed, with the model's own launch sequence.
 * Needs finalized weights. x [n][c][H][W] (c must be the block's width; H * W a multiple of 8) is staged as a ResBlock leaves it (a
 * 3-pass identity conv: the block sees hi + lo of x, with GroupNorm partials). context [n][lmax][768] with per-sample lengths
 * lens[n] in [1, lmax] goes through the context K/V preparation of the sampling entries (zero padded to a multiple of 32).
 * flags: 1 = the output carries an fp16 hi + lo copy (else out16 is zero). Outputs: out, out16 [n][C][H][W]; out_norm =
 * SiLU(GroupNorm(out; the block's own norm)) staged the way the next ResBlock stages its input; taps_y [4][n*H*W][C] = the residual
 * stream (hi + lo) after proj_in, attn1, attn2 and the MLP; taps_ln [3][n*H*W][2] = (sum, sum of squares) per token row that
 * norm1 / norm2 / norm3 read. trace: NULL or SDB_TRACE_INTS ints (see above). */
int sdb_test_spatial_transformer(sdb_ctx* ctx, int index, const float* x, int n, int c, int H, int W, const float* context,
                                 int lmax, const int32_t* lens, int flags, float* out, float* out16, float* out_norm, float* taps_y,
                                 float* taps_ln, int32_t* trace);
/* One stage of the autoencoder, or one of the two CUDA-core convs the UNet shares with it, run on the weights
 * sdb_finalize_weights packed with the model's own launch code. Needs finalized weights. stage (x [n][c][H][W] NCHW, c as listed):
 *   SDB_VAE_DEC_IN     decoder conv_in with post_quant_conv and the pre-scale `scale` folded in; x = latent (c 4) -> out 512 ch
 *   SDB_VAE_DEC_ATTN,  decoder / encoder mid attention (c 512; H * W a multiple of 64, at most 9216); tap = the attention output
 *   SDB_VAE_ENC_ATTN   before proj_out (fp16 hi + lo), out_norm = SiLU(GroupNorm(out; mid/block_2/norm1)) from proj_out's partials
 *   SDB_VAE_DEC_OUT,   norm_out + SiLU + conv_out, fused (c 128 -> 3, 320 -> 4, 512 -> 8); for SDB_VAE_ENC_OUT, tap receives
 *   SDB_VAE_UNET_OUT,  quant_conv + the slice [0, 4): [n][4][H][W], or with flags & 2 strided and scaled as the inpainting tensor
 *   SDB_VAE_ENC_OUT    [n][5][H][W] is filled (channels 1-4, times `scale`); values the slice does not write are kept from entry
 *   SDB_VAE_ENC_IN     encoder conv_in on the zero-padded 3 -> 4 channel weights (c 4) -> 128 ch
 *   SDB_VAE_UNET_IN    the UNet's conv_in (c 4) -> 320 ch with out16 = its fp16 hi + lo copy; on a 9- / 8-channel context cond
 *                      [n][cin-4][H][W] holds the extra channels, read as the sampler stages them (sample s reads cond[s % m])
 *   SDB_VAE_ENC_DOWN0..2  encoder/blocks/i/downsampler (c 128 / 256 / 512, H and W even) -> [n][c][H/2][W/2]; out_norm =
 *                      SiLU(GroupNorm(out; blocks/i+1/res1/norm1)) from the conv's partials
 * flags: 1 = x is staged with GroupNorm partials, as a ResnetBlock leaves it (a 3-pass identity conv: the stage sees hi + lo of x);
 * else the fp32 tensor without statistics. out16 / tap / out_norm may be NULL where a stage has none. trace: NULL or
 * SDB_TRACE_INTS ints (see above). */
enum {
  SDB_VAE_DEC_IN = 0,
  SDB_VAE_DEC_ATTN = 1,
  SDB_VAE_ENC_ATTN = 2,
  SDB_VAE_DEC_OUT = 3,
  SDB_VAE_UNET_OUT = 4,
  SDB_VAE_ENC_OUT = 5,
  SDB_VAE_ENC_IN = 6,
  SDB_VAE_UNET_IN = 7,
  SDB_VAE_ENC_DOWN0 = 8,
  SDB_VAE_ENC_DOWN1 = 9,
  SDB_VAE_ENC_DOWN2 = 10
};
int sdb_test_vae_stage(sdb_ctx* ctx, int stage, const float* x, const float* cond, int n, int c, int H, int W, float scale,
                       int flags, float* out, float* out16, float* tap, float* out_norm, int32_t* trace);
/* One block of the CLIP text encoder (clip/mod.rs:109-115), index 0..11, or with index 12 its final LayerNorm, run on the weights
 * sdb_finalize_weights packed with the encoder's own launch code. Needs finalized weights. x [n][L][768] (1 <= L <= 77) is the
 * residual stream entering the block, staged at the encoder's per-sample row pitch round_up(L, 8) as the embedding leaves it;
 * flags: 1 = the pad rows hold large finite junk instead of zeros. out [n][L][768] = the block output (index 12: the final
 * LayerNorm). taps (NULL, or unused for index 12) = 11 planes of [n][L][768] floats: LN1 (fp16 hi + lo), q, k (fp16), V (read
 * back from V^T, fp16), the attention output (hi + lo), x after the attention, LN2 (hi + lo), then QuickGELU(fc1) (hi + lo) as
 * [n][L][3072]. trace: NULL or SDB_TRACE_INTS ints (see above). */
int sdb_test_clip_block(sdb_ctx* ctx, int index, const float* x, int n, int L, int flags, float* out, float* taps,
                        int32_t* trace);
/* The first `count` values of stochastic DDIM's noise z at timestep t (0 <= t < 1000) for noise_seed, as the fused sampler step
 * draws them (see sdb_set_sampler). Host buffer out [count]. */
int sdb_test_step_noise(sdb_ctx* ctx, uint64_t noise_seed, int t, int64_t count, float* out);

#ifdef __cplusplus
}
#endif
#endif /* SDB200_H */
