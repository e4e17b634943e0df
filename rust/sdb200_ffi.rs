//! Reference-side binding of libsdb200.so — SOURCE ONLY (no rustc/cargo in the build image; see DESIGN.md).
//!
//! Drop this file into the reference as `src/sdb200.rs`, add `pub mod sdb200;` to `src/lib.rs`, link with
//! `println!("cargo:rustc-link-lib=dylib=sdb200")` from a build script, and replace the three hot-path calls in
//! `src/bin/sample/main.rs:100-109`:
//!
//!   let images = sd.sample_image(context, unconditional_context, scale, n_steps);
//! becomes
//!   let sdb = sdb200::StableDiffusion::new(0)?;
//!   sdb.load_dump_dir(&model_name)?;          // in place of load_stable_diffusion(&model_name, &device)
//!   sdb.finalize_weights()?;
//!   let images = sdb.sample_image(&context_f32, [n, l], &uncond_f32, lu, scale, n_steps, None, 0)?;
//!
//! The signatures keep the reference's argument meaning (src/model/stablediffusion/mod.rs:51-57,
//! src/model/unet/mod.rs:109-114, src/model/autoencoder/mod.rs:68) with plain fp32 slices in place of
//! `Tensor<B, D>` (same contiguous row-major contents: NCHW / [n, L, 768]).

use std::ffi::{c_char, c_int, c_void, CStr, CString};

#[repr(C)]
pub struct SdbCtx {
    _private: [u8; 0],
}

/// include/sdb200.h: sdb_batch — n different requests of one sampling call (DESIGN.md §7 f7).
#[repr(C)]
pub struct SdbBatch {
    pub n: c_int,
    pub l: c_int,
    pub context: *const f32,
    pub context_len: *const i32,
    pub lu: c_int,
    pub uncond: *const f32,
    pub uncond_len: *const i32,
    pub guidance_scale: *const f64,
    pub seed: *const u64,
    pub noise_seed: *const u64,
}

extern "C" {
    fn sdb_create(device: c_int, out: *mut *mut SdbCtx) -> c_int;
    fn sdb_create_inpaint(device: c_int, out: *mut *mut SdbCtx) -> c_int;
    fn sdb_create_pix2pix(device: c_int, out: *mut *mut SdbCtx) -> c_int;
    fn sdb_destroy(ctx: *mut SdbCtx) -> c_int;
    fn sdb_last_error(ctx: *mut SdbCtx) -> *const c_char;
    fn sdb_set_tensor(ctx: *mut SdbCtx, name: *const c_char, host: *const f32, dims: *const i64, ndim: c_int) -> c_int;
    fn sdb_load_dump_dir(ctx: *mut SdbCtx, path: *const c_char) -> c_int;
    fn sdb_load_safetensors(ctx: *mut SdbCtx, path: *const c_char) -> c_int;
    fn sdb_probe_safetensors(path: *const c_char, kind: *mut c_int, conv_in_width: *mut c_int) -> c_int;
    fn sdb_finalize_weights(ctx: *mut SdbCtx) -> c_int;
    fn sdb_clip_forward(ctx: *mut SdbCtx, tokens: *const i32, n: c_int, l: c_int, out: *mut f32) -> c_int;
    fn sdb_encode_image(ctx: *mut SdbCtx, img: *const f32, n: c_int, h: c_int, w: c_int, latent: *mut f32) -> c_int;
    fn sdb_unet_forward(ctx: *mut SdbCtx, x: *const f32, timestep: i32, context: *const f32, n: c_int, h: c_int,
                        w: c_int, l: c_int, out: *mut f32) -> c_int;
    fn sdb_decode_latent(ctx: *mut SdbCtx, latent: *const f32, n: c_int, h: c_int, w: c_int, img: *mut f32) -> c_int;
    fn sdb_sample_image(ctx: *mut SdbCtx, context: *const f32, n: c_int, l: c_int, uncond: *const f32, lu: c_int,
                        guidance_scale: f64, n_steps: c_int, init_latent: *const f32, seed: u64, h: c_int, w: c_int,
                        rgb: *mut u8) -> c_int;
    fn sdb_sample_latent(ctx: *mut SdbCtx, context: *const f32, n: c_int, l: c_int, uncond: *const f32, lu: c_int,
                         guidance_scale: f64, n_steps: c_int, init_latent: *const f32, seed: u64, h: c_int, w: c_int,
                         latent_out: *mut f32) -> c_int;
    fn sdb_latent_to_image(ctx: *mut SdbCtx, latent: *const f32, n: c_int, h: c_int, w: c_int, rgb: *mut u8) -> c_int;
    fn sdb_forward_diffuser(ctx: *mut SdbCtx, latent: *const f32, timestep: i32, context: *const f32, n: c_int, l: c_int,
                            uncond: *const f32, lu: c_int, guidance_scale: f64, h: c_int, w: c_int, pred: *mut f32,
                            out_uncond: *mut f32, out_cond: *mut f32) -> c_int;
    fn sdb_img2img(ctx: *mut SdbCtx, image: *const u8, mask: *const u8, strength: f64, context: *const f32, n: c_int, l: c_int,
                   uncond: *const f32, lu: c_int, guidance_scale: f64, n_steps: c_int, noise: *const f32, seed: u64, h: c_int,
                   w: c_int, latent_out: *mut f32, rgb_out: *mut u8) -> c_int;
    #[allow(dead_code)]
    fn sdb_img2img_dev(ctx: *mut SdbCtx, d_image: *const c_void, d_mask: *const c_void, strength: f64, d_context: *const c_void,
                       n: c_int, l: c_int, d_uncond: *const c_void, lu: c_int, guidance_scale: f64, n_steps: c_int,
                       d_noise: *const c_void, h: c_int, w: c_int, d_latent_out: *mut c_void, d_rgb_out: *mut c_void,
                       stream: *mut c_void) -> c_int;
    fn sdb_edit_image(ctx: *mut SdbCtx, image: *const u8, context: *const f32, n: c_int, l: c_int, uncond: *const f32, lu: c_int,
                      text_scale: f64, image_scale: f64, n_steps: c_int, init_latent: *const f32, seed: u64, h: c_int, w: c_int,
                      latent_out: *mut f32, rgb_out: *mut u8) -> c_int;
    #[allow(dead_code)]
    fn sdb_edit_image_dev(ctx: *mut SdbCtx, d_image: *const c_void, d_context: *const c_void, n: c_int, l: c_int,
                          d_uncond: *const c_void, lu: c_int, text_scale: f64, image_scale: f64, n_steps: c_int,
                          d_init_latent: *const c_void, h: c_int, w: c_int, d_latent_out: *mut c_void, d_rgb_out: *mut c_void,
                          stream: *mut c_void) -> c_int;
    fn sdb_set_sampler(ctx: *mut SdbCtx, kind: c_int, eta: f64, noise_seed: u64) -> c_int;
    fn sdb_set_schedule(ctx: *mut SdbCtx, kind: c_int) -> c_int;
    fn sdb_unet_forward_at(ctx: *mut SdbCtx, x: *const f32, t: f64, context: *const f32, n: c_int, h: c_int, w: c_int, l: c_int,
                           out: *mut f32) -> c_int;
    fn sdb_tensor_count(ctx: *mut SdbCtx) -> c_int;
    fn sdb_tensor_info(ctx: *mut SdbCtx, index: c_int, name: *mut *const c_char, dims: *mut i64, ndim: *mut c_int) -> c_int;
    fn sdb_lora_add(ctx: *mut SdbCtx, adapter: c_int, tensor: *const c_char, rank: c_int, down: *const f32, up: *const f32,
                    alpha: f64) -> c_int;
    fn sdb_lora_scale(ctx: *mut SdbCtx, adapter: c_int, multiplier: f64) -> c_int;
    fn sdb_lora_remove(ctx: *mut SdbCtx, adapter: c_int) -> c_int;
    fn sdb_lora_apply(ctx: *mut SdbCtx) -> c_int;
    fn sdb_get_merged_tensor(ctx: *mut SdbCtx, tensor: *const c_char, host: *mut f32, count: i64) -> c_int;
    fn sdb_sample_batch(ctx: *mut SdbCtx, batch: *const SdbBatch, n_steps: c_int, init_latent: *const f32, h: c_int, w: c_int,
                        latent_out: *mut f32, rgb_out: *mut u8) -> c_int;
    fn sdb_img2img_batch(ctx: *mut SdbCtx, batch: *const SdbBatch, image: *const u8, mask: *const u8, strength: f64, n_steps: c_int,
                         noise: *const f32, h: c_int, w: c_int, latent_out: *mut f32, rgb_out: *mut u8) -> c_int;
    fn sdb_nccl_unique_id(id128: *mut c_void) -> c_int;
    fn sdb_broadcast_weights(ctx: *mut SdbCtx, id128: *const c_void, rank: c_int, world: c_int) -> c_int;
    #[allow(dead_code)]
    fn sdb_sample_image_dev(ctx: *mut SdbCtx, d_context: *const c_void, n: c_int, l: c_int, d_uncond: *const c_void,
                            lu: c_int, guidance_scale: f64, n_steps: c_int, d_init_latent: *const c_void, h: c_int,
                            w: c_int, d_rgb: *mut c_void, stream: *mut c_void) -> c_int;
}

#[derive(Debug)]
pub struct SdbError(pub String);

const SDB_SAMPLER_DDIM: c_int = 0;
const SDB_SAMPLER_DPMPP_2M: c_int = 1;
const SDB_SCHEDULE_DDIM: c_int = 0;
const SDB_SCHEDULE_KARRAS: c_int = 1;

/// The sampler of the sampling calls (include/sdb200.h: sdb_set_sampler).
#[derive(Clone, Copy, Debug)]
pub enum Sampler {
    Ddim { eta: f64 },
    DpmPp2M,
}

/// The grid the sampler walks (include/sdb200.h: sdb_set_schedule): the reference's timesteps, or the sigma grid of Karras et
/// al. 2022 (rho = 7) at fractional timesteps.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum Schedule {
    Ddim,
    Karras,
}

pub struct StableDiffusion {
    ctx: *mut SdbCtx,
}

/// What an SD-1.x .safetensors file holds (include/sdb200.h: sdb_probe_safetensors).
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum Checkpoint {
    /// every weight; the UNet's conv_in takes this many channels: 4 (`new`), 9 (`new_inpaint`) or 8 (`new_pix2pix`)
    Full { conv_in_width: i32 },
    /// the autoencoder's weights only (a standalone SD VAE release)
    Vae,
}

/// Validates an SD-1.x single-file .safetensors checkpoint without a context or a device (DESIGN.md §7 f13).
pub fn probe_safetensors(path: &str) -> Result<Checkpoint, SdbError> {
    let cpath = CString::new(path).unwrap();
    let (mut kind, mut width) = (0 as c_int, 0 as c_int);
    if unsafe { sdb_probe_safetensors(cpath.as_ptr(), &mut kind, &mut width) } != 0 {
        return Err(SdbError(unsafe { CStr::from_ptr(sdb_last_error(std::ptr::null_mut())) }.to_string_lossy().into()));
    }
    Ok(if kind == 0 { Checkpoint::Full { conv_in_width: width } } else { Checkpoint::Vae })
}

impl StableDiffusion {
    /// Replaces `StableDiffusionConfig::new().init(&device)` (src/model/stablediffusion/mod.rs:22-39).
    pub fn new(device: i32) -> Result<Self, SdbError> {
        let mut ctx = std::ptr::null_mut();
        let rc = unsafe { sdb_create(device, &mut ctx) };
        if rc != 0 {
            return Err(SdbError(unsafe { CStr::from_ptr(sdb_last_error(std::ptr::null_mut())) }.to_string_lossy().into()));
        }
        Ok(Self { ctx })
    }

    /// A context for an inpainting checkpoint: a 9-channel `conv_in` reading latent | mask | masked-image latent (DESIGN.md §7 f9).
    /// `img2img` then needs the mask; the text-to-image calls fail.
    pub fn new_inpaint(device: i32) -> Result<Self, SdbError> {
        let mut ctx = std::ptr::null_mut();
        let rc = unsafe { sdb_create_inpaint(device, &mut ctx) };
        if rc != 0 {
            return Err(SdbError(unsafe { CStr::from_ptr(sdb_last_error(std::ptr::null_mut())) }.to_string_lossy().into()));
        }
        Ok(Self { ctx })
    }

    /// A context for an InstructPix2Pix checkpoint: an 8-channel `conv_in` reading latent | image latent (DESIGN.md §7 f10).
    /// `edit_image` is then the sampling call; the text-to-image, `img2img` and batch calls fail.
    pub fn new_pix2pix(device: i32) -> Result<Self, SdbError> {
        let mut ctx = std::ptr::null_mut();
        let rc = unsafe { sdb_create_pix2pix(device, &mut ctx) };
        if rc != 0 {
            return Err(SdbError(unsafe { CStr::from_ptr(sdb_last_error(std::ptr::null_mut())) }.to_string_lossy().into()));
        }
        Ok(Self { ctx })
    }

    fn check(&self, rc: c_int) -> Result<(), SdbError> {
        if rc == 0 {
            Ok(())
        } else {
            Err(SdbError(unsafe { CStr::from_ptr(sdb_last_error(self.ctx)) }.to_string_lossy().into()))
        }
    }

    /// Replaces `load_tensor` + `Param::from_tensor` (src/model/load.rs:30-47): `name` is the dump-dir path
    /// without the `.npy` suffix, e.g. "unet/input_blocks/rt1/res/conv_in/weight".
    pub fn set_tensor(&self, name: &str, data: &[f32], dims: &[i64]) -> Result<(), SdbError> {
        let cname = CString::new(name).unwrap();
        self.check(unsafe { sdb_set_tensor(self.ctx, cname.as_ptr(), data.as_ptr(), dims.as_ptr(), dims.len() as c_int) })
    }

    /// Replaces `load_stable_diffusion(path, device)` (src/model/stablediffusion/load.rs:16-33): reads the dump-dir tree.
    pub fn load_dump_dir(&self, path: &str) -> Result<(), SdbError> {
        let cpath = CString::new(path).unwrap();
        self.check(unsafe { sdb_load_dump_dir(self.ctx, cpath.as_ptr()) })
    }

    /// An SD-1.x single-file .safetensors checkpoint in the original LDM layout, or a VAE-only file (DESIGN.md §7 f13), in
    /// place of converting it to a dump-dir tree; then `finalize_weights`. A rejected file leaves the weights as they were.
    pub fn load_safetensors(&self, path: &str) -> Result<(), SdbError> {
        let cpath = CString::new(path).unwrap();
        self.check(unsafe { sdb_load_safetensors(self.ctx, cpath.as_ptr()) })
    }

    pub fn finalize_weights(&self) -> Result<(), SdbError> {
        self.check(unsafe { sdb_finalize_weights(self.ctx) })
    }

    /// `Autoencoder::encode_image(x)` (src/model/autoencoder/mod.rs:60-66): [n, 3, h, w] -> [n, 4, h/8, w/8].
    pub fn encode_image(&self, img: &[f32], [n, h, w]: [usize; 3]) -> Result<Vec<f32>, SdbError> {
        let mut latent = vec![0f32; n * 4 * (h / 8) * (w / 8)];
        self.check(unsafe { sdb_encode_image(self.ctx, img.as_ptr(), n as c_int, h as c_int, w as c_int, latent.as_mut_ptr()) })?;
        Ok(latent)
    }

    /// `CLIP::forward(tokens)` (src/model/clip/mod.rs:56-75): ids [n, l] (l <= 77, unpadded) -> [n, l, 768].
    pub fn clip_forward(&self, tokens: &[i32], [n, l]: [usize; 2]) -> Result<Vec<f32>, SdbError> {
        let mut out = vec![0f32; n * l * 768];
        self.check(unsafe { sdb_clip_forward(self.ctx, tokens.as_ptr(), n as c_int, l as c_int, out.as_mut_ptr()) })?;
        Ok(out)
    }

    /// `UNet::forward(x, timesteps, context)` (src/model/unet/mod.rs:109-114).
    pub fn unet_forward(&self, x: &[f32], [n, h, w]: [usize; 3], timestep: i32, context: &[f32], l: usize) -> Result<Vec<f32>, SdbError> {
        let mut out = vec![0f32; n * 4 * h * w];
        self.check(unsafe {
            sdb_unet_forward(self.ctx, x.as_ptr(), timestep, context.as_ptr(), n as c_int, h as c_int, w as c_int, l as c_int, out.as_mut_ptr())
        })?;
        Ok(out)
    }

    /// `unet_forward` at a real timestep t in [0, 999] (an extension, DESIGN.md §7 f15): at an integer t the same bits.
    pub fn unet_forward_at(&self, x: &[f32], [n, h, w]: [usize; 3], t: f64, context: &[f32], l: usize) -> Result<Vec<f32>, SdbError> {
        let mut out = vec![0f32; n * 4 * h * w];
        self.check(unsafe {
            sdb_unet_forward_at(self.ctx, x.as_ptr(), t, context.as_ptr(), n as c_int, h as c_int, w as c_int, l as c_int, out.as_mut_ptr())
        })?;
        Ok(out)
    }

    /// `Autoencoder::decode_latent(latent)` (src/model/autoencoder/mod.rs:68-71).
    pub fn decode_latent(&self, latent: &[f32], [n, h, w]: [usize; 3]) -> Result<Vec<f32>, SdbError> {
        let mut img = vec![0f32; n * 3 * 64 * h * w];
        self.check(unsafe { sdb_decode_latent(self.ctx, latent.as_ptr(), n as c_int, h as c_int, w as c_int, img.as_mut_ptr()) })?;
        Ok(img)
    }

    /// `StableDiffusion::sample_image(context, unconditional_context, scale, n_steps) -> Vec<Vec<u8>>`
    /// (src/model/stablediffusion/mod.rs:51-67). `init_latent = None` draws N(0,1) on the device from `seed`.
    #[allow(clippy::too_many_arguments)]
    pub fn sample_image(&self, context: &[f32], [n, l]: [usize; 2], unconditional_context: &[f32], lu: usize,
                        unconditional_guidance_scale: f64, n_steps: usize, init_latent: Option<&[f32]>, seed: u64)
                        -> Result<Vec<Vec<u8>>, SdbError> {
        let (h, w) = (64usize, 64usize); // the reference hard-codes 512x512 (stablediffusion/mod.rs:74-75,116)
        let mut rgb = vec![0u8; n * 8 * h * 8 * w * 3];
        self.check(unsafe {
            sdb_sample_image(self.ctx, context.as_ptr(), n as c_int, l as c_int, unconditional_context.as_ptr(), lu as c_int,
                             unconditional_guidance_scale, n_steps as c_int,
                             init_latent.map_or(std::ptr::null(), |s| s.as_ptr()), seed, h as c_int, w as c_int, rgb.as_mut_ptr())
        })?;
        Ok(rgb.chunks(8 * h * 8 * w * 3).map(|c| c.to_vec()).collect())
    }
}

impl StableDiffusion {
    /// `StableDiffusion::sample_latent(context, unconditional_context, scale, n_steps) -> Tensor<B, 4>`
    /// (src/model/stablediffusion/mod.rs:102-160); returns the final latent [n, 4, 64, 64].
    #[allow(clippy::too_many_arguments)]
    pub fn sample_latent(&self, context: &[f32], [n, l]: [usize; 2], unconditional_context: &[f32], lu: usize,
                         unconditional_guidance_scale: f64, n_steps: usize, init_latent: Option<&[f32]>, seed: u64)
                         -> Result<Vec<f32>, SdbError> {
        let (h, w) = (64usize, 64usize);
        let mut latent = vec![0f32; n * 4 * h * w];
        self.check(unsafe {
            sdb_sample_latent(self.ctx, context.as_ptr(), n as c_int, l as c_int, unconditional_context.as_ptr(), lu as c_int,
                              unconditional_guidance_scale, n_steps as c_int,
                              init_latent.map_or(std::ptr::null(), |s| s.as_ptr()), seed, h as c_int, w as c_int, latent.as_mut_ptr())
        })?;
        Ok(latent)
    }

    /// `StableDiffusion::latent_to_image(latent) -> Vec<Vec<u8>>` (src/model/stablediffusion/mod.rs:69-100).
    pub fn latent_to_image(&self, latent: &[f32], [n, h, w]: [usize; 3]) -> Result<Vec<Vec<u8>>, SdbError> {
        let mut rgb = vec![0u8; n * 8 * h * 8 * w * 3];
        self.check(unsafe { sdb_latent_to_image(self.ctx, latent.as_ptr(), n as c_int, h as c_int, w as c_int, rgb.as_mut_ptr()) })?;
        Ok(rgb.chunks(8 * h * 8 * w * 3).map(|c| c.to_vec()).collect())
    }

    /// `forward_diffuser(latent, timestep, context, unconditional_context, scale)` (src/model/stablediffusion/mod.rs:162-192):
    /// the guided noise prediction of one step.
    #[allow(clippy::too_many_arguments)]
    pub fn forward_diffuser(&self, latent: &[f32], [n, h, w]: [usize; 3], timestep: i32, context: &[f32], l: usize,
                            unconditional_context: &[f32], lu: usize, unconditional_guidance_scale: f64) -> Result<Vec<f32>, SdbError> {
        let mut pred = vec![0f32; n * 4 * h * w];
        self.check(unsafe {
            sdb_forward_diffuser(self.ctx, latent.as_ptr(), timestep, context.as_ptr(), n as c_int, l as c_int,
                                 unconditional_context.as_ptr(), lu as c_int, unconditional_guidance_scale, h as c_int, w as c_int,
                                 pred.as_mut_ptr(), std::ptr::null_mut(), std::ptr::null_mut())
        })?;
        Ok(pred)
    }

    /// Image-to-image / masked inpainting, an extension built from the reference's encode_image
    /// (src/model/autoencoder/mod.rs:60-66) and the schedule and DDIM step of sample_latent (src/model/stablediffusion/mod.rs:123-156).
    /// `image`: n RGB images of `height` x `width` (multiples of 64) as HWC u8, the format `sample_image` returns; `mask`:
    /// n x height x width u8 (255 = regenerate, 0 = keep) or None; `strength` in (0, 1]: the last floor(strength * N) of the N
    /// timesteps run. `noise = None` draws the latent `sample_image` would start from for `seed`.
    #[allow(clippy::too_many_arguments)]
    pub fn img2img(&self, image: &[u8], [n, height, width]: [usize; 3], mask: Option<&[u8]>, strength: f64, context: &[f32],
                   l: usize, unconditional_context: &[f32], lu: usize, unconditional_guidance_scale: f64, n_steps: usize,
                   noise: Option<&[f32]>, seed: u64) -> Result<Vec<Vec<u8>>, SdbError> {
        let (h, w) = (height / 8, width / 8);
        if image.len() != n * height * width * 3 || mask.map_or(false, |m| m.len() != n * height * width)
            || noise.map_or(false, |z| z.len() != n * 4 * h * w) {
            return Err(SdbError("img2img: buffer sizes do not match [n, height, width]".into()));
        }
        let mut rgb = vec![0u8; n * height * width * 3];
        self.check(unsafe {
            sdb_img2img(self.ctx, image.as_ptr(), mask.map_or(std::ptr::null(), |m| m.as_ptr()), strength, context.as_ptr(),
                        n as c_int, l as c_int, unconditional_context.as_ptr(), lu as c_int, unconditional_guidance_scale,
                        n_steps as c_int, noise.map_or(std::ptr::null(), |z| z.as_ptr()), seed, h as c_int, w as c_int,
                        std::ptr::null_mut(), rgb.as_mut_ptr())
        })?;
        Ok(rgb.chunks(height * width * 3).map(|c| c.to_vec()).collect())
    }

    /// InstructPix2Pix editing on a `new_pix2pix` context (DESIGN.md §7 f10). `image`: n RGB images of `height` x `width`
    /// (multiples of 64) as HWC u8, the format `sample_image` returns; `context`: n instructions of `l` rows; every step runs the
    /// UNet on (no image, negative), (image, negative) and (image, instruction) and combines them with `text_scale` and
    /// `image_scale` (7.5 and 1.5 in the original pipeline). `init_latent = None` draws the latent `sample_image` would start
    /// from for `seed`.
    #[allow(clippy::too_many_arguments)]
    pub fn edit_image(&self, image: &[u8], [n, height, width]: [usize; 3], context: &[f32], l: usize,
                      unconditional_context: &[f32], lu: usize, text_scale: f64, image_scale: f64, n_steps: usize,
                      init_latent: Option<&[f32]>, seed: u64) -> Result<Vec<Vec<u8>>, SdbError> {
        let (h, w) = (height / 8, width / 8);
        if image.len() != n * height * width * 3 || context.len() != n * l * 768
            || init_latent.map_or(false, |z| z.len() != n * 4 * h * w) {
            return Err(SdbError("edit_image: buffer sizes do not match [n, height, width] and [n, l, 768]".into()));
        }
        let mut rgb = vec![0u8; n * height * width * 3];
        self.check(unsafe {
            sdb_edit_image(self.ctx, image.as_ptr(), context.as_ptr(), n as c_int, l as c_int, unconditional_context.as_ptr(),
                           lu as c_int, text_scale, image_scale, n_steps as c_int,
                           init_latent.map_or(std::ptr::null(), |z| z.as_ptr()), seed, h as c_int, w as c_int,
                           std::ptr::null_mut(), rgb.as_mut_ptr())
        })?;
        Ok(rgb.chunks(height * width * 3).map(|c| c.to_vec()).collect())
    }

    /// The sampler of `sample_image` / `sample_latent` / `img2img` until changed (an extension: the reference samples with DDIM at
    /// eta = 0, src/model/stablediffusion/mod.rs:119). `Sampler::Ddim { eta }` with eta in [0, 1] (0 = the reference's sampler,
    /// the default) or `Sampler::DpmPp2M` (DPM-Solver++(2M), good at 10-15 steps); `noise_seed` keys stochastic DDIM's noise.
    pub fn set_sampler(&self, sampler: Sampler, noise_seed: u64) -> Result<(), SdbError> {
        let (kind, eta) = match sampler {
            Sampler::Ddim { eta } => (SDB_SAMPLER_DDIM, eta),
            Sampler::DpmPp2M => (SDB_SAMPLER_DPMPP_2M, 0.0),
        };
        self.check(unsafe { sdb_set_sampler(self.ctx, kind, eta, noise_seed) })
    }

    /// The grid `set_sampler`'s sampler walks until changed (an extension, DESIGN.md §7 f15): `Schedule::Ddim` (the reference's,
    /// the default) or `Schedule::Karras`. Euler Karras = `Ddim { eta: 0 }`, Euler a Karras = `Ddim { eta: 1 }`, DPM++ 2M Karras =
    /// `DpmPp2M`, each with `Schedule::Karras`.
    pub fn set_schedule(&self, schedule: Schedule) -> Result<(), SdbError> {
        let kind = match schedule {
            Schedule::Ddim => SDB_SCHEDULE_DDIM,
            Schedule::Karras => SDB_SCHEDULE_KARRAS,
        };
        self.check(unsafe { sdb_set_schedule(self.ctx, kind) })
    }

    /// One term of LoRA adapter `adapter` (an extension, DESIGN.md §7 f8) on registry weight `tensor`: `down` = rank x fan-in
    /// floats, `up` = out x rank floats, `alpha`. Pending until `lora_apply`; the lengths are checked here, the rest in C.
    pub fn lora_add(&self, adapter: i32, tensor: &str, rank: usize, down: &[f32], up: &[f32], alpha: f64) -> Result<(), SdbError> {
        // the C side reads rank * fan_in floats from `down` and out * rank from `up`: check both lengths against the registry
        // shape first, so that a short slice is an error and never read past its end
        let (out, fan_in) = self.lora_geometry(tensor)?;
        if rank == 0 || down.len() != rank * fan_in || up.len() != out * rank {
            return Err(SdbError(format!("lora_add {tensor}: rank {rank} needs down = {} and up = {} floats, got {} and {}",
                                        rank * fan_in, out * rank, down.len(), up.len())));
        }
        let name = CString::new(tensor).map_err(|_| SdbError("tensor name contains NUL".into()))?;
        self.check(unsafe { sdb_lora_add(self.ctx, adapter, name.as_ptr(), rank as c_int, down.as_ptr(), up.as_ptr(), alpha) })
    }

    /// (out, fan-in) of a registry weight: [in][out] for a Linear, OIHW for a conv.
    fn lora_geometry(&self, tensor: &str) -> Result<(usize, usize), SdbError> {
        let n = unsafe { sdb_tensor_count(self.ctx) };
        for i in 0..n {
            let mut name: *const c_char = std::ptr::null();
            let mut dims = [0i64; 4];
            let mut ndim: c_int = 0;
            self.check(unsafe { sdb_tensor_info(self.ctx, i, &mut name, dims.as_mut_ptr(), &mut ndim) })?;
            if unsafe { CStr::from_ptr(name) }.to_bytes() != tensor.as_bytes() {
                continue;
            }
            return match ndim {
                2 => Ok((dims[1] as usize, dims[0] as usize)),
                4 => Ok((dims[0] as usize, (dims[1] * dims[2] * dims[3]) as usize)),
                _ => Err(SdbError(format!("lora_add {tensor}: not a LoRA target (a {ndim}-d tensor)"))),
            };
        }
        Err(SdbError(format!("lora_add: unknown tensor '{tensor}'")))
    }

    /// Multiplier of an adapter (0 disables it without freeing it). Pending until `lora_apply`.
    pub fn lora_scale(&self, adapter: i32, multiplier: f64) -> Result<(), SdbError> {
        self.check(unsafe { sdb_lora_scale(self.ctx, adapter, multiplier) })
    }

    /// Removes an adapter (-1 = all). Pending until `lora_apply`.
    pub fn lora_remove(&self, adapter: i32) -> Result<(), SdbError> {
        self.check(unsafe { sdb_lora_remove(self.ctx, adapter) })
    }

    /// Merges and re-packs the layers whose adapters changed; cached step graphs stay valid.
    pub fn lora_apply(&self) -> Result<(), SdbError> {
        self.check(unsafe { sdb_lora_apply(self.ctx) })
    }

    /// The merged weight the packers read (the base tensor when no active term targets it); `out` holds its element count.
    pub fn get_merged_tensor(&self, tensor: &str, out: &mut [f32]) -> Result<(), SdbError> {
        let name = CString::new(tensor).map_err(|_| SdbError("tensor name contains NUL".into()))?;
        self.check(unsafe { sdb_get_merged_tensor(self.ctx, name.as_ptr(), out.as_mut_ptr(), out.len() as i64) })
    }

    /// n different requests in one call (an extension, DESIGN.md §7 f7): request i is (`contexts[i]` = L_i x 768 floats,
    /// `unconditional_contexts[i]` = Lu_i x 768, `guidance_scales[i]`, `seeds[i]`) and gives, to rounding, what `sample_image`
    /// gives for it alone, while every step runs one UNet pass for all of them. `noise_seeds` keys stochastic DDIM per request
    /// (None = the `set_sampler` seed). The sampler and `n_steps` hold for the whole call. 512 x 512 like `sample_image`.
    pub fn sample_batch(&self, contexts: &[&[f32]], unconditional_contexts: &[&[f32]], guidance_scales: &[f64], n_steps: usize,
                        seeds: &[u64], noise_seeds: Option<&[u64]>) -> Result<Vec<Vec<u8>>, SdbError> {
        let (h, w) = (64usize, 64usize);
        let packed = Packed::new(contexts, unconditional_contexts, guidance_scales, Some(seeds), noise_seeds)?;
        let mut rgb = vec![0u8; packed.n * 8 * h * 8 * w * 3];
        self.check(unsafe {
            sdb_sample_batch(self.ctx, &packed.batch(), n_steps as c_int, std::ptr::null(), h as c_int, w as c_int,
                             std::ptr::null_mut(), rgb.as_mut_ptr())
        })?;
        Ok(rgb.chunks(8 * h * 8 * w * 3).map(|c| c.to_vec()).collect())
    }

    /// `img2img` over n different requests (arguments as `sample_batch`; `image`, `mask` as `img2img`). `noise = None` draws each
    /// request's noise from its seed.
    #[allow(clippy::too_many_arguments)]
    pub fn img2img_batch(&self, image: &[u8], [height, width]: [usize; 2], mask: Option<&[u8]>, strength: f64, contexts: &[&[f32]],
                         unconditional_contexts: &[&[f32]], guidance_scales: &[f64], n_steps: usize, noise: Option<&[f32]>,
                         seeds: Option<&[u64]>, noise_seeds: Option<&[u64]>) -> Result<Vec<Vec<u8>>, SdbError> {
        let (h, w) = (height / 8, width / 8);
        let packed = Packed::new(contexts, unconditional_contexts, guidance_scales, seeds, noise_seeds)?;
        let n = packed.n;
        if image.len() != n * height * width * 3 || mask.map_or(false, |m| m.len() != n * height * width)
            || noise.map_or(false, |z| z.len() != n * 4 * h * w) {
            return Err(SdbError("img2img_batch: buffer sizes do not match [n, height, width]".into()));
        }
        let mut rgb = vec![0u8; n * height * width * 3];
        self.check(unsafe {
            sdb_img2img_batch(self.ctx, &packed.batch(), image.as_ptr(), mask.map_or(std::ptr::null(), |m| m.as_ptr()), strength,
                              n_steps as c_int, noise.map_or(std::ptr::null(), |z| z.as_ptr()), h as c_int, w as c_int,
                              std::ptr::null_mut(), rgb.as_mut_ptr())
        })?;
        Ok(rgb.chunks(height * width * 3).map(|c| c.to_vec()).collect())
    }

    /// Multi-GPU init: rank 0 calls `nccl_unique_id()` and ships the 128 bytes to the other ranks by any means; every rank then
    /// calls `broadcast_weights(&id, rank, world)` (one ncclBroadcast of the weight arena from rank 0) and `finalize_weights()`.
    pub fn nccl_unique_id() -> Result<[u8; 128], SdbError> {
        let mut id = [0u8; 128];
        if unsafe { sdb_nccl_unique_id(id.as_mut_ptr() as *mut c_void) } != 0 {
            return Err(SdbError("ncclGetUniqueId failed".into()));
        }
        Ok(id)
    }
    pub fn broadcast_weights(&self, id: &[u8; 128], rank: usize, world: usize) -> Result<(), SdbError> {
        self.check(unsafe { sdb_broadcast_weights(self.ctx, id.as_ptr() as *const c_void, rank as c_int, world as c_int) })
    }
}

/// The requests of a batch call padded to the longest prompt / negative (rows past a request's length are zero and never read).
struct Packed {
    n: usize,
    l: usize,
    lu: usize,
    context: Vec<f32>,
    context_len: Vec<i32>,
    uncond: Vec<f32>,
    uncond_len: Vec<i32>,
    scales: Vec<f64>,
    seeds: Option<Vec<u64>>,
    noise_seeds: Option<Vec<u64>>,
}

impl Packed {
    fn new(contexts: &[&[f32]], uncond: &[&[f32]], scales: &[f64], seeds: Option<&[u64]>, noise_seeds: Option<&[u64]>)
           -> Result<Self, SdbError> {
        let n = contexts.len();
        if n == 0 || uncond.len() != n || scales.len() != n || seeds.map_or(false, |s| s.len() != n)
            || noise_seeds.map_or(false, |s| s.len() != n) {
            return Err(SdbError("batch: every per-request list must hold the same number (>= 1) of requests".into()));
        }
        if contexts.iter().chain(uncond.iter()).any(|c| c.is_empty() || c.len() % 768 != 0) {
            return Err(SdbError("batch: every context must be a non-empty multiple of 768 floats".into()));
        }
        let pad = |rows: &[&[f32]]| {
            let lmax = rows.iter().map(|c| c.len() / 768).max().unwrap_or(1);
            let mut out = vec![0f32; n * lmax * 768];
            for (i, c) in rows.iter().enumerate() {
                out[i * lmax * 768..i * lmax * 768 + c.len()].copy_from_slice(c);
            }
            (lmax, out, rows.iter().map(|c| (c.len() / 768) as i32).collect::<Vec<_>>())
        };
        let (l, context, context_len) = pad(contexts);
        let (lu, uncond, uncond_len) = pad(uncond);
        Ok(Self { n, l, lu, context, context_len, uncond, uncond_len, scales: scales.to_vec(), seeds: seeds.map(|s| s.to_vec()),
                  noise_seeds: noise_seeds.map(|s| s.to_vec()) })
    }

    fn batch(&self) -> SdbBatch {
        SdbBatch {
            n: self.n as c_int, l: self.l as c_int, context: self.context.as_ptr(), context_len: self.context_len.as_ptr(),
            lu: self.lu as c_int, uncond: self.uncond.as_ptr(), uncond_len: self.uncond_len.as_ptr(),
            guidance_scale: self.scales.as_ptr(), seed: self.seeds.as_ref().map_or(std::ptr::null(), |s| s.as_ptr()),
            noise_seed: self.noise_seeds.as_ref().map_or(std::ptr::null(), |s| s.as_ptr()),
        }
    }
}

impl Drop for StableDiffusion {
    fn drop(&mut self) {
        unsafe { sdb_destroy(self.ctx) };
    }
}
