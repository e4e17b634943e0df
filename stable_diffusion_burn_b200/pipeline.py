"""Host-side mirror of the reference's Rust interface for the hot path, over the C ABI.

Same names, argument meaning and error behaviour as
  StableDiffusion::{sample_image, sample_latent, latent_to_image}  src/model/stablediffusion/mod.rs:51-160
  UNet::forward                                                    src/model/unet/mod.rs:109-142
  Autoencoder::decode_latent                                       src/model/autoencoder/mod.rs:68-71
Tensors are numpy fp32 arrays with the reference's shapes (NCHW, [n, L, 768]); errors raise
(the reference panics). No computation happens in Python and there is no fallback path: every call
goes to libsdb200.so and fails loudly if the CUDA library or an H100 is missing.

Differences forced by the tier (documented in DESIGN.md): the initial latent is an explicit argument
(the reference draws it from an unseeded backend RNG) and H/W are parameters (the reference hard-codes 64x64).
"""
from __future__ import annotations

import contextlib

import numpy as np

from ._lib import CKPT_FULL, Context, probe_safetensors


class UNet:
    def __init__(self, ctx: Context):
        self._c = ctx

    def forward(self, x: np.ndarray, timesteps, context: np.ndarray) -> np.ndarray:
        """x [n,4,H,W] (an inpainting UNet: [n,9,H,W] = latent | mask | masked-image latent; an InstructPix2Pix UNet:
        [n,8,H,W] = latent | image latent); timesteps Int[1] (one t for the batch); context [n,L,768] -> [n,4,H,W]."""
        ts = np.asarray(timesteps).reshape(-1)
        if ts.size != 1:
            raise ValueError("timesteps must hold exactly one value (reference: Tensor<B,1,Int> of length 1)")
        return self._c.unet_forward(x, int(ts[0]), context)


class Autoencoder:
    def __init__(self, ctx: Context):
        self._c = ctx

    def decode_latent(self, latent: np.ndarray) -> np.ndarray:
        """latent [n,4,H,W] -> image [n,3,8H,8W]."""
        return self._c.decode_latent(latent)

    def encode_image(self, img: np.ndarray) -> np.ndarray:
        """Autoencoder::encode_image (src/model/autoencoder/mod.rs:60-66): image [n,3,H,W] -> latent [n,4,H/8,W/8]."""
        return self._c.encode_image(img)

    def forward(self, img: np.ndarray) -> np.ndarray:
        """Autoencoder::forward (:56-58) = decode_latent(encode_image(x))."""
        return self.decode_latent(self.encode_image(img))


class CLIP:
    def __init__(self, ctx: Context):
        self._c = ctx

    def forward(self, tokens) -> np.ndarray:
        """CLIP::forward (src/model/clip/mod.rs:56-75): int ids [n,L] (L <= 77, unpadded) -> [n,L,768]."""
        return self._c.clip_forward(tokens)


class StableDiffusion:
    """Owns the device context; `diffusion`, `autoencoder` and `clip` mirror the reference's fields. inpaint=True holds an
    inpainting checkpoint (a 9-channel UNet, DESIGN.md §7 f9): img2img then needs a mask, and the txt2img calls fail.
    pix2pix=True holds an InstructPix2Pix checkpoint (an 8-channel UNet, f10): edit_image is then the sampling call, and the
    txt2img, img2img and batch calls fail."""

    def __init__(self, device: int = 0, inpaint: bool = False, pix2pix: bool = False):
        self.ctx = Context(device, inpaint=inpaint, pix2pix=pix2pix)
        self.diffusion = UNet(self.ctx)
        self.autoencoder = Autoencoder(self.ctx)
        self.clip = CLIP(self.ctx)

    # ---- prompt -> context (reference stablediffusion/mod.rs:194-211)
    def context(self, tokenizer, text: str) -> np.ndarray:
        """[1, L, 768]: CLIP of "<|startoftext|>{text}<|endoftext|>" (no padding to 77, like the reference)."""
        ids = tokenizer.encode(f"<|startoftext|>{text}<|endoftext|>")
        return self.clip.forward(np.asarray(ids, np.int32)[None])

    def unconditional_context(self, tokenizer) -> np.ndarray:
        """[Lu, 768] = context("").squeeze(0); Lu = 2 for the empty prompt."""
        return self.context(tokenizer, "")[0]

    # ---- weights (reference: load_stable_diffusion / load_record)
    def init_synthetic(self, seed: int = 0):
        self.ctx.init_synthetic(seed)
        self.ctx.finalize_weights()
        return self

    def load_dump_dir(self, path: str):
        """load_stable_diffusion(path, device) (src/model/stablediffusion/load.rs:16-33): the reference's dump-dir tree."""
        self.ctx.load_dump_dir(path)
        self.ctx.finalize_weights()
        return self

    @classmethod
    def from_checkpoint(cls, path, device: int = 0):
        """A context of the kind an SD-1.x single-file .safetensors checkpoint needs (a 4-, 9- (inpaint=True) or 8-channel
        (pix2pix=True) UNet, read from its conv_in), loaded from it and finalized. A VAE-only file raises ValueError: load it
        into an existing model with load_checkpoint."""
        kind, width = probe_safetensors(path)
        if kind != CKPT_FULL:
            raise ValueError(f"{path} holds only a VAE: load it with load_checkpoint into a model created from a full checkpoint")
        sd = cls(device, inpaint=width == 9, pix2pix=width == 8)
        try:
            return sd.load_checkpoint(path)
        except Exception:
            sd.close()
            raise

    def load_checkpoint(self, path):
        """An SD-1.x single-file .safetensors checkpoint (every weight and the schedule) or a VAE-only file (the autoencoder's
        weights only) (DESIGN.md §7 f13), then finalize. A rejected file leaves the weights as they were."""
        self.ctx.load_safetensors(path)
        self.ctx.finalize_weights()
        return self

    def load_arrays(self, arrays: dict):
        for name, a in arrays.items():
            self.ctx.set_tensor(name, a)
        self.ctx.finalize_weights()
        return self

    # ---- LoRA adapters (an extension, DESIGN.md §7 f8): merged into the packed weights, shared by every sample of a call
    def load_lora(self, path, adapter: int, multiplier: float = 1.0):
        """Reads a kohya or diffusers/PEFT .safetensors LoRA file into adapter id `adapter` (>= 0, not in use) and applies it."""
        from .lora import lora_terms, read_safetensors
        if int(adapter) in self.ctx.lora_adapters():
            raise ValueError(f"load_lora: adapter {adapter} is in use: unload_lora({adapter}) first or pick another id")
        terms = lora_terms(read_safetensors(path))
        if not terms:
            raise ValueError(f"{path}: no LoRA terms")
        try:
            for reg, down, up, alpha in terms:
                self.ctx.lora_add(adapter, reg, down, up, alpha)
            self.ctx.lora_scale(adapter, multiplier)
        except Exception:
            # the adapter is new: removing it undoes every add, and nothing else that is pending gets applied
            if int(adapter) in self.ctx.lora_adapters():
                self.ctx.lora_remove(adapter)
            raise
        self.ctx.lora_apply()
        return self

    def set_lora_scale(self, adapter: int, multiplier: float):
        """Rescales a loaded adapter (0 disables it and keeps it loaded) and applies the change."""
        self.ctx.lora_scale(adapter, multiplier)
        self.ctx.lora_apply()
        return self

    def unload_lora(self, adapter: int = -1):
        """Removes one adapter (-1: all) and applies the change."""
        self.ctx.lora_remove(adapter)
        self.ctx.lora_apply()
        return self

    # ---- hot path
    # sampler / eta / noise_seed (an extension, DESIGN.md §7 f6): "ddim" (eta in [0, 1]; eta = 0 is the reference's sampler) or
    # "dpmpp_2m" (DPM-Solver++(2M), eta = 0). schedule (f15): "ddim" (the reference's timesteps) or "karras" (the sigma grid of
    # Karras et al. 2022). They hold for the one call; the context's default sampler and schedule are restored after it.
    @contextlib.contextmanager
    def _sampler(self, sampler, eta, noise_seed, schedule="ddim"):
        self.ctx.set_sampler(sampler, eta, noise_seed)
        try:
            self.ctx.set_schedule(schedule)
            yield
        finally:
            self.ctx.set_sampler(0, 0.0, 0)
            self.ctx.set_schedule(0)

    def sample_image(self, context, unconditional_context, unconditional_guidance_scale: float, n_steps: int,
                     init_latent=None, seed: int = 0, height: int = 512, width: int = 512, sampler: str = "ddim",
                     eta: float = 0.0, noise_seed: int = 0, schedule: str = "ddim"):
        """-> list of n flat uint8 arrays of H*W*3 (HWC RGB), like the reference's Vec<Vec<u8>>."""
        with self._sampler(sampler, eta, noise_seed, schedule):
            rgb = self.ctx.sample_image(context, unconditional_context, unconditional_guidance_scale, n_steps,
                                        init_latent=init_latent, seed=seed, H=height // 8, W=width // 8)
        return [rgb[i].reshape(-1) for i in range(rgb.shape[0])]

    def sample_latent(self, context, unconditional_context, unconditional_guidance_scale: float, n_steps: int,
                      init_latent=None, seed: int = 0, height: int = 512, width: int = 512, sampler: str = "ddim",
                      eta: float = 0.0, noise_seed: int = 0, schedule: str = "ddim") -> np.ndarray:
        with self._sampler(sampler, eta, noise_seed, schedule):
            return self.ctx.sample_latent(context, unconditional_context, unconditional_guidance_scale, n_steps,
                                          init_latent=init_latent, seed=seed, H=height // 8, W=width // 8)

    def img2img(self, image, context, unconditional_context, unconditional_guidance_scale: float, n_steps: int,
                strength: float, mask=None, noise=None, seed: int = 0, sampler: str = "ddim", eta: float = 0.0,
                noise_seed: int = 0, schedule: str = "ddim"):
        """Image-to-image / masked inpainting (an extension: the reference has none; DESIGN.md §7 f5). image u8
        [n, height, width, 3] HWC RGB, the format sample_image returns; mask u8 [n, height, width] (255 = regenerate,
        0 = keep) or None; strength in (0, 1]. With inpaint=True the mask is required, binary (>= 128 regenerates), and
        conditions the UNet, which sees the masked image, instead of a blend after each step. -> list of n flat uint8 arrays of
        height*width*3, like sample_image."""
        with self._sampler(sampler, eta, noise_seed, schedule):
            rgb = self.ctx.img2img(image, context, unconditional_context, unconditional_guidance_scale, n_steps, strength,
                                   mask=mask, noise=noise, seed=seed)
        return [rgb[i].reshape(-1) for i in range(rgb.shape[0])]

    def edit_image(self, image, context, unconditional_context, guidance_scale: float = 7.5, image_guidance_scale: float = 1.5,
                   n_steps: int = 100, init_latent=None, seed: int = 0, sampler: str = "ddim", eta: float = 0.0,
                   noise_seed: int = 0, schedule: str = "ddim"):
        """InstructPix2Pix editing (pix2pix=True; DESIGN.md §7 f10): image u8 [n, height, width, 3] HWC RGB, the format
        sample_image returns; context [n, L, 768] the instructions; unconditional_context [Lu, 768]. Every step runs the UNet on
        (no image, negative), (image, negative) and (image, instruction) and combines them with guidance_scale (text) and
        image_guidance_scale, the defaults of the original pipeline. -> list of n flat uint8 arrays of height*width*3, like
        sample_image."""
        with self._sampler(sampler, eta, noise_seed, schedule):
            rgb = self.ctx.edit_image(image, context, unconditional_context, guidance_scale, image_guidance_scale, n_steps,
                                      init_latent=init_latent, seed=seed)
        return [rgb[i].reshape(-1) for i in range(rgb.shape[0])]

    # ---- batches of different requests (an extension, DESIGN.md §7 f7): one UNet pass per step for all of them
    def sample_batch(self, contexts, unconditional_contexts, guidance_scales, n_steps: int, seeds, height: int = 512,
                     width: int = 512, sampler: str = "ddim", eta: float = 0.0, noise_seeds=None, schedule: str = "ddim"):
        """contexts: list of n [1, L_i, 768] (what `context` returns; lengths may differ); unconditional_contexts: one [Lu, 768]
        shared by every request or a list of n; guidance_scales: one number or a list of n; seeds: list of n (request i gets the
        image sample_image gives for seeds[i] alone, to rounding); noise_seeds: list of n keying eta > 0 noise per request, or None.
        -> list of n flat uint8 arrays of height*width*3, like sample_image."""
        with self._sampler(sampler, eta, 0, schedule):
            rgb = self.ctx.sample_batch(contexts, unconditional_contexts, guidance_scales, n_steps, seeds=seeds,
                                        noise_seeds=noise_seeds, H=height // 8, W=width // 8)
        return [rgb[i].reshape(-1) for i in range(rgb.shape[0])]

    def img2img_batch(self, images, contexts, unconditional_contexts, guidance_scales, n_steps: int, strength: float,
                      masks=None, seeds=None, noise=None, sampler: str = "ddim", eta: float = 0.0, noise_seeds=None,
                      schedule: str = "ddim"):
        """img2img over a batch of different requests: images u8 [n, height, width, 3]; masks u8 [n, height, width] or None;
        the other arguments as sample_batch. -> list of n flat uint8 arrays of height*width*3."""
        with self._sampler(sampler, eta, 0, schedule):
            rgb = self.ctx.img2img_batch(images, contexts, unconditional_contexts, guidance_scales, n_steps, strength, mask=masks,
                                         noise=noise, seeds=seeds, noise_seeds=noise_seeds)
        return [rgb[i].reshape(-1) for i in range(rgb.shape[0])]

    def latent_to_image(self, latent):
        rgb = self.ctx.latent_to_image(latent)
        return [rgb[i].reshape(-1) for i in range(rgb.shape[0])]

    def close(self):
        self.ctx.close()
