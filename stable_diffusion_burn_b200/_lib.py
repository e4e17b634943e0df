"""ctypes binding of libsdb200.so (the C ABI declared in include/sdb200.h).

The library is built in-tree by `make -C stable_diffusion_burn_b200/csrc` (see __graft_entry__.build).
There is no fallback: a missing library or a missing GPU raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsdb200.so")

_f32p = C.POINTER(C.c_float)
_u8p = C.POINTER(C.c_uint8)
_i64p = C.POINTER(C.c_int64)
_ctx = C.c_void_p


class SdbBatch(C.Structure):
    """include/sdb200.h: sdb_batch (DESIGN.md §7 f7)."""
    _fields_ = [("n", C.c_int), ("L", C.c_int), ("context", C.c_void_p), ("context_len", C.POINTER(C.c_int32)),
                ("Lu", C.c_int), ("uncond", C.c_void_p), ("uncond_len", C.POINTER(C.c_int32)),
                ("guidance_scale", C.POINTER(C.c_double)), ("seed", C.POINTER(C.c_uint64)),
                ("noise_seed", C.POINTER(C.c_uint64))]


_batchp = C.POINTER(SdbBatch)

# (name, restype, argtypes) — every symbol declared in include/sdb200.h
SIGNATURES = [
    ("sdb_create", C.c_int, [C.c_int, C.POINTER(_ctx)]),
    ("sdb_create_inpaint", C.c_int, [C.c_int, C.POINTER(_ctx)]),
    ("sdb_create_pix2pix", C.c_int, [C.c_int, C.POINTER(_ctx)]),
    ("sdb_destroy", C.c_int, [_ctx]),
    ("sdb_last_error", C.c_char_p, [_ctx]),
    ("sdb_version", C.c_char_p, []),
    ("sdb_tensor_count", C.c_int, [_ctx]),
    ("sdb_tensor_info", C.c_int, [_ctx, C.c_int, C.POINTER(C.c_char_p), _i64p, C.POINTER(C.c_int)]),
    ("sdb_set_tensor", C.c_int, [_ctx, C.c_char_p, _f32p, _i64p, C.c_int]),
    ("sdb_get_tensor", C.c_int, [_ctx, C.c_char_p, _f32p, C.c_int64]),
    ("sdb_init_synthetic", C.c_int, [_ctx, C.c_uint32]),
    ("sdb_weight_arena", C.c_int, [_ctx, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]),
    ("sdb_finalize_weights", C.c_int, [_ctx]),
    ("sdb_unet_forward", C.c_int, [_ctx, _f32p, C.c_int32, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, _f32p]),
    ("sdb_decode_latent", C.c_int, [_ctx, _f32p, C.c_int, C.c_int, C.c_int, _f32p]),
    ("sdb_sample_latent", C.c_int, [_ctx, _f32p, C.c_int, C.c_int, _f32p, C.c_int, C.c_double, C.c_int, _f32p,
                                    C.c_uint64, C.c_int, C.c_int, _f32p]),
    ("sdb_latent_to_image", C.c_int, [_ctx, _f32p, C.c_int, C.c_int, C.c_int, _u8p]),
    ("sdb_sample_image", C.c_int, [_ctx, _f32p, C.c_int, C.c_int, _f32p, C.c_int, C.c_double, C.c_int, _f32p,
                                   C.c_uint64, C.c_int, C.c_int, _u8p]),
    ("sdb_load_dump_dir", C.c_int, [_ctx, C.c_char_p]),
    ("sdb_nccl_unique_id", C.c_int, [C.c_void_p]),
    ("sdb_broadcast_weights", C.c_int, [_ctx, C.c_void_p, C.c_int, C.c_int]),
    ("sdb_forward_diffuser", C.c_int, [_ctx, _f32p, C.c_int32, _f32p, C.c_int, C.c_int, _f32p, C.c_int, C.c_double, C.c_int,
                                       C.c_int, _f32p, _f32p, _f32p]),
    ("sdb_forward_diffuser_dev", C.c_int, [_ctx, C.c_void_p, C.c_int32, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                           C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    ("sdb_test_gemm_ex", C.c_int, [_ctx, _f32p, _f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _f32p, _f32p,
                                   C.c_int, _f32p, C.POINTER(C.c_int32)]),
    ("sdb_read_dump_tensor", C.c_int64, [C.c_char_p, C.c_int, C.POINTER(C.c_int64), _f32p, C.c_int64]),
    ("sdb_load_safetensors", C.c_int, [_ctx, C.c_char_p]),
    ("sdb_probe_safetensors", C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("sdb_encode_image", C.c_int, [_ctx, _f32p, C.c_int, C.c_int, C.c_int, _f32p]),
    ("sdb_encode_image_dev", C.c_int, [_ctx, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    ("sdb_clip_forward", C.c_int, [_ctx, C.POINTER(C.c_int32), C.c_int, C.c_int, _f32p]),
    ("sdb_clip_forward_dev", C.c_int, [_ctx, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    ("sdb_unet_forward_dev", C.c_int, [_ctx, C.c_void_p, C.c_int32, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_void_p, C.c_void_p]),
    ("sdb_decode_latent_dev", C.c_int, [_ctx, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    ("sdb_sample_image_dev", C.c_int, [_ctx, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_int,
                                       C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    ("sdb_img2img", C.c_int, [_ctx, _u8p, _u8p, C.c_double, _f32p, C.c_int, C.c_int, _f32p, C.c_int, C.c_double, C.c_int, _f32p,
                              C.c_uint64, C.c_int, C.c_int, _f32p, _u8p]),
    ("sdb_img2img_dev", C.c_int, [_ctx, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                  C.c_double, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sdb_edit_image", C.c_int, [_ctx, _u8p, _f32p, C.c_int, C.c_int, _f32p, C.c_int, C.c_double, C.c_double, C.c_int, _f32p,
                                 C.c_uint64, C.c_int, C.c_int, _f32p, _u8p]),
    ("sdb_edit_image_dev", C.c_int, [_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_double,
                                     C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sdb_set_sampler", C.c_int, [_ctx, C.c_int, C.c_double, C.c_uint64]),
    ("sdb_set_schedule", C.c_int, [_ctx, C.c_int]),
    ("sdb_unet_forward_at", C.c_int, [_ctx, _f32p, C.c_double, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, _f32p]),
    ("sdb_lora_add", C.c_int, [_ctx, C.c_int, C.c_char_p, C.c_int, _f32p, _f32p, C.c_double]),
    ("sdb_lora_scale", C.c_int, [_ctx, C.c_int, C.c_double]),
    ("sdb_lora_remove", C.c_int, [_ctx, C.c_int]),
    ("sdb_lora_apply", C.c_int, [_ctx]),
    ("sdb_get_merged_tensor", C.c_int, [_ctx, C.c_char_p, _f32p, C.c_int64]),
    ("sdb_sample_batch", C.c_int, [_ctx, _batchp, C.c_int, _f32p, C.c_int, C.c_int, _f32p, _u8p]),
    ("sdb_sample_batch_dev", C.c_int, [_ctx, _batchp, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    ("sdb_img2img_batch", C.c_int, [_ctx, _batchp, _u8p, _u8p, C.c_double, C.c_int, _f32p, C.c_int, C.c_int, _f32p, _u8p]),
    ("sdb_img2img_batch_dev", C.c_int, [_ctx, _batchp, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_int,
                                        C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sdb_set_option", C.c_int, [_ctx, C.c_char_p, C.c_int]),
    ("sdb_profile_enable", C.c_int, [_ctx, C.c_int]),
    ("sdb_profile_reset", C.c_int, [_ctx]),
    ("sdb_profile_class_count", C.c_int, [_ctx]),
    ("sdb_profile_get", C.c_int, [_ctx, C.c_int, C.POINTER(C.c_char_p), _i64p, C.POINTER(C.c_double),
                                  C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    ("sdb_profile_get_issued", C.c_int, [_ctx, C.c_int, C.POINTER(C.c_double)]),
    ("sdb_launch_count", C.c_int64, [_ctx]),
    ("sdb_test_conv2d", C.c_int, [_ctx, _f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_int, C.c_int, C.c_int, _f32p, C.POINTER(C.c_int32)]),
    ("sdb_test_ln_fold", C.c_int, [_ctx, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_int, C.c_int, _f32p, C.POINTER(C.c_int32)]),
    ("sdb_test_conv_groupnorm", C.c_int, [_ctx, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _f32p, C.POINTER(C.c_int),
                                          C.POINTER(C.c_int32)]),
    ("sdb_test_resblock", C.c_int, [_ctx, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p,
                                    C.c_int, C.c_int, _f32p, _f32p, _f32p, C.POINTER(C.c_int32)]),
    ("sdb_test_groupnorm_cat", C.c_int, [_ctx, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _f32p, _f32p,
                                         C.c_int, C.c_int, _f32p, C.POINTER(C.c_int32)]),
    ("sdb_test_spatial_transformer", C.c_int, [_ctx, C.c_int, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, _f32p, C.c_int,
                                               C.POINTER(C.c_int32), C.c_int, _f32p, _f32p, _f32p, _f32p, _f32p,
                                               C.POINTER(C.c_int32)]),
    ("sdb_test_vae_stage", C.c_int, [_ctx, C.c_int, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int,
                                     _f32p, _f32p, _f32p, _f32p, C.POINTER(C.c_int32)]),
    ("sdb_test_clip_block", C.c_int, [_ctx, C.c_int, _f32p, C.c_int, C.c_int, C.c_int, _f32p, _f32p, C.POINTER(C.c_int32)]),
    ("sdb_test_step_noise", C.c_int, [_ctx, C.c_uint64, C.c_int, C.c_int64, _f32p]),
    ("sdb_test_layernorm", C.c_int, [_ctx, _f32p, _f32p, _f32p, C.c_int, C.c_int, _f32p]),
    ("sdb_test_attention", C.c_int, [_ctx, _f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.POINTER(C.c_int32), C.c_int, _f32p]),
]

_lib = None


def load():
    """dlopen the in-tree library and type every entry point. Raises if it was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, res, args in SIGNATURES:
            fn = getattr(lib, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def ptr(a: np.ndarray):
    return a.ctypes.data_as(_f32p)


class SdbError(RuntimeError):
    pass


CKPT_FULL, CKPT_VAE = 0, 1  # include/sdb200.h: SDB_CKPT_FULL, SDB_CKPT_VAE


def probe_safetensors(path):
    """Validates an SD-1.x .safetensors checkpoint without a context or a GPU (include/sdb200.h: sdb_probe_safetensors) ->
    (kind, conv_in_width): (CKPT_FULL, 4 / 8 / 9) or (CKPT_VAE, 0). Raises SdbError naming what is wrong."""
    lib = load()
    kind, width = C.c_int(), C.c_int()
    if lib.sdb_probe_safetensors(os.fsencode(path), C.byref(kind), C.byref(width)) != 0:
        raise SdbError(lib.sdb_last_error(None).decode())
    return kind.value, width.value


def _rows(a, what):
    a = f32(a)
    if a.ndim == 3 and a.shape[0] == 1:
        a = a[0]
    if a.ndim != 2 or a.shape[1] != 768 or a.shape[0] < 1:
        raise ValueError(f"{what} must be [L, 768] or [1, L, 768] with L >= 1, got {a.shape}")
    return a


def pack_batch(contexts, unconds, scales, seeds=None, noise_seeds=None):
    """The arrays of an sdb_batch (DESIGN.md §7 f7) from n requests. contexts: list of [L_i, 768] or [1, L_i, 768]; unconds: one
    [Lu, 768] (or [1, Lu, 768]) array shared by every request, or a list of n; scales: a number or a list of n; seeds,
    noise_seeds: lists of n or None. -> dict of context [n, Lmax, 768] and uncond [n, Lumax, 768] (rows past a request's length
    zero), context_len / uncond_len int32 [n], scale float64 [n], seed / noise_seed uint64 [n] or None."""
    if isinstance(contexts, np.ndarray) or not len(contexts):
        raise ValueError("contexts must be a non-empty list of [L, 768] arrays")
    ctx = [_rows(a, f"contexts[{i}]") for i, a in enumerate(contexts)]
    n = len(ctx)
    if isinstance(unconds, np.ndarray):
        unc = [_rows(unconds, "uncond")] * n
    else:
        unc = [_rows(a, f"unconds[{i}]") for i, a in enumerate(unconds)]
        if len(unc) != n:
            raise ValueError(f"{len(unc)} unconditional contexts for {n} requests")

    def per_request(v, what, dtype):
        if v is None:
            return None
        a = np.array([v] * n if np.ndim(v) == 0 else v, dtype)
        if a.shape != (n,):
            raise ValueError(f"{what} must be one value or a list of {n}, got shape {a.shape}")
        return a

    scale = per_request(scales, "scales", np.float64)
    if scale is None or not np.isfinite(scale).all():
        raise ValueError("scales must be finite")

    def stack(rows):
        out = np.zeros((n, max(a.shape[0] for a in rows), 768), np.float32)
        for i, a in enumerate(rows):
            out[i, :a.shape[0]] = a
        return out, np.array([a.shape[0] for a in rows], np.int32)

    context, context_len = stack(ctx)
    uncond, uncond_len = stack(unc)
    return dict(context=context, context_len=context_len, uncond=uncond, uncond_len=uncond_len, scale=scale,
                seed=per_request(seeds, "seeds", np.uint64), noise_seed=per_request(noise_seeds, "noise_seeds", np.uint64))


def batch_struct(b, context_ptr=None, uncond_ptr=None):
    """An SdbBatch over the arrays of pack_batch (kept alive by the caller). context_ptr / uncond_ptr: device addresses that
    replace the host arrays (the _dev entries)."""
    p = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
    n, L, _ = b["context"].shape
    return SdbBatch(n, L, context_ptr or b["context"].ctypes.data, p(b["context_len"], C.c_int32), b["uncond"].shape[1],
                    uncond_ptr or b["uncond"].ctypes.data, p(b["uncond_len"], C.c_int32), p(b["scale"], C.c_double),
                    p(b["seed"], C.c_uint64), p(b["noise_seed"], C.c_uint64))


def _check_outputs(latent, rgb):
    if not (latent or rgb):
        raise ValueError("request the latent, the image or both")


def _outputs(n, H, W, latent, rgb):
    """the requested outputs: the latent [n,4,H,W] and / or the u8 image [n,8H,8W,3], None for the other"""
    return (np.empty((n, 4, H, W), np.float32) if latent else None,
            np.empty((n, 8 * H, 8 * W, 3), np.uint8) if rgb else None)


def _result(lat, out):
    """a tuple (latent, rgb) when both were requested, else the one that was"""
    if lat is not None and out is not None:
        return lat, out
    return out if lat is None else lat


def _u8ptr(a):
    return None if a is None else a.ctypes.data_as(_u8p)


def _fptr(a):
    return None if a is None else ptr(a)


def _image(image, n=None):
    """u8 [n, 8H, 8W, 3] (n checked when given) -> (the contiguous image, H, W) of the latent"""
    image = np.ascontiguousarray(image, dtype=np.uint8)
    if (image.ndim != 4 or (n is not None and image.shape[0] != n) or image.shape[3] != 3 or image.shape[1] % 8
            or image.shape[2] % 8):
        raise ValueError("image must be u8 [n, 8H, 8W, 3]")
    return image, image.shape[1] // 8, image.shape[2] // 8


def _mask(mask, image):
    if mask is None:
        return None
    mask = np.ascontiguousarray(mask, dtype=np.uint8)
    if mask.shape != image.shape[:3]:
        raise ValueError("mask must be u8 [n, 8H, 8W]")
    return mask


def _latent(a, shape, what):
    """None, or `a` as f32 of `shape` [n, 4, H, W]"""
    if a is None:
        return None
    a = f32(a)
    if a.shape != shape:
        raise ValueError(f"{what} must be [n, 4, H, W]")
    return a


class Context:
    """Owns one sdb_ctx (one CUDA device). inpaint=True: a 9-channel inpainting UNet (sdb_create_inpaint, DESIGN.md §7 f9);
    pix2pix=True: an 8-channel InstructPix2Pix UNet (sdb_create_pix2pix, f10)."""

    def __init__(self, device: int = 0, inpaint: bool = False, pix2pix: bool = False):
        if inpaint and pix2pix:
            raise ValueError("a context is either an inpainting (inpaint=True) or an InstructPix2Pix (pix2pix=True) one, not both")
        self.lib = load()
        h = _ctx()
        create = self.lib.sdb_create_inpaint if inpaint else (self.lib.sdb_create_pix2pix if pix2pix else self.lib.sdb_create)
        rc = create(device, C.byref(h))
        if rc != 0:
            raise SdbError(self.lib.sdb_last_error(None).decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.sdb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc):
        if rc != 0:
            raise SdbError(self.lib.sdb_last_error(self.h).decode())

    # ---- weights
    def tensor_list(self):
        out = []
        n = self.lib.sdb_tensor_count(self.h)
        for i in range(n):
            name = C.c_char_p()
            dims = (C.c_int64 * 4)()
            nd = C.c_int()
            self.check(self.lib.sdb_tensor_info(self.h, i, C.byref(name), dims, C.byref(nd)))
            out.append((name.value.decode(), tuple(int(dims[j]) for j in range(nd.value))))
        return out

    def unet_in_channels(self) -> int:
        """4, 9 on an inpainting context or 8 on an InstructPix2Pix one: read from the registry's unet/input_blocks/conv/weight."""
        if getattr(self, "_cin", None) is None:
            self._cin = next(s[1] for n, s in self.tensor_list() if n == "unet/input_blocks/conv/weight")
        return self._cin

    def set_tensor(self, name, arr):
        a = f32(arr)
        dims = (C.c_int64 * 4)(*a.shape)
        self.check(self.lib.sdb_set_tensor(self.h, name.encode(), ptr(a), dims, a.ndim))

    def get_tensor(self, name, shape):
        a = np.empty(shape, np.float32)
        self.check(self.lib.sdb_get_tensor(self.h, name.encode(), ptr(a), a.size))
        return a

    def init_synthetic(self, seed=0):
        self.check(self.lib.sdb_init_synthetic(self.h, seed))

    def finalize_weights(self):
        self.check(self.lib.sdb_finalize_weights(self.h))

    def weight_arena(self):
        p = C.c_void_p()
        n = C.c_size_t()
        self.check(self.lib.sdb_weight_arena(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def set_option(self, key, value):
        self.check(self.lib.sdb_set_option(self.h, key.encode(), int(value)))

    SAMPLERS = {"ddim": 0, "dpmpp_2m": 1}  # SDB_SAMPLER_DDIM, SDB_SAMPLER_DPMPP_2M

    def set_sampler(self, kind=0, eta=0.0, noise_seed=0):
        """Sampler of every sampling entry until changed (include/sdb200.h: sdb_set_sampler; DESIGN.md §7 f6). kind: 0 / "ddim"
        (eta in [0, 1]) or 1 / "dpmpp_2m" (eta 0). noise_seed keys stochastic DDIM's per-step noise."""
        if isinstance(kind, str):
            if kind not in self.SAMPLERS:
                raise ValueError(f"unknown sampler {kind!r}: one of {', '.join(self.SAMPLERS)}")
            kind = self.SAMPLERS[kind]
        self.check(self.lib.sdb_set_sampler(self.h, int(kind), float(eta), int(noise_seed)))

    SCHEDULES = {"ddim": 0, "karras": 1}  # SDB_SCHEDULE_DDIM, SDB_SCHEDULE_KARRAS

    def set_schedule(self, kind=0):
        """The grid every sampling entry walks until changed (include/sdb200.h: sdb_set_schedule; DESIGN.md §7 f15). kind: 0 /
        "ddim" (the reference's integer timesteps) or 1 / "karras" (the sigma grid of Karras et al. 2022, rho = 7)."""
        if isinstance(kind, str):
            if kind not in self.SCHEDULES:
                raise ValueError(f"unknown schedule {kind!r}: one of {', '.join(self.SCHEDULES)}")
            kind = self.SCHEDULES[kind]
        self.check(self.lib.sdb_set_schedule(self.h, int(kind)))

    # ---- LoRA adapters (include/sdb200.h: sdb_lora_*; DESIGN.md §7 f8)
    def lora_add(self, adapter, tensor, down, up, alpha):
        """One term of adapter `adapter`: registry weight `tensor`, down [r, fan-in] (a conv's [r, in, k, k] is flattened), up
        [out, r] (or [out, r, 1, 1]), alpha. Pending until lora_apply."""
        down = f32(down); up = f32(up)
        r = down.shape[0] if down.ndim else 0
        down = down.reshape(r, -1) if r else down
        up = up.reshape(up.shape[0], -1) if up.ndim else up
        if up.ndim != 2 or up.shape[1] != r:
            raise ValueError(f"lora_add {tensor}: up {up.shape} does not match rank {r} of down {down.shape}")
        if getattr(self, "_shapes", None) is None:  # one registry walk per context, not one per term
            self._shapes = dict(self.tensor_list())
        shape = self._shapes.get(tensor)
        if shape is not None:
            out, fan_in = (shape[1], shape[0]) if len(shape) == 2 else (shape[0], int(np.prod(shape[1:])))
            if down.shape[1] != fan_in or up.shape[0] != out:
                raise ValueError(f"lora_add {tensor}: down {down.shape} / up {up.shape} do not fit a weight of {out} outputs "
                                 f"and fan-in {fan_in}")
        self.check(self.lib.sdb_lora_add(self.h, int(adapter), tensor.encode(), int(r), ptr(down), ptr(up), float(alpha)))
        self._lora_ids = self.lora_adapters() | {int(adapter)}

    def lora_scale(self, adapter, multiplier):
        self.check(self.lib.sdb_lora_scale(self.h, int(adapter), float(multiplier)))

    def lora_remove(self, adapter=-1):
        self.check(self.lib.sdb_lora_remove(self.h, int(adapter)))
        self._lora_ids = set() if int(adapter) == -1 else self.lora_adapters() - {int(adapter)}

    def lora_adapters(self) -> set:
        """Ids of the adapters added through this Context and not removed."""
        return set(getattr(self, "_lora_ids", ()))

    def lora_apply(self):
        self.check(self.lib.sdb_lora_apply(self.h))

    def get_merged_tensor(self, name, shape):
        a = np.empty(shape, np.float32)
        self.check(self.lib.sdb_get_merged_tensor(self.h, name.encode(), ptr(a), a.size))
        return a

    # ---- hot path (host buffers)
    def unet_forward(self, x, t, context):
        """x [n,4,H,W] ([n,9,H,W] = latent | mask | masked-image latent on an inpainting context, [n,8,H,W] = latent | image
        latent on an InstructPix2Pix one) -> [n,4,H,W]."""
        x = f32(x); context = f32(context)
        n, ch, H, W = x.shape
        if ch != self.unet_in_channels():
            raise ValueError(f"x has {ch} channels; this context's UNet takes {self.unet_in_channels()}")
        L = context.shape[1]
        out = np.empty((n, 4, H, W), np.float32)
        self.check(self.lib.sdb_unet_forward(self.h, ptr(x), int(t), ptr(context), n, H, W, L, ptr(out)))
        return out

    def unet_forward_at(self, x, t, context):
        """unet_forward at a real timestep t (finite, in [0, 999], rounded once to float32); at an integer t the same bits."""
        x = f32(x); context = f32(context)
        n, ch, H, W = x.shape
        if ch != self.unet_in_channels():
            raise ValueError(f"x has {ch} channels; this context's UNet takes {self.unet_in_channels()}")
        out = np.empty((n, 4, H, W), np.float32)
        self.check(self.lib.sdb_unet_forward_at(self.h, ptr(x), float(t), ptr(context), n, H, W, context.shape[1], ptr(out)))
        return out

    def forward_diffuser(self, latent, t, context, uncond, scale):
        """latent [n,4,H,W] ([n,9,H,W] on an inpainting context) -> (pred, uncond UNet output, cond UNet output), each
        [n,4,H,W]."""
        latent = f32(latent); context = f32(context); uncond = f32(uncond)
        n, ch, H, W = latent.shape
        if ch != self.unet_in_channels():
            raise ValueError(f"latent has {ch} channels; this context's UNet takes {self.unet_in_channels()}")
        outs = [np.empty((n, 4, H, W), np.float32) for _ in range(3)]
        self.check(self.lib.sdb_forward_diffuser(self.h, ptr(latent), int(t), ptr(context), n, context.shape[1], ptr(uncond),
                                                 uncond.shape[0], float(scale), H, W, ptr(outs[0]), ptr(outs[1]), ptr(outs[2])))
        return tuple(outs)

    def nccl_unique_id(self) -> bytes:
        buf = C.create_string_buffer(128)
        if self.lib.sdb_nccl_unique_id(buf) != 0:
            raise SdbError(self.lib.sdb_last_error(None).decode())
        return buf.raw

    def broadcast_weights(self, unique_id: bytes, rank: int, world: int):
        self.check(self.lib.sdb_broadcast_weights(self.h, C.create_string_buffer(unique_id, 128), rank, world))

    def load_dump_dir(self, path):
        self.check(self.lib.sdb_load_dump_dir(self.h, os.fsencode(path)))

    def load_safetensors(self, path):
        """An SD-1.x single-file checkpoint or a VAE-only file (include/sdb200.h: sdb_load_safetensors); finalize_weights
        afterwards."""
        self.check(self.lib.sdb_load_safetensors(self.h, os.fsencode(path)))

    def encode_image(self, img):
        a = f32(img)
        n, ch, H, W = a.shape
        assert ch == 3
        out = np.empty((n, 4, H // 8, W // 8), np.float32)
        self.check(self.lib.sdb_encode_image(self.h, ptr(a), n, H, W, ptr(out)))
        return out

    def clip_forward(self, tokens):
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        if t.ndim == 1:
            t = t[None]
        n, L = t.shape
        out = np.empty((n, L, 768), np.float32)
        self.check(self.lib.sdb_clip_forward(self.h, t.ctypes.data_as(C.POINTER(C.c_int32)), n, L, ptr(out)))
        return out

    def decode_latent(self, latent):
        latent = f32(latent)
        n, _, H, W = latent.shape
        img = np.empty((n, 3, 8 * H, 8 * W), np.float32)
        self.check(self.lib.sdb_decode_latent(self.h, ptr(latent), n, H, W, ptr(img)))
        return img

    def sample_latent(self, context, uncond, scale, n_steps, init_latent=None, seed=0, H=64, W=64):
        context = f32(context); uncond = f32(uncond)
        n, L, _ = context.shape
        Lu = uncond.shape[0]
        if init_latent is not None:
            init_latent = f32(init_latent)
            H, W = init_latent.shape[2:]
        out = np.empty((n, 4, H, W), np.float32)
        self.check(self.lib.sdb_sample_latent(self.h, ptr(context), n, L, ptr(uncond), Lu, float(scale), int(n_steps),
                                              ptr(init_latent) if init_latent is not None else None, seed, H, W, ptr(out)))
        return out

    def latent_to_image(self, latent):
        latent = f32(latent)
        n, _, H, W = latent.shape
        rgb = np.empty((n, 8 * H, 8 * W, 3), np.uint8)
        self.check(self.lib.sdb_latent_to_image(self.h, ptr(latent), n, H, W, rgb.ctypes.data_as(_u8p)))
        return rgb

    def sample_image(self, context, uncond, scale, n_steps, init_latent=None, seed=0, H=64, W=64):
        context = f32(context); uncond = f32(uncond)
        n, L, _ = context.shape
        Lu = uncond.shape[0]
        if init_latent is not None:
            init_latent = f32(init_latent)
            H, W = init_latent.shape[2:]
        rgb = np.empty((n, 8 * H, 8 * W, 3), np.uint8)
        self.check(self.lib.sdb_sample_image(self.h, ptr(context), n, L, ptr(uncond), Lu, float(scale), int(n_steps),
                                             ptr(init_latent) if init_latent is not None else None, seed, H, W,
                                             rgb.ctypes.data_as(_u8p)))
        return rgb

    def img2img(self, image, context, uncond, scale, n_steps, strength, mask=None, noise=None, seed=0, latent=False, rgb=True):
        """Image-to-image / masked inpainting (include/sdb200.h: sdb_img2img). image u8 [n,8H,8W,3]; mask u8 [n,8H,8W]
        (255 = regenerate, 0 = keep) or None; noise [n,4,H,W] or None (the seeded stream sample_image starts from). On an
        inpainting context the mask is required and binary (>= 128 regenerates) and conditions the UNet instead of a blend.
        -> the latent [n,4,H,W] and / or the u8 image [n,8H,8W,3]: a tuple (latent, rgb) when both are requested."""
        _check_outputs(latent, rgb)
        image, H, W = _image(image)
        n = image.shape[0]
        context = f32(context); uncond = f32(uncond)
        mask = _mask(mask, image)
        noise = _latent(noise, (n, 4, H, W), "noise")
        lat, out = _outputs(n, H, W, latent, rgb)
        self.check(self.lib.sdb_img2img(self.h, _u8ptr(image), _u8ptr(mask), float(strength), ptr(context), n, context.shape[1],
                                        ptr(uncond), uncond.shape[0], float(scale), int(n_steps), _fptr(noise), int(seed), H, W,
                                        _fptr(lat), _u8ptr(out)))
        return _result(lat, out)

    def edit_image(self, image, context, uncond, text_scale, image_scale, n_steps, init_latent=None, seed=0, latent=False,
                   rgb=True):
        """InstructPix2Pix image editing on an 8-channel context (include/sdb200.h: sdb_edit_image). image u8 [n,8H,8W,3];
        context [n,L,768]; uncond [Lu,768]; init_latent [n,4,H,W] or None (the seeded stream sample_image starts from).
        -> the latent [n,4,H,W] and / or the u8 image [n,8H,8W,3]: a tuple (latent, rgb) when both are requested."""
        _check_outputs(latent, rgb)
        image, H, W = _image(image)
        n = image.shape[0]
        context = f32(context); uncond = f32(uncond)
        if context.ndim != 3 or context.shape[0] != n:
            raise ValueError("context must be [n, L, 768], one prompt per image")
        init_latent = _latent(init_latent, (n, 4, H, W), "init_latent")
        lat, out = _outputs(n, H, W, latent, rgb)
        self.check(self.lib.sdb_edit_image(self.h, _u8ptr(image), ptr(context), n, context.shape[1], ptr(uncond), uncond.shape[0],
                                           float(text_scale), float(image_scale), int(n_steps), _fptr(init_latent), int(seed), H, W,
                                           _fptr(lat), _u8ptr(out)))
        return _result(lat, out)

    def sample_batch(self, contexts, unconds, scales, n_steps, seeds=None, noise_seeds=None, init_latent=None, H=64, W=64,
                     latent=False, rgb=True):
        """n different requests in one call (include/sdb200.h: sdb_sample_batch; pack_batch for the arguments). init_latent
        [n,4,H,W] or None (each request's latent from its seed). -> the latent [n,4,H,W] and / or the u8 image [n,8H,8W,3]: a
        tuple (latent, rgb) when both are requested."""
        _check_outputs(latent, rgb)
        b = pack_batch(contexts, unconds, scales, seeds, noise_seeds)
        n = b["context"].shape[0]
        if init_latent is not None:
            init_latent = f32(init_latent)
            if init_latent.ndim != 4 or init_latent.shape[:2] != (n, 4):
                raise ValueError("init_latent must be [n, 4, H, W]")
            H, W = init_latent.shape[2:]
        lat, out = _outputs(n, H, W, latent, rgb)
        self.check(self.lib.sdb_sample_batch(self.h, C.byref(batch_struct(b)), int(n_steps), _fptr(init_latent), H, W, _fptr(lat),
                                             _u8ptr(out)))
        return _result(lat, out)

    def img2img_batch(self, image, contexts, unconds, scales, n_steps, strength, mask=None, noise=None, seeds=None,
                      noise_seeds=None, latent=False, rgb=True):
        """n different requests of image-to-image / inpainting in one call (include/sdb200.h: sdb_img2img_batch). image u8
        [n,8H,8W,3]; mask u8 [n,8H,8W] or None (required on an inpainting context); noise [n,4,H,W] or None (each request's
        noise from its seed)."""
        _check_outputs(latent, rgb)
        b = pack_batch(contexts, unconds, scales, seeds, noise_seeds)
        n = b["context"].shape[0]
        image, H, W = _image(image, n)
        mask = _mask(mask, image)
        noise = _latent(noise, (n, 4, H, W), "noise")
        lat, out = _outputs(n, H, W, latent, rgb)
        self.check(self.lib.sdb_img2img_batch(self.h, C.byref(batch_struct(b)), _u8ptr(image), _u8ptr(mask), float(strength),
                                              int(n_steps), _fptr(noise), H, W, _fptr(lat), _u8ptr(out)))
        return _result(lat, out)

    # ---- profiling
    def profile(self, on=True):
        self.check(self.lib.sdb_profile_enable(self.h, 1 if on else 0))

    def profile_reset(self):
        self.check(self.lib.sdb_profile_reset(self.h))

    def profile_table(self):
        rows = {}
        for i in range(self.lib.sdb_profile_class_count(self.h)):
            name = C.c_char_p(); ln = C.c_int64(); ms = C.c_double(); fl = C.c_double(); by = C.c_double()
            self.check(self.lib.sdb_profile_get(self.h, i, C.byref(name), C.byref(ln), C.byref(ms), C.byref(fl), C.byref(by)))
            iss = C.c_double()
            self.check(self.lib.sdb_profile_get_issued(self.h, i, C.byref(iss)))
            rows[name.value.decode()] = dict(launches=ln.value, ms=ms.value, flops=fl.value, bytes=by.value, issued_flops=iss.value)
        return rows

    def launch_count(self):
        return int(self.lib.sdb_launch_count(self.h))

    # ---- single-kernel test entries
    # The traced entries fill SDB_TRACE_INTS ints with one 16-int record per launch (include/sdb200.h); _decode_trace turns them
    # into the lists of the record kinds an entry launches, in launch order. The GEMM entries take trace=True to also return
    # their "gemms" list.
    TRACE_INTS = 1024
    _TRACE_KINDS = {1: "gemms", 2: "attn", 3: "gn", 4: "conv", 5: "softmax", 6: "cond_mod"}
    _GEMM_TRACE_KEYS = ("kind", "N", "BN", "split", "TN", "TH", "TW", "xk", "gn_slots", "a1", "passes", "epi", "act", "stages")
    _ATTN_TRACE_KEYS = ("dpad", "Nq", "Nk", "qk3", "kvlen")
    _EPI_ROLES = ("lns", "lnc", "geglu", "res16", "res32", "gn")
    _GN_PATHS = {1: "fused", 2: "apply", 3: "apply+fold", 4: "sums:stats", 5: "sums:partials", 6: "sums:fold"}

    @staticmethod
    def _trace_buf(trace=True):
        if not trace:
            return None, None
        t = np.zeros(Context.TRACE_INTS, np.int32)
        return t, t.ctypes.data_as(C.POINTER(C.c_int32))

    @classmethod
    def _decode_trace(cls, t, kinds):
        """-> {kind: entries} for the record kinds `kinds` of _TRACE_KINDS the entry launches (a record of another kind is an
        error): "gemms": dicts of _GEMM_TRACE_KEYS with "epi" as the set of _EPI_ROLES names; "attn": dicts of _ATTN_TRACE_KEYS,
        plus causal=1 on a causal launch; "gn": _GN_PATHS names; "conv": (rows per tile, channels per round, channel groups);
        "softmax": values per thread; one entry per launch. "cond_mod": m of the one conditioned conv_in, 0 without one."""
        tr = {k: 0 if k == "cond_mod" else [] for k in kinds}
        for i in range(int(t[0])):
            kind, *f = (int(v) for v in t[1 + 16 * i:17 + 16 * i])
            name = cls._TRACE_KINDS.get(kind)
            if name not in tr:
                raise ValueError(f"trace record {i}: kind {kind} is not one of {kinds}")
            if name == "cond_mod":
                if tr[name]:
                    raise ValueError("trace: more than one conditioned conv_in")
                tr[name] = f[0]
                continue
            if kind == 1:
                rec = dict(zip(cls._GEMM_TRACE_KEYS, f))
                rec["epi"] = {r for b, r in enumerate(cls._EPI_ROLES) if rec["epi"] >> b & 1}
            elif kind == 2:
                rec = dict(zip(cls._ATTN_TRACE_KEYS, f))
                if f[5]:
                    rec["causal"] = f[5]
            elif kind == 3:
                rec = cls._GN_PATHS[f[0]]
            elif kind == 4:
                rec = tuple(f[:3])
            else:
                rec = f[0]
            tr[name].append(rec)
        return tr

    def test_linear(self, a, w, bias=None, passes=1, trace=False):
        """The plain Linear product a w (+ bias), fp32 out: test_gemm_ex without its other epilogues and K-loop forms."""
        return self.test_gemm_ex(a, w, bias, passes=passes, trace=trace)

    def test_gemm_ex(self, a, w, bias=None, residual=None, passes=1, geglu=False, from_f16=False, xa=None, xw=None,
                     planes=False, trace=False):
        """planes: return the fp16 outputs as the pair (hi, lo) of float arrays instead of hi + lo (implies from_f16)."""
        a = f32(a); w = f32(w)
        M, K = a.shape; N = w.shape[1]
        shape = (M, N // 2 if geglu else N)
        out = np.empty((2, *shape) if planes else shape, np.float32)
        opt = lambda v: (None, None) if v is None else (f32(v), ptr(f32(v)))
        keep = [opt(bias), opt(residual), opt(xa), opt(xw)]
        for i, (arr, _) in enumerate(keep):  # keep the contiguous copies alive across the call
            if arr is not None:
                keep[i] = (arr, ptr(arr))
        XK = 0 if xa is None else keep[2][0].shape[1]
        flags = (1 if geglu else 0) | (4 if (from_f16 or planes) else 0) | (8 if planes else 0)
        t, tp = self._trace_buf(trace)
        self.check(self.lib.sdb_test_gemm_ex(self.h, ptr(a), ptr(w), keep[0][1], keep[1][1], M, K, N, passes, flags, keep[2][1],
                                             keep[3][1], XK, ptr(out), tp))
        res = (out[0], out[1]) if planes else out
        return (res, self._decode_trace(t, ("gemms",))["gemms"]) if trace else res

    def test_conv2d(self, x, w, bias=None, stride=1, upsample=0, passes=1, trace=False):
        x = f32(x); w = f32(w)
        n, cin, H, W = x.shape
        cout, _, k, _ = w.shape
        Ho = 2 * H if upsample else (H // 2 if stride == 2 else H)
        Wo = 2 * W if upsample else (W // 2 if stride == 2 else W)
        y = np.empty((n, cout, Ho, Wo), np.float32)
        b = f32(bias) if bias is not None else None
        t, tp = self._trace_buf(trace)
        self.check(self.lib.sdb_test_conv2d(self.h, ptr(x), ptr(w), ptr(b) if b is not None else None, n, cin, H, W, cout,
                                            k, stride, upsample, passes, ptr(y), tp))
        return (y, self._decode_trace(t, ("gemms",))["gemms"]) if trace else y

    def test_ln_fold(self, a, w0, b0, gamma, beta, w1, b1=None, a2=None, passes=3, geglu=False, trace=False):
        a, w0, b0, gamma, beta, w1 = (f32(v) for v in (a, w0, b0, gamma, beta, w1))
        b1 = f32(b1) if b1 is not None else None
        a2 = f32(a2) if a2 is not None else None
        M, K0 = a.shape; Cc = w0.shape[1]; N = w1.shape[1]
        out = np.empty((M, N // 2 if geglu else N), np.float32)
        t, tp = self._trace_buf(trace)
        self.check(self.lib.sdb_test_ln_fold(self.h, ptr(a), ptr(a2) if a2 is not None else None, ptr(w0), ptr(b0), ptr(gamma),
                                             ptr(beta), ptr(w1), ptr(b1) if b1 is not None else None, M, K0, Cc, N, passes,
                                             1 if geglu else 0, ptr(out), tp))
        return (out, self._decode_trace(t, ("gemms",))["gemms"]) if trace else out

    def test_conv_groupnorm(self, x, w, bias, gamma, beta, passes=3, silu=False, stride=1, upsample=0, trace=False):
        x = f32(x); w = f32(w); bias = f32(bias); gamma = f32(gamma); beta = f32(beta)
        n, cin, H, W = x.shape
        cout, _, k, _ = w.shape
        Ho = 2 * H if upsample else (H // 2 if stride == 2 else H)
        Wo = 2 * W if upsample else (W // 2 if stride == 2 else W)
        y = np.empty((n, cout, Ho, Wo), np.float32)
        slots = C.c_int()
        t, tp = self._trace_buf(trace)
        self.check(self.lib.sdb_test_conv_groupnorm(self.h, ptr(x), ptr(w), ptr(bias), ptr(gamma), ptr(beta), n, cin, H, W, cout, k,
                                                    stride, upsample, passes, 1 if silu else 0, ptr(y), C.byref(slots), tp))
        return (y, slots.value, self._decode_trace(t, ("gemms",))["gemms"]) if trace else (y, slots.value)

    def test_resblock(self, x0, x1, norm1, conv1, norm2, conv2, skip=None, emb_bias=None, passes=1, x0_stats=True,
                      x1_stats=True):
        """One ResBlock (emb_bias given) or VAE ResnetBlock (emb_bias None) on cat([x0, x1]); norm* = (gamma, beta),
        conv* / skip = (weight OIHW, bias). -> (out, out16, out_norm, trace): the block output, its fp16 hi + lo copy,
        SiLU(GroupNorm(out; norm2)) from the statistics conv2 left, and what ran (_decode_trace, plus "skip": "merged" |
        "separate" | "none")."""
        x0 = f32(x0)
        n, c0, H, W = x0.shape
        x1 = f32(x1) if x1 is not None else None
        c1 = 0 if x1 is None else x1.shape[1]
        cout = conv1[0].shape[0]
        keep = [f32(v) for v in (*norm1, *conv1, *norm2, *conv2)]
        sk = [f32(v) for v in skip] if skip is not None else [None, None]
        eb = f32(emb_bias) if emb_bias is not None else None
        p = lambda a: None if a is None else ptr(a)
        out, out16, outn = (np.empty((n, cout, H, W), np.float32) for _ in range(3))
        t, tp = self._trace_buf()
        flags = (1 if x0_stats else 0) | (2 if (x1 is not None and x1_stats) else 0)
        self.check(self.lib.sdb_test_resblock(self.h, ptr(x0), p(x1), n, c0, c1, H, W, cout, *(ptr(a) for a in keep), p(sk[0]),
                                              p(sk[1]), p(eb), passes, flags, ptr(out), ptr(out16), ptr(outn), tp))
        tr = self._decode_trace(t, ("gn", "gemms"))
        g = tr["gemms"]
        tr["skip"] = "separate" if len(g) == 3 else ("merged" if g and g[-1]["xk"] > 0 else "none")
        return out, out16, outn, tr

    def test_groupnorm_cat(self, x0, x1, gamma, beta, silu=False, mode=1):
        """GroupNorm(+SiLU) of cat([x0, x1]) as the fp16 hi + lo operand. mode 1: fused kernel, 2: apply from identity-producer
        partials (inputs pass as hi + lo). -> (y NCHW, trace)"""
        x0 = f32(x0)
        n, c0, H, W = x0.shape
        x1 = f32(x1) if x1 is not None else None
        c1 = 0 if x1 is None else x1.shape[1]
        g = f32(gamma); b = f32(beta)
        y = np.empty((n, c0 + c1, H, W), np.float32)
        t, tp = self._trace_buf()
        self.check(self.lib.sdb_test_groupnorm_cat(self.h, ptr(x0), None if x1 is None else ptr(x1), n, c0, c1, H, W, ptr(g), ptr(b),
                                                   1 if silu else 0, int(mode), ptr(y), tp))
        return y, self._decode_trace(t, ("gn", "gemms"))

    def test_spatial_transformer(self, index, x, context, lens, act16=True):
        """The UNet's SpatialTransformer number `index` (execution order, 0..15) on its finalized weights. x [n, C, H, W];
        context [n, Lmax, 768] with per-sample lengths lens [n]. -> dict: out, out16 (its fp16 hi + lo copy, zero unless act16),
        out_norm = SiLU(GroupNorm(out; the block's norm)), y [4, n*H*W, C] (the residual stream after proj_in, attn1, attn2, MLP),
        ln [3, n*H*W, 2] (the row sums norm1..3 read), trace (_decode_trace)."""
        x = f32(x); context = f32(context)
        n, c, H, W = x.shape
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        assert context.shape[0] == n and context.shape[2] == 768 and lens.shape == (n,)
        out, out16, outn = (np.empty((n, c, H, W), np.float32) for _ in range(3))
        y = np.empty((4, n * H * W, c), np.float32)
        ln = np.empty((3, n * H * W, 2), np.float32)
        t, tp = self._trace_buf()
        self.check(self.lib.sdb_test_spatial_transformer(self.h, int(index), ptr(x), n, c, H, W, ptr(context), context.shape[1],
                                                         lens.ctypes.data_as(C.POINTER(C.c_int32)), 1 if act16 else 0, ptr(out),
                                                         ptr(out16), ptr(outn), ptr(y), ptr(ln), tp))
        return dict(out=out, out16=out16, out_norm=outn, y=y, ln=ln, trace=self._decode_trace(t, ("gn", "gemms", "attn")))

    # sdb_test_vae_stage stages (include/sdb200.h: SDB_VAE_*): name -> (stage, input channels, output channels)
    VAE_STAGES = {"dec_in": (0, 4, 512), "dec_attn": (1, 512, 512), "enc_attn": (2, 512, 512), "dec_out": (3, 128, 3),
                  "unet_out": (4, 320, 4), "enc_out": (5, 512, 8), "enc_in": (6, 4, 128), "unet_in": (7, 4, 320),
                  "enc_down0": (8, 128, 128), "enc_down1": (9, 256, 256), "enc_down2": (10, 512, 512)}

    def test_vae_stage(self, stage, x, cond=None, scale=1.0, stats=True, quant=None):
        """One autoencoder stage (or the UNet's conv_in / out conv) on the finalized weights, by name of VAE_STAGES. x
        [n, c, H, W]; cond [n, cin - 4, H, W] for "unet_in" on a 9- / 8-channel context; scale: the decoder conv_in's pre-scale, or
        the strided quant slice's scale; stats: x carries producer GroupNorm partials; quant ("enc_out" only): None for the plain
        quant slice, or an [n, 5, H, W] array the strided + scaled slice writes channels 1-4 of (the rest is kept).
        -> dict: out [n, cout, Ho, Wo]; out16 (its fp16 hi + lo copy, "unet_in"); tap (the attention output before proj_out, or
        the quant slice's output); out_norm (the next ResnetBlock's norm1 operand); trace (_decode_trace)."""
        sid, cin, cout = self.VAE_STAGES[stage]
        x = f32(x)
        n, c, H, W = x.shape
        down = stage.startswith("enc_down")
        Ho, Wo = (H // 2, W // 2) if down else (H, W)
        out = np.empty((n, cout, Ho, Wo), np.float32)
        out16 = np.zeros((n, cout, Ho, Wo), np.float32) if stage == "unet_in" else None
        out_norm = np.zeros((n, cout, Ho, Wo), np.float32) if (down or stage.endswith("attn")) else None
        tap = None
        if stage.endswith("attn"):
            tap = np.zeros((n, 512, H, W), np.float32)
        elif stage == "enc_out":
            tap = np.zeros((n, 4, H, W), np.float32) if quant is None else f32(quant).copy()
            assert quant is None or tap.shape == (n, 5, H, W)
        cnd = f32(cond) if cond is not None else None
        t, tp = self._trace_buf()
        p = lambda a: None if a is None else ptr(a)
        flags = (1 if stats else 0) | (2 if quant is not None else 0)
        self.check(self.lib.sdb_test_vae_stage(self.h, sid, ptr(x), p(cnd), n, c, H, W, float(scale), flags, ptr(out), p(out16),
                                               p(tap), p(out_norm), tp))
        return dict(out=out, out16=out16, tap=tap, out_norm=out_norm,
                    trace=self._decode_trace(t, ("gn", "gemms", "conv", "softmax", "cond_mod")))

    CLIP_TAPS = ("ln1", "q", "k", "v", "o", "x_attn", "ln2", "h")

    def test_clip_block(self, index, x, junk=False, taps=True):
        """CLIP block `index` (0..11), or the final LayerNorm (12), on the finalized weights. x [n, L, 768] is the residual
        stream entering it; junk: the pad rows of the row pitch hold large finite values instead of zeros. -> dict: out
        [n, L, 768]; the taps of CLIP_TAPS ([n, L, 768], h [n, L, 3072]) unless taps is False or index is 12; trace
        (_decode_trace)."""
        x = f32(x)
        n, L, D = x.shape
        assert D == 768
        out = np.empty((n, L, 768), np.float32)
        tp = np.zeros((11, n, L, 768), np.float32) if taps and index < 12 else None
        t, trp = self._trace_buf()
        self.check(self.lib.sdb_test_clip_block(self.h, int(index), ptr(x), n, L, 1 if junk else 0, ptr(out),
                                                None if tp is None else ptr(tp), trp))
        res = dict(out=out, trace=self._decode_trace(t, ("gemms", "attn")))
        if tp is not None:
            res.update({k: tp[i] for i, k in enumerate(self.CLIP_TAPS[:7])})
            res["h"] = tp[7:].reshape(n, L, 3072)
        return res

    def test_step_noise(self, noise_seed, t, count):
        """stochastic DDIM's noise z at timestep t: the first `count` values (numpy mirror: synth.step_noise)."""
        out = np.empty(int(count), np.float32)
        self.check(self.lib.sdb_test_step_noise(self.h, int(noise_seed), int(t), int(count), ptr(out)))
        return out

    def test_layernorm(self, x, gamma, beta):
        x = f32(x); rows, c = x.shape
        y = np.empty_like(x)
        g = f32(gamma); b = f32(beta)
        self.check(self.lib.sdb_test_layernorm(self.h, ptr(x), ptr(g), ptr(b), rows, c, ptr(y)))
        return y

    def test_attention(self, q, k, v, heads, kvlen=None, causal=False, v_transposed=False):
        """kvlen: per-sample key counts (None = all Nk keys); causal: key j visible to query i only if j <= i;
        v_transposed: the CLIP layout (V^T, single fp16 q / k)."""
        q = f32(q); k = f32(k); v = f32(v)
        n, Nq, Cc = q.shape; Nk = k.shape[1]
        out = np.empty_like(q)
        lens = None if kvlen is None else np.ascontiguousarray(kvlen, dtype=np.int32)
        assert lens is None or lens.shape == (n,), "kvlen needs one length per sample"
        flags = (1 if causal else 0) | (2 if v_transposed else 0)
        self.check(self.lib.sdb_test_attention(self.h, ptr(q), ptr(k), ptr(v), n, Nq, Nk, Cc, heads,
                                               None if lens is None else lens.ctypes.data_as(C.POINTER(C.c_int32)), flags,
                                               ptr(out)))
        return out
