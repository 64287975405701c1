"""Image pre/post-processing around the sampler (reference: SUPIR/util.py:60-94).

`PIL2Tensor` is host-side input preparation (a PIL resize) and is kept as the reference has it. `Tensor2PIL` — bicubic
resize back to the requested size, scale to 0..255, clip, uint8, HWC — sits right after the final VAE decode and runs as one
CUDA kernel (supir_image_to_uint8_bicubic); only the uint8 image crosses PCIe."""
import os

import numpy as np
import torch

from ._native import call
from .ops import _need_cuda, _ptr, _stream


# ----------------------------------------------------------------------------------------------------------------------
# model construction and checkpoint formats (reference: SUPIR/util.py:11-57, 183-191) — the entry points test.py and the
# gradio demos import; usable without a reference checkout (PyYAML instead of OmegaConf, this package's factory)
# ----------------------------------------------------------------------------------------------------------------------
def get_state_dict(d):
    return d.get("state_dict", d)


def load_state_dict(ckpt_path, location="cpu"):
    """.safetensors (sd_xl_base_1.0_0.9vae.safetensors) or a torch pickle, optionally wrapped in {'state_dict': ...}
    (SUPIR-v0Q.ckpt / SUPIR-v0F.ckpt) — SUPIR/util.py:15-24."""
    _, extension = os.path.splitext(ckpt_path)
    if extension.lower() == ".safetensors":
        import safetensors.torch
        state_dict = safetensors.torch.load_file(ckpt_path, device=location)
    else:
        state_dict = get_state_dict(torch.load(ckpt_path, map_location=torch.device(location)))
    return get_state_dict(state_dict)


def create_model(config_path):
    from .config import instantiate_from_config, load_yaml
    return instantiate_from_config(load_yaml(config_path, attr_access=True).model).cpu()


def create_SUPIR_model(config_path, SUPIR_sign=None, load_default_setting=False):
    """SUPIR/util.py:34-51: build `config.model` (every `target:` resolves to this package's classes), then load — each with
    strict=False, in this order — SDXL_CKPT (UNet, VAE and both text towers), SUPIR_CKPT, and the Quality / Fidelity adapter
    checkpoint selected by `SUPIR_sign`."""
    from .config import instantiate_from_config, load_yaml
    config = load_yaml(config_path, attr_access=True)
    model = instantiate_from_config(config.model).cpu()
    if config.get("SDXL_CKPT") is not None:
        model.load_state_dict(load_state_dict(config.SDXL_CKPT), strict=False)
    if config.get("SUPIR_CKPT") is not None:
        model.load_state_dict(load_state_dict(config.SUPIR_CKPT), strict=False)
    if SUPIR_sign is not None:
        assert SUPIR_sign in ["F", "Q"]
        model.load_state_dict(load_state_dict(config.SUPIR_CKPT_F if SUPIR_sign == "F" else config.SUPIR_CKPT_Q), strict=False)
    if load_default_setting:
        return model, config.default_setting
    return model


def load_QF_ckpt(config_path):
    """SUPIR/util.py:53-57 (gradio_demo*.py switch between the two adapter checkpoints at run time)."""
    from .config import load_yaml
    config = load_yaml(config_path, attr_access=True)
    return torch.load(config.SUPIR_CKPT_Q, map_location="cpu"), torch.load(config.SUPIR_CKPT_F, map_location="cpu")


def convert_dtype(dtype_str):
    try:
        return {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16, "fp8": torch.float8_e4m3fn}[dtype_str]
    except KeyError:
        raise NotImplementedError(dtype_str) from None


def _target_size(size, upscale, min_size, fix_resize):
    """Working size (multiples of 64) and requested output size of PIL2Tensor, with the reference's float operation order
    (SUPIR/util.py:65-79): scale, report the rounded size, grow the short side to `min_size`, optionally pin the short side to
    `fix_resize` (which also redefines the reported size), snap to 64."""
    dims = [float(size[0]) * upscale, float(size[1]) * upscale]          # (w, h)
    report = tuple(round(d) for d in dims)
    short = min(dims)
    if short < min_size:
        grow = min_size / short
        dims = [d * grow for d in dims]
    if fix_resize is not None:
        pin = fix_resize / min(dims)
        dims = [d * pin for d in dims]
        report = tuple(round(d) for d in dims)
    work = tuple(int(np.round(d / 64.0)) * 64 for d in dims)
    return work, report


def PIL2Tensor(img, upsacle=1, min_size=1024, fix_resize=None):
    """PIL.Image -> (Tensor[C, H, W] RGB in [-1, 1], h0, w0) — SUPIR/util.py:60-84 (the keyword `upsacle` is the reference's)."""
    from PIL import Image
    (w, h), (w0, h0) = _target_size(img.size, upsacle, min_size, fix_resize)
    pixels = np.array(img.resize((w, h), Image.BICUBIC)).round().clip(0, 255).astype(np.uint8)
    x = torch.tensor(pixels / 255 * 2 - 1, dtype=torch.float32).permute(2, 0, 1)
    return x, h0, w0


def tensor_to_uint8(x, h0, w0):
    """fp32 CUDA tensor [C, H, W] in [-1, 1] -> uint8 CUDA tensor [h0, w0, C] (the arithmetic of Tensor2PIL)."""
    _need_cuda(x)
    x = x.contiguous().float()
    C, H, W = x.shape
    out = torch.empty((h0, w0, C), dtype=torch.uint8, device=x.device)
    call("supir_image_to_uint8_bicubic", _ptr(x), C, H, W, _ptr(out), int(h0), int(w0), _stream())
    return out


def Tensor2PIL(x, h0, w0):
    """Tensor[C, H, W], RGB, [-1, 1] -> PIL.Image (SUPIR/util.py:87-94)."""
    from PIL import Image
    return Image.fromarray(tensor_to_uint8(x, h0, w0).cpu().numpy())


def HWC3(x):
    """uint8 image -> 3 channels (grey replicated, alpha composited over white) — SUPIR/util.py:97-114."""
    assert x.dtype == np.uint8
    if x.ndim == 2:
        x = x[:, :, None]
    assert x.ndim == 3
    C = x.shape[2]
    assert C == 1 or C == 3 or C == 4
    if C == 3:
        return x
    if C == 1:
        return np.concatenate([x, x, x], axis=2)
    color = x[:, :, 0:3].astype(np.float32)
    alpha = x[:, :, 3:4].astype(np.float32) / 255.0
    return (color * alpha + 255.0 * (1.0 - alpha)).clip(0, 255).astype(np.uint8)


def Numpy2Tensor(img):
    """np.array[H, W, C] in [0, 255] -> Tensor[C, H, W], RGB, [-1, 1] (SUPIR/util.py:153-160)."""
    return torch.tensor(np.array(img) / 255 * 2 - 1, dtype=torch.float32).permute(2, 0, 1)


def Tensor2Numpy(x, h0=None, w0=None):
    """Tensor[C, H, W] in [-1, 1] -> uint8 array [H, W, C], bicubic-resized to (h0, w0) when given (SUPIR/util.py:163-172):
    the same kernel as Tensor2PIL (a resize to the tensor's own size is the identity of that kernel's interpolation)."""
    if h0 is None or w0 is None:
        h0, w0 = x.shape[1], x.shape[2]
    return tensor_to_uint8(x, h0, w0).cpu().numpy()
