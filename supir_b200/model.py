"""SUPIRModel engine on the H100 backend (reference: SUPIR/models/SUPIR_model.py:12-179 on top of
sgm/models/diffusion.py:22-83).

The reference keeps this layer as Python orchestration (stage-1 encode/decode, conditioning, sampler call, decode); it is
the CALLER of the hot path. This class offers the same constructor keys (so `options/SUPIR_v0*.yaml` instantiates it
through supir_b200.config) and the same methods, wired to this package's networks, samplers and VAE. The text conditioner
(SURVEY.md §8(f)2) resolves to supir_b200.conditioner (kernel-backed CLIP-L / bigG text towers with the reference's state_dict
keys); without a CLIP BPE vocabulary on disk, hand token ids to the embedders or `c` / `uc` dictionaries to `batchify_sample`.
"""
import copy
import random

import numpy as np
import torch
import torch.nn as nn

from .config import get_obj_from_str, instantiate_from_config
from .sampling import FusedDenoiser
from .vae import DiagonalGaussianDistribution, VAEHook


def _get(cfg, key, default=None):
    return cfg.get(key, default) if hasattr(cfg, "get") else getattr(cfg, key, default)


class SUPIRModel(nn.Module):
    def __init__(self, control_stage_config, network_config, denoiser_config, first_stage_config, conditioner_config=None,
                 sampler_config=None, network_wrapper=None, ae_dtype="fp32", diffusion_dtype="fp32", scale_factor=1.0,
                 p_p="", n_p="", disable_first_stage_autocast=False, **unused):
        super().__init__()
        wrapper_cls = get_obj_from_str(network_wrapper or "sgm.modules.diffusionmodules.wrappers.ControlWrapper")
        self.model = wrapper_cls(instantiate_from_config(network_config))
        self.model.load_control_model(instantiate_from_config(control_stage_config))
        self.denoiser = instantiate_from_config(denoiser_config)
        self.sampler_config = copy.deepcopy(sampler_config)
        self.sampler = instantiate_from_config(sampler_config) if sampler_config is not None else None
        self.conditioner = None
        if conditioner_config is not None:
            try:
                self.conditioner = instantiate_from_config(conditioner_config)
            except (ImportError, ModuleNotFoundError, AttributeError) as e:  # text encoders live outside this package
                self._conditioner_error = e
        self.first_stage_model = instantiate_from_config(first_stage_config).eval()
        for p in self.first_stage_model.parameters():
            p.requires_grad = False
        self.first_stage_model.denoise_encoder = copy.deepcopy(self.first_stage_model.encoder)
        self.scale_factor = scale_factor
        assert ae_dtype in ("fp32", "fp16", "bf16") and diffusion_dtype in ("fp32", "fp16", "bf16")
        if ae_dtype == "fp16":
            raise RuntimeError("fp16 cause NaN in AE")
        self.ae_dtype = {"fp32": torch.float32, "bf16": torch.bfloat16}[ae_dtype]
        self.model.dtype = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}[diffusion_dtype]
        self.p_p, self.n_p = p_p, n_p
        self._shard_group, self._shard = None, False

    # ---- first stage (SUPIR_model.py:41-69) ----
    @torch.no_grad()
    def encode_first_stage(self, x):
        return self.scale_factor * self.first_stage_model.encode(x)

    @torch.no_grad()
    def encode_first_stage_with_denoise(self, x, use_sample=True, is_stage1=False):
        enc = self.first_stage_model.denoise_encoder_s1 if is_stage1 else self.first_stage_model.denoise_encoder
        posterior = DiagonalGaussianDistribution(self.first_stage_model.quant_conv(enc(x)))
        z = posterior.sample() if use_sample else posterior.mode()
        return self.scale_factor * z

    @torch.no_grad()
    def decode_first_stage(self, z):
        return self.first_stage_model.decode(1.0 / self.scale_factor * z).float()

    @torch.no_grad()
    def batchify_denoise(self, x, is_stage1=False):
        return self.decode_first_stage(self.encode_first_stage_with_denoise(x, use_sample=False, is_stage1=is_stage1))

    def init_tile_vae(self, encoder_tile_size=512, decoder_tile_size=64):
        """SUPIR_model.py:138-150."""
        fs = self.first_stage_model
        for net, size, dec in ((fs.denoise_encoder, encoder_tile_size, False), (fs.encoder, encoder_tile_size, False),
                               (fs.decoder, decoder_tile_size, True)):
            net.forward = VAEHook(net, size, is_decoder=dec, fast_decoder=False, fast_encoder=False, color_fix=False, to_gpu=True)
            net.forward.shard, net.forward.process_group = self._shard, self._shard_group

    def enable_tile_sharding(self, process_group=None, enabled=True):
        """Opt in to sharding ONE image's sampler windows and VAE tiles over the ranks of `process_group` (default: the
        world group). Every rank must call batchify_sample with the same inputs; the seed is broadcast from rank 0 so
        `noised_z` and the per-step noise agree. Without this call torch.distributed is never touched (a data-parallel
        caller with different images per rank is safe)."""
        self._shard, self._shard_group = bool(enabled), process_group
        fs = self.first_stage_model
        for net in (fs.denoise_encoder, fs.encoder, fs.decoder, getattr(fs, "denoise_encoder_s1", None)):
            hook = getattr(net, "forward", None) if net is not None else None
            if isinstance(hook, VAEHook):
                hook.shard, hook.process_group = self._shard, process_group

    def _sharded_world(self):
        import torch.distributed as dist
        return self._shard and dist.is_available() and dist.is_initialized() and dist.get_world_size(self._shard_group) > 1

    # ---- sampling (SUPIR_model.py:79-136) ----
    def make_sampler(self, num_steps, restoration_scale, s_churn, s_noise, cfg_scale, use_linear_CFG, cfg_scale_start):
        cfg = copy.deepcopy(self.sampler_config)
        params = cfg["params"]
        params["num_steps"] = num_steps
        g = params["guider_config"]["params"]
        g["scale_min"] = cfg_scale
        g["scale"] = cfg_scale_start if use_linear_CFG else cfg_scale
        params["restore_cfg"], params["s_churn"], params["s_noise"] = restoration_scale, s_churn, s_noise
        smp = instantiate_from_config(cfg)
        if hasattr(smp, "shard"):
            smp.shard, smp.process_group = self._shard, self._shard_group
        return smp

    def prepare_condition(self, _z, p, p_p, n_p, N):
        if self.conditioner is None:
            raise RuntimeError("no text conditioner is attached (conditioner_config was None or failed to build: "
                               f"{getattr(self, '_conditioner_error', None)!r}): pass c= and uc= to batchify_sample")
        batch = {"original_size_as_tuple": torch.tensor([1024, 1024]).repeat(N, 1).to(_z.device),
                 "crop_coords_top_left": torch.tensor([0, 0]).repeat(N, 1).to(_z.device),
                 "target_size_as_tuple": torch.tensor([1024, 1024]).repeat(N, 1).to(_z.device),
                 "aesthetic_score": torch.tensor([9.0]).repeat(N, 1).to(_z.device), "control": _z}
        batch_uc = copy.deepcopy(batch)
        batch_uc["txt"] = [n_p for _ in p]
        if not isinstance(p[0], list):
            batch["txt"] = ["".join([_p, p_p]) for _p in p]
            return self.conditioner.get_unconditional_conditioning(batch, batch_uc)
        # local prompts: one conditioning per sampler window (SUPIR_model.py:163-176)
        assert len(p) == 1, "Support bs=1 only for local prompt conditioning."
        from .conditioner import GeneralConditioner
        if isinstance(self.conditioner, GeneralConditioner) and N == 1:
            # this package's conditioner treats batch rows independently: ALL window prompts go through the text towers as one
            # batch (225 windows at 8192^2: one pass instead of the reference's 225 x 2), then split into the per-window list
            T = len(p[0])
            rows = lambda v: v.repeat(T, *([1] * (v.dim() - 1)))  # noqa: E731
            batch_t = {k: (rows(v) if torch.is_tensor(v) and k != "control" else v) for k, v in batch.items()}
            batch_t["txt"] = ["".join([p_tile, p_p]) for p_tile in p[0]]
            c_all, uc = self.conditioner.get_unconditional_conditioning(batch_t, batch_uc)
            c = [dict({k: v[i:i + 1] for k, v in c_all.items() if k != "control"}, control=_z) for i in range(T)]
            return c, uc
        c, uc = [], None
        for i, p_tile in enumerate(p[0]):
            batch["txt"] = ["".join([p_tile, p_p])]
            if i == 0:
                _c, uc = self.conditioner.get_unconditional_conditioning(batch, batch_uc)
            else:
                _c, _ = self.conditioner.get_unconditional_conditioning(batch, None)
            c.append(_c)
        return c, uc

    @torch.no_grad()
    def batchify_sample(self, x, p=None, p_p="default", n_p="default", num_steps=100, restoration_scale=4.0, s_churn=0,
                        s_noise=1.003, cfg_scale=4.0, seed=-1, num_samples=1, control_scale=1, color_fix_type="None",
                        use_linear_CFG=False, use_linear_control_scale=False, cfg_scale_start=1.0, control_scale_start=0.0,
                        c=None, uc=None, **kwargs):
        """x: [N, 3, H, W] in [-1, 1]. `c` / `uc` (dicts with 'crossattn' [N,77,2048] and 'vector' [N,2816]) replace the
        text conditioner when given; 'control' is filled in here like prepare_condition does."""
        assert color_fix_type in ["Wavelet", "AdaIn", "None"]
        N = len(x)
        if c is None:
            assert p is not None and len(x) == len(p), "one prompt per image (SUPIR_model.py:86), or pass c= / uc="
        if num_samples > 1:
            assert N == 1
            N = num_samples
            x = x.repeat(N, 1, 1, 1)
            p = p * N if p is not None else p            # SUPIR_model.py:94
        self.sampler = self.make_sampler(num_steps, restoration_scale, s_churn, s_noise, cfg_scale, use_linear_CFG, cfg_scale_start)
        if seed == -1:
            seed = random.randint(0, 65535)
        if self._sharded_world():         # all ranks of a sharded run must draw the same noise: rank 0's seed wins
            import torch.distributed as dist
            box = [seed]
            dist.broadcast_object_list(box, src=dist.get_global_rank(self._shard_group, 0) if self._shard_group is not None else 0,
                                       group=self._shard_group)
            seed = int(box[0])
        random.seed(seed)                  # pytorch_lightning.seed_everything (SUPIR_model.py:115): python, numpy and torch
        np.random.seed(seed)
        torch.manual_seed(seed)
        _z = self.encode_first_stage_with_denoise(x, use_sample=False)
        x_stage1 = self.decode_first_stage(_z)
        z_stage1 = self.encode_first_stage(x_stage1)
        if c is None:
            c, uc = self.prepare_condition(_z, p, self.p_p if p_p == "default" else p_p, self.n_p if n_p == "default" else n_p, N)
        else:
            def with_control(d):
                d = {k: (v.repeat(N // v.shape[0], *([1] * (v.dim() - 1))) if torch.is_tensor(v) and v.shape[0] != N and N % v.shape[0] == 0 else v)
                     for k, v in d.items()}          # num_samples > 1: one conditioning row per sample
                return dict(d, control=_z)
            c = [with_control(ci) for ci in c] if isinstance(c, list) else with_control(c)     # list = local prompts, one per window
            uc = with_control(uc)
        denoiser = FusedDenoiser(self.denoiser, self.model)
        noised_z = torch.randn_like(_z).to(_z.device)
        _samples = self.sampler(denoiser, noised_z, cond=c, uc=uc, x_center=z_stage1, control_scale=control_scale,
                                use_linear_control_scale=use_linear_control_scale, control_scale_start=control_scale_start)
        samples = self.decode_first_stage(_samples)
        if color_fix_type == "Wavelet":
            from .colorfix import wavelet_reconstruction
            samples = wavelet_reconstruction(samples, x_stage1)
        elif color_fix_type == "AdaIn":
            from .colorfix import adaptive_instance_normalization
            samples = adaptive_instance_normalization(samples, x_stage1)
        return samples
