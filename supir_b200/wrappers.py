"""ControlWrapper: the network object the denoiser calls (reference: sgm/modules/diffusionmodules/wrappers.py:68-102).

Same surface — `ControlWrapper(diffusion_model, compile_model=False, dtype=...)`, `.load_control_model(m)`, settable
`.dtype`, `forward(x, t, c, control_scale=1) -> fp32 [B, 4, h, w]`, state_dict keys `diffusion_model.*` / `control_model.*` —
but one call is one CUDA-graph replay: GLVControl + LightGLVUNet are captured once per (batch, h, w, context length) with
static input/output buffers, so the ~2000 kernel launches of a denoiser call cost no Python or launch-API time.

`.dtype` selects the compute dtype of both networks: torch.float16 runs them in fp16 (torch.autocast(float16) numerics, the
reference's default `diffusion_dtype`), torch.bfloat16 in bf16, torch.float8_e4m3fn in bf16 with the transformer blocks'
Linear layers on FP8 tensor cores (nets.py); any other value (fp32) warns and computes bf16. `.fp8_convs = True` (FP8 dtype
only, default False) also runs the ResBlocks' 3x3 convolutions on FP8 tensor cores, and `.fp8_attention = True` (FP8 dtype
only, default False, independent of fp8_convs) the self-attentions and ZeroCrossAttn.
"""
import os
import warnings

import torch
import torch.nn as nn

from . import _native, ops
from .nets import Ctx

_USE_GRAPHS = os.environ.get("SUPIR_B200_NO_GRAPH", "0") != "1"


class _Plan:
    """Static buffers + captured graph for one input signature."""

    def __init__(self, wrapper, B, H, W, Lctx, ctx_dim, y_dim, device):
        self.key = (B, H, W, Lctx)
        self.dtype = wrapper.compute_dtype
        f32 = dict(dtype=torch.float32, device=device)
        self.x = torch.zeros(B, 4, H, W, **f32)
        self.control = torch.zeros(B, 4, H, W, **f32)
        self.t = torch.zeros(B, **f32)
        self.context = torch.zeros(B * Lctx, ctx_dim, **f32)
        self.context_16 = torch.zeros(B * Lctx, ctx_dim, dtype=self.dtype, device=device)      # in the compute dtype
        self.y = torch.zeros(B, y_dim, **f32)
        self.cs = torch.ones(1, **f32)
        self.out = torch.zeros(B, wrapper.diffusion_model.out_channels, H, W, **f32)
        # text K|V projections of both networks: computed OUTSIDE the captured graph, only when the context changes
        # (it is constant over the sampler steps; attention.py:248-251 recomputes it in every call)
        self.kv_ctrl = torch.zeros(B * Lctx, wrapper.control_model._ctx_kv_cols, dtype=self.dtype, device=device)
        self.kv_unet = torch.zeros(B * Lctx, wrapper.diffusion_model._ctx_kv_cols, dtype=self.dtype, device=device)
        self.context_token = None
        self.pool = ops.Pool()
        self.graph = None
        self.B, self.Lctx = B, Lctx
        self.wrapper = wrapper

    def project_context(self):
        w = self.wrapper
        ops.f32_to_16(self.context, self.context_16)
        w.control_model.project_context(self.context_16, self.kv_ctrl)
        w.diffusion_model.project_context(self.context_16, self.kv_unet)

    def _run(self):
        w = self.wrapper
        ctx = Ctx(self.pool, self.B, self.dtype)
        ctx.control_scale = self.cs
        control = w.control_model.run(ctx, self.control, self.t, self.x, self.context_16, self.Lctx, self.y, ctx_kv=self.kv_ctrl)
        w.diffusion_model.run(ctx, self.x, self.t, self.context_16, self.Lctx, self.y, control, self.out, ctx_kv=self.kv_unet)

    def build(self):
        self._run()                      # eager warm-up: one-time attribute setup, fills the scratch pool
        torch.cuda.synchronize()
        if _USE_GRAPHS:
            g = torch.cuda.CUDAGraph()
            n0 = _native.launch_count()
            with torch.cuda.graph(g):
                self._run()
            self.n_launches = _native.launch_count() - n0     # kernels inside one replay
            self.graph = g
        return self

    def launch(self):
        if self.graph is not None:
            self.graph.replay()
            self.wrapper.replayed_launches += self.n_launches
        else:
            self._run()


class ControlWrapper(nn.Module):
    supports_context_token = True       # forward(..., context_token=) — see FusedDenoiser.run_network

    def __init__(self, diffusion_model, compile_model: bool = False, dtype=torch.float32):
        super().__init__()
        self.diffusion_model = diffusion_model
        self.control_model = None
        self._plans = {}                # (B, H, W, Lctx) -> _Plan, most recently used last
        self.max_plans = int(os.environ.get("SUPIR_B200_MAX_PLANS", "4"))   # each plan owns a captured graph + its activation pool
        self._packed = False
        self._warned = False
        self.replayed_launches = 0      # kernels launched through CUDA-graph replays (supir_launch_count() sees eager ones)
        self.dtype = dtype
        self.fp8_convs = False
        self.fp8_attention = False
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate())

    @staticmethod
    def _compute_dtype(dtype):
        """dtype of the activations, plans and pools: fp16 or bf16 (also in the FP8 mode)."""
        return torch.float16 if dtype == torch.float16 else torch.bfloat16

    @classmethod
    def _pack_mode(cls, dtype):
        """What the networks are packed for (nets._UNetBase.pack): the compute dtype, or float8_e4m3fn for the FP8 linears."""
        return ops.FP8 if dtype == ops.FP8 else cls._compute_dtype(dtype)

    @property
    def dtype(self):
        """The requested dtype (`diffusion_dtype`): float16 computes in fp16, float8_e4m3fn in bf16 with FP8 transformer
        linears, anything else in bf16."""
        return self._dtype

    @dtype.setter
    def dtype(self, value):
        old = getattr(self, "_dtype", None)
        self._dtype = value
        if old is not None and self._pack_mode(old) != self._pack_mode(value):
            self.invalidate()           # packed weights and captured graphs are in the old mode: drop them

    @property
    def fp8_convs(self):
        """FP8 mode option: the two 3x3 convolutions of every ResBlock also run on e4m3 operands (nets._UNetBase.pack). Part of
        the pack mode: packing with it under another dtype raises."""
        return self._fp8_convs

    @fp8_convs.setter
    def fp8_convs(self, value):
        old = getattr(self, "_fp8_convs", None)
        self._fp8_convs = bool(value)
        if old is not None and old != self._fp8_convs:
            self.invalidate()           # packed weights and captured graphs are in the old mode: drop them

    @property
    def fp8_attention(self):
        """FP8 mode option: the self-attention of every transformer block and the attention of every ZeroCrossAttn run on e4m3
        operands (nets.attention); the text cross-attention stays bf16. Part of the pack mode: packing with it under another
        dtype raises."""
        return self._fp8_attention

    @fp8_attention.setter
    def fp8_attention(self, value):
        old = getattr(self, "_fp8_attention", None)
        self._fp8_attention = bool(value)
        if old is not None and old != self._fp8_attention:
            self.invalidate()           # packed weights and captured graphs are in the old mode: drop them

    @property
    def compute_dtype(self):
        return self._compute_dtype(self._dtype)

    def load_control_model(self, control_model):
        self.control_model = control_model
        self.invalidate()

    def invalidate(self):
        """Weights changed (load_state_dict / .to()): re-pack and re-capture on the next call."""
        self._plans = {}
        self._packed = False

    def clear_plans(self):
        """Drop every captured graph and its activation pool (several GB each); the next call re-captures."""
        self._plans = {}

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self.invalidate()
        return r

    def pack(self):
        for net in (self.diffusion_model, self.control_model):
            net.pack(self._pack_mode(self._dtype), fp8_convs=self._fp8_convs, fp8_attention=self._fp8_attention)
        self._packed = True
        return self

    @torch.no_grad()
    def forward(self, x: torch.Tensor, t: torch.Tensor, c: dict, control_scale=1, context_token=None, **kwargs) -> torch.Tensor:
        """`context_token` (any hashable, optional) is the caller's name for the CONTENT of c['crossattn']: while consecutive
        calls of one input signature carry the same token, the text K|V projections of the previous call are reused (this
        package's samplers pass a token that is unique per run and batch group — the conditioning is constant over the
        steps). Without a token they are recomputed on every call, like the reference does."""
        if self.control_model is None:
            raise RuntimeError("ControlWrapper.forward called before load_control_model()")
        if not x.is_cuda:
            raise RuntimeError("supir_b200.ControlWrapper needs CUDA tensors: the backend has no CPU path")
        if self.dtype not in (torch.bfloat16, torch.float16, ops.FP8) and not self._warned:
            warnings.warn(f"supir_b200 computes the diffusion networks in bf16, fp16 or fp8; dtype {self.dtype} computes in bf16")
            self._warned = True
        if not self._packed:
            self.pack()
        context, y, control = c.get("crossattn"), c.get("vector"), c.get("control")
        assert (y is not None), "must specify y if and only if the model is class-conditional"
        B, _, H, W = x.shape
        Lctx = context.shape[1]
        key = (B, H, W, Lctx)
        plan = self._plans.get(key)
        if plan is None:
            plan = _Plan(self, B, H, W, Lctx, context.shape[2], y.shape[1], x.device)
            self._fill(plan, x, t, context, y, control, control_scale, context_token)
            plan.build()
            self._plans[key] = plan
            while len(self._plans) > max(self.max_plans, 1):      # least recently used first: frees its graph and pool
                self._plans.pop(next(iter(self._plans)))
        else:
            self._plans[key] = self._plans.pop(key)               # mark as most recently used
            self._fill(plan, x, t, context, y, control, control_scale, context_token)
        plan.launch()
        return plan.out.clone()

    @staticmethod
    def _fill(plan, x, t, context, y, control, control_scale, token=None):
        plan.x.copy_(x)
        plan.control.copy_(control)
        plan.t.copy_(t)
        if token is None or token != plan.context_token:
            plan.context.copy_(context.reshape(plan.context.shape))
            plan.project_context()
            plan.context_token = token
        plan.y.copy_(y)
        if torch.is_tensor(control_scale):
            plan.cs.copy_(control_scale.reshape(-1)[:1])
        else:
            plan.cs.fill_(float(control_scale))
