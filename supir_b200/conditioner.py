"""Text conditioner on the H100 backend (SURVEY.md §8(f)2): `GeneralConditioner` / `GeneralConditionerWithControl`,
`FrozenCLIPEmbedder` (CLIP ViT-L/14 text tower), `FrozenOpenCLIPEmbedder2` (OpenCLIP ViT-bigG/14 text tower) and
`ConcatTimestepEmbedderND` with the reference's class names, constructor parameters, state_dict keys and outputs
(sgm/modules/encoders/modules.py:81-243, 445-609, 1027-1043; wired by options/SUPIR_v0.yaml:66-105).

The reference runs the two towers through third-party packages (transformers==4.28.1 `CLIPTextModel`, open-clip-torch==2.17.1
`open_clip.create_model_and_transforms`) under fp16 autocast, once per image for the positive and once for the negative prompt.
Here the torch modules only OWN the parameters (HF / open_clip key layout, so SUPIR checkpoints and the upstream CLIP weight
files load unchanged) and `forward()` drives this library's kernels: fp32 residual stream like the reference (autocast
lowers only the matmuls), LayerNorm -> bf16, fused QKV projection on the wgmma GEMM, causal attention, out-projection / MLP
GEMMs with fp32 output accumulated into the stream. There is no torch compute fallback.

Tokenisation (host-side string processing) is native too — supir_b200/clip_bpe.py, CLIP's byte-level BPE with the two layouts the
reference feeds its towers — whenever the vocabulary files are at the path the reference configures (CKPT_PTH.SDXL_CLIP1_PATH /
the `version` argument: a Hugging Face directory, or open_clip's bpe_simple_vocab_16e6.txt.gz); the embedders also accept
token-id tensors directly.
"""
import os
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .config import instantiate_from_config
from .ops import BF16

SOT_TOKEN, EOT_TOKEN = 49406, 49407          # <|startoftext|>, <|endoftext|> of the CLIP BPE vocabulary (both towers)

# openai/clip-vit-large-patch14 text_config (the tower behind FrozenCLIPEmbedder's default `version`)
CLIP_L_ARCH = dict(vocab=49408, width=768, heads=12, layers=12, mlp=3072, ctx=77, act="quick_gelu", eps=1e-5)
# open_clip model_configs/<arch>.json text_cfg (FrozenOpenCLIPEmbedder2's `arch`); bigG is what SUPIR_v0.yaml names
OPENCLIP_ARCHS = {
    "ViT-bigG-14": dict(vocab=49408, width=1280, heads=20, layers=32, mlp=5120, ctx=77, proj=1280, act="gelu", eps=1e-5),
    "ViT-H-14": dict(vocab=49408, width=1024, heads=16, layers=24, mlp=4096, ctx=77, proj=1024, act="gelu", eps=1e-5),
}


def _reference_path(name):
    """The reference keeps its weight locations in a top-level CKPT_PTH.py (SDXL_CLIP1_PATH, SDXL_CLIP2_CKPT_PTH) that overrides
    the `version` arguments (modules.py:462-463, 533); honour it when such a module is importable."""
    try:
        import CKPT_PTH
        return getattr(CKPT_PTH, name, None)
    except Exception:
        return None


# ----------------------------------------------------------------------------------------------------------------------
# parameter shells (state_dict layouts of the upstream packages)
# ----------------------------------------------------------------------------------------------------------------------
class _HFAttention(nn.Module):
    def __init__(self, w):
        super().__init__()
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = nn.Linear(w, w), nn.Linear(w, w), nn.Linear(w, w), nn.Linear(w, w)


class _HFMLP(nn.Module):
    def __init__(self, w, inner):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(w, inner), nn.Linear(inner, w)


class _HFLayer(nn.Module):
    def __init__(self, a):
        super().__init__()
        self.self_attn = _HFAttention(a["width"])
        self.layer_norm1 = nn.LayerNorm(a["width"], eps=a["eps"])
        self.mlp = _HFMLP(a["width"], a["mlp"])
        self.layer_norm2 = nn.LayerNorm(a["width"], eps=a["eps"])


class _HFEncoder(nn.Module):
    def __init__(self, a):
        super().__init__()
        self.layers = nn.ModuleList([_HFLayer(a) for _ in range(a["layers"])])


class _HFEmbeddings(nn.Module):
    def __init__(self, a):
        super().__init__()
        self.token_embedding = nn.Embedding(a["vocab"], a["width"])
        self.position_embedding = nn.Embedding(a["ctx"], a["width"])
        # transformers 4.28 saved this buffer with the weights; keep the name so such checkpoints load without complaints
        self.register_buffer("position_ids", torch.arange(a["ctx"]).expand((1, -1)), persistent=False)


class _HFTextModel(nn.Module):
    def __init__(self, a):
        super().__init__()
        self.embeddings = _HFEmbeddings(a)
        self.encoder = _HFEncoder(a)
        self.final_layer_norm = nn.LayerNorm(a["width"], eps=a["eps"])


class CLIPTextModelShell(nn.Module):
    """Parameter layout of transformers.CLIPTextModel (`text_model.*`)."""

    def __init__(self, a):
        super().__init__()
        self.text_model = _HFTextModel(a)


class _OCBlock(nn.Module):
    def __init__(self, a):
        super().__init__()
        w = a["width"]
        self.ln_1 = nn.LayerNorm(w, eps=a["eps"])
        self.attn = nn.MultiheadAttention(w, a["heads"])          # in_proj_weight / in_proj_bias / out_proj.*
        self.ln_2 = nn.LayerNorm(w, eps=a["eps"])
        self.mlp = nn.Sequential(OrderedDict([("c_fc", nn.Linear(w, a["mlp"])), ("gelu", nn.GELU()), ("c_proj", nn.Linear(a["mlp"], w))]))


class _OCTransformer(nn.Module):
    def __init__(self, a):
        super().__init__()
        self.resblocks = nn.ModuleList([_OCBlock(a) for _ in range(a["layers"])])


class OpenCLIPTextShell(nn.Module):
    """Parameter layout of open_clip.CLIP after `del model.visual` (modules.py:530-536)."""

    def __init__(self, a):
        super().__init__()
        w = a["width"]
        self.transformer = _OCTransformer(a)
        self.token_embedding = nn.Embedding(a["vocab"], w)
        self.positional_embedding = nn.Parameter(torch.empty(a["ctx"], w).normal_(std=0.01))
        self.ln_final = nn.LayerNorm(w, eps=a["eps"])
        self.text_projection = nn.Parameter(torch.empty(w, a["proj"]).normal_(std=w ** -0.5))
        self.logit_scale = nn.Parameter(torch.ones([]) * np.log(1 / 0.07))
        self.register_buffer("attn_mask", torch.empty(a["ctx"], a["ctx"]).fill_(float("-inf")).triu_(1), persistent=False)


# ----------------------------------------------------------------------------------------------------------------------
# packed weights + the kernel driver
# ----------------------------------------------------------------------------------------------------------------------
def _f32(t):
    return t.detach().to(torch.float32).contiguous()


def _bf(t):
    return t.detach().to(BF16).contiguous()


class _PackedTower:
    """Kernel-layout weights of one text tower: fp32 embedding tables / LayerNorm parameters / biases, bf16 K-major matrices
    with Q|K|V stacked into one [3W, W] operand."""

    def __init__(self, arch, tok, pos, layers, lnf, proj=None):
        self.arch = arch
        self.tok, self.pos = _f32(tok), _f32(pos)
        self.layers = []
        for L in layers:
            self.layers.append(dict(
                ln1=(_f32(L["ln1_w"]), _f32(L["ln1_b"])), ln2=(_f32(L["ln2_w"]), _f32(L["ln2_b"])),
                wqkv=_bf(L["wqkv"]), bqkv=_f32(L["bqkv"]), wo=_bf(L["wo"]), bo=_f32(L["bo"]),
                w1=_bf(L["w1"]), b1=_f32(L["b1"]), w2=_bf(L["w2"]), b2=_f32(L["b2"])))
        self.lnf = (_f32(lnf[0]), _f32(lnf[1]))
        self.proj = None if proj is None else _bf(proj.detach().t())        # [P, W]: pooled @ text_projection as a Linear

    @staticmethod
    def from_hf(shell, arch):
        tm = shell.text_model
        layers = []
        for l in tm.encoder.layers:
            a = l.self_attn
            layers.append(dict(ln1_w=l.layer_norm1.weight, ln1_b=l.layer_norm1.bias, ln2_w=l.layer_norm2.weight, ln2_b=l.layer_norm2.bias,
                               wqkv=torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0),
                               bqkv=torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], 0),
                               wo=a.out_proj.weight, bo=a.out_proj.bias, w1=l.mlp.fc1.weight, b1=l.mlp.fc1.bias,
                               w2=l.mlp.fc2.weight, b2=l.mlp.fc2.bias))
        return _PackedTower(arch, tm.embeddings.token_embedding.weight, tm.embeddings.position_embedding.weight, layers,
                            (tm.final_layer_norm.weight, tm.final_layer_norm.bias))

    @staticmethod
    def from_open_clip(shell, arch):
        layers = []
        for r in shell.transformer.resblocks:
            layers.append(dict(ln1_w=r.ln_1.weight, ln1_b=r.ln_1.bias, ln2_w=r.ln_2.weight, ln2_b=r.ln_2.bias,
                               wqkv=r.attn.in_proj_weight, bqkv=r.attn.in_proj_bias, wo=r.attn.out_proj.weight, bo=r.attn.out_proj.bias,
                               w1=r.mlp.c_fc.weight, b1=r.mlp.c_fc.bias, w2=r.mlp.c_proj.weight, b2=r.mlp.c_proj.bias))
        return _PackedTower(arch, shell.token_embedding.weight, shell.positional_embedding, layers,
                            (shell.ln_final.weight, shell.ln_final.bias), shell.text_projection)


class _TowerRun:
    """One pass of a tower over tokens int32 [B, L]: `advance(n)` runs the next n transformer blocks on the fp32 residual
    stream `x` [B*L, W] (pre-LN blocks, causal self-attention; HF CLIPEncoderLayer == open_clip ResidualAttentionBlock)."""

    def __init__(self, packed, tokens, pool):
        a = packed.arch
        assert tokens.dim() == 2 and tokens.shape[1] <= a["ctx"], tokens.shape
        self.P, self.pool, self.B, self.L = packed, pool, tokens.shape[0], tokens.shape[1]
        self.done = 0
        self.tokens = tokens.to(torch.int32).contiguous()
        self.x = pool.get((self.B * self.L, a["width"]), torch.float32, tokens.device)
        ops.gather_rows_f32(packed.tok, self.tokens.view(-1), self.x, pos=packed.pos, L=self.L)

    def advance(self, n):
        a, pool, M = self.P.arch, self.pool, self.B * self.L
        W, inner, dev = a["width"], a["mlp"], self.x.device
        for lay in self.P.layers[self.done:self.done + n]:
            xb = pool.get((M, W), BF16, dev)
            ops.layernorm_f32(self.x, lay["ln1"][0], lay["ln1"][1], a["eps"], out_bf16=xb)
            qkv = pool.get((M, 3 * W), BF16, dev)
            ops.gemm(xb, lay["wqkv"], qkv, bias=lay["bqkv"])
            att = xb                                                   # the normalised copy is dead: reuse it for the heads' output
            ops.attention_small(qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:], att, self.B, a["heads"], self.L, causal=True)
            y = pool.get((M, W), torch.float32, dev)
            ops.gemm(att, lay["wo"], y, bias=lay["bo"])
            self._accumulate(y)                                        # x += out_proj(attn)
            ops.layernorm_f32(self.x, lay["ln2"][0], lay["ln2"][1], a["eps"], out_bf16=xb)
            h = pool.get((M, inner), BF16, dev)
            ops.gemm(xb, lay["w1"], h, bias=lay["b1"])
            ops.activation(h, h, a["act"])
            ops.gemm(h, lay["w2"], y, bias=lay["b2"])
            self._accumulate(y)                                        # x += mlp(ln_2(x))
            pool.put(xb, qkv, y, h)
        self.done += n
        return self.x

    def _accumulate(self, y):
        nx = self.pool.get(tuple(self.x.shape), torch.float32, self.x.device)      # out of place: the kernel's operands do not alias
        ops.axpby_f32(self.x, 1.0, y, 1.0, nx)
        self.pool.put(self.x)
        self.x = nx

    def snapshot(self):
        return self.x.clone().view(self.B, self.L, -1)

    def final_norm(self):
        out = torch.empty_like(self.x)
        ops.layernorm_f32(self.x, self.P.lnf[0], self.P.lnf[1], self.P.arch["eps"], out_f32=out)
        return out.view(self.B, self.L, -1)

    def pooled_rows(self):
        """ln_final of the row at each sequence's highest token id (the EOT token): open_clip `pool` (modules.py:584-590) and
        HF CLIPTextTransformer's legacy pooler (eos_token_id == 2 in openai/clip-vit-large-patch14's config)."""
        W = self.P.arch["width"]
        rows = (torch.arange(self.B, device=self.tokens.device) * self.L + self.tokens.argmax(dim=-1)).to(torch.int32).contiguous()
        raw = torch.empty(self.B, W, dtype=torch.float32, device=self.x.device)
        ops.gather_rows_f32(self.x, rows, raw)
        out = torch.empty_like(raw)
        ops.layernorm_f32(raw, self.P.lnf[0], self.P.lnf[1], self.P.arch["eps"], out_f32=out)
        return out

    def release(self):
        self.pool.put(self.x)


class AbstractEmbModel(nn.Module):
    """sgm/modules/encoders/modules.py:38-78 (plain attributes instead of the property boilerplate)."""

    def __init__(self):
        super().__init__()
        self.is_trainable = False
        self.ucg_rate = 0.0
        self.input_key = None
        self.legacy_ucg_val = None


class _KernelTextEmbedder(AbstractEmbModel):
    """Shared plumbing: lazily packed weights that follow load_state_dict / .to(), a scratch pool, token handling."""
    _tokenizer = None           # transformers.CLIPTokenizer, only when the vocabulary is in a layout clip_bpe does not read
    _native_bpe = None
    _bpe_cache = {}             # vocabulary path -> ClipBPE, shared by the embedders that point at the same files
    _hf_cache = {}              # vocabulary path -> transformers.CLIPTokenizer
    tokenizer_path = None

    def _init_packing(self):
        self._packed = None
        self._pool = ops.Pool()
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate())

    def invalidate(self):
        self._packed = None
        self._pool = ops.Pool()

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self.invalidate()
        return r

    def freeze(self):
        self.eval()
        for p in self.parameters():
            p.requires_grad = False

    def _bpe(self):
        """The native CLIP BPE (supir_b200/clip_bpe.py) when its vocabulary files are at `tokenizer_path`, else None."""
        if self._native_bpe is None and isinstance(self.tokenizer_path, str) and os.path.exists(self.tokenizer_path):
            from .clip_bpe import ClipBPE          # imported on first use: only tokenising strings needs the `regex` package
            if ClipBPE.available(self.tokenizer_path):
                if self.tokenizer_path not in _KernelTextEmbedder._bpe_cache:
                    _KernelTextEmbedder._bpe_cache[self.tokenizer_path] = ClipBPE.from_path(self.tokenizer_path)
                self._native_bpe = _KernelTextEmbedder._bpe_cache[self.tokenizer_path]
        return self._native_bpe

    def _hf_tokenizer(self):
        if self._tokenizer is None:
            cached = _KernelTextEmbedder._hf_cache.get(self.tokenizer_path)
            if cached is None:
                try:
                    from transformers import CLIPTokenizer
                    cached = _KernelTextEmbedder._hf_cache[self.tokenizer_path] = CLIPTokenizer.from_pretrained(self.tokenizer_path)
                except Exception as e:  # no vocabulary files offline
                    raise RuntimeError(f"no CLIP BPE vocabulary at {self.tokenizer_path!r}: pass token ids (int tensor [B, <= {self.max_length}]) "
                                       "instead of strings") from e
            self._tokenizer = cached
        return self._tokenizer

    def _tokens(self, text):
        if torch.is_tensor(text):
            return text
        return self.tokenize(list(text))

    def encode(self, text):
        return self(text)


class FrozenCLIPEmbedder(_KernelTextEmbedder):
    """sgm/modules/encoders/modules.py:445-507: transformers.CLIPTextModel (ViT-L/14 text tower); `layer` in
    last / pooled / hidden (+ layer_idx into the tuple of hidden states: 0 = embeddings, i = output of block i)."""
    LAYERS = ["last", "pooled", "hidden"]

    def __init__(self, version="openai/clip-vit-large-patch14", device="cuda", max_length=77, freeze=True, layer="last",
                 layer_idx=None, always_return_pooled=False, arch=None):
        super().__init__()
        assert layer in self.LAYERS
        path = _reference_path("SDXL_CLIP1_PATH") or version
        pretrained = None
        if arch is None and isinstance(path, str) and os.path.isdir(path):       # a local HF checkpoint directory, like the reference loads
            from transformers import CLIPTextModel
            pretrained = CLIPTextModel.from_pretrained(path)
            c = pretrained.config
            arch = dict(vocab=c.vocab_size, width=c.hidden_size, heads=c.num_attention_heads, layers=c.num_hidden_layers,
                        mlp=c.intermediate_size, ctx=c.max_position_embeddings, act=c.hidden_act, eps=c.layer_norm_eps)
        self.arch = dict(CLIP_L_ARCH, **(arch or {}))
        assert self.arch["act"] in ("quick_gelu", "gelu"), self.arch["act"]
        self.tokenizer_path = path
        self.transformer = CLIPTextModelShell(self.arch)
        if pretrained is not None:
            self.transformer.load_state_dict(pretrained.state_dict(), strict=False)
        self.device = device
        self.max_length = max_length
        self.layer, self.layer_idx, self.return_pooled = layer, layer_idx, always_return_pooled
        if layer == "hidden":
            assert layer_idx is not None
            assert 0 <= abs(layer_idx) <= self.arch["layers"]
        self._init_packing()
        if freeze:
            self.freeze()

    def tokenize(self, texts):
        """CLIPTokenizer(..., truncation=True, max_length=77, padding='max_length') (modules.py:485-494): pads with <|endoftext|>."""
        if self._bpe() is not None:
            return torch.tensor(self._bpe().tokenize_hf(texts, self.max_length), dtype=torch.long)
        enc = self._hf_tokenizer()(texts, truncation=True, max_length=self.max_length, return_length=True,
                                   return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
        return enc["input_ids"]

    @torch.no_grad()
    def forward(self, text):
        tokens = self._tokens(text).to(self.transformer.text_model.final_layer_norm.weight.device)
        if self._packed is None:
            self._packed = _PackedTower.from_hf(self.transformer, self.arch)
        n = self.arch["layers"]
        run = _TowerRun(self._packed, tokens, self._pool)
        if self.layer == "hidden":
            k = self.layer_idx % (n + 1)                      # hidden_states has n + 1 entries
            run.advance(k)
            z = run.snapshot()
            if self.return_pooled:
                run.advance(n - k)
        else:
            run.advance(n)
            z = run.final_norm() if self.layer == "last" else run.pooled_rows()[:, None, :]
        pooled = run.pooled_rows() if self.return_pooled else None
        run.release()
        return (z, pooled) if self.return_pooled else z


class FrozenOpenCLIPEmbedder2(_KernelTextEmbedder):
    """sgm/modules/encoders/modules.py:510-609: open_clip text tower; with legacy=False returns the `last` / `penultimate`
    residual stream (no ln_final on it) and, if asked, the pooled EOT feature ln_final(last)[eot] @ text_projection."""
    LAYERS = ["pooled", "last", "penultimate"]

    def __init__(self, arch="ViT-H-14", version="laion2b_s32b_b79k", device="cuda", max_length=77, freeze=True, layer="last",
                 always_return_pooled=False, legacy=True, text_cfg=None, tokenizer_path=None):
        super().__init__()
        assert layer in self.LAYERS
        if arch not in OPENCLIP_ARCHS and text_cfg is None:
            raise NotImplementedError(f"open_clip arch {arch!r}: known text towers are {sorted(OPENCLIP_ARCHS)} (or pass text_cfg=)")
        self.arch = dict(OPENCLIP_ARCHS.get(arch, OPENCLIP_ARCHS["ViT-bigG-14"]), **(text_cfg or {}))
        self.model = OpenCLIPTextShell(self.arch)
        ckpt = _reference_path("SDXL_CLIP2_CKPT_PTH") or version
        if isinstance(ckpt, str) and os.path.isfile(ckpt):                         # open_clip_pytorch_model.bin: drop the image tower
            sd = torch.load(ckpt, map_location="cpu")
            sd = sd.get("state_dict", sd)
            self.model.load_state_dict({k: v for k, v in sd.items() if not k.startswith("visual.")}, strict=False)
        self.tokenizer_path = tokenizer_path or _reference_path("SDXL_CLIP1_PATH") or "openai/clip-vit-large-patch14"   # same BPE vocabulary
        self.device = device
        self.max_length = max_length
        self.return_pooled = always_return_pooled
        self.layer = layer
        if self.layer == "last":
            self.layer_idx = 0
        elif self.layer == "penultimate":
            self.layer_idx = 1
        else:
            raise NotImplementedError()
        self.legacy = legacy
        self._init_packing()
        if freeze:
            self.freeze()

    def tokenize(self, texts):
        """open_clip.tokenize (modules.py:554): [SOT] + BPE(text) + [EOT], truncated to the context with EOT last, ZERO padded."""
        if self._bpe() is not None:
            return torch.tensor(self._bpe().tokenize_open_clip(texts, self.arch["ctx"]), dtype=torch.long)
        tk = self._hf_tokenizer()
        ctx = self.arch["ctx"]
        out = torch.zeros(len(texts), ctx, dtype=torch.long)
        for i, t in enumerate(texts):
            ids = [SOT_TOKEN] + list(tk(t, add_special_tokens=False)["input_ids"]) + [EOT_TOKEN]
            if len(ids) > ctx:
                ids = ids[:ctx]
                ids[-1] = EOT_TOKEN
            out[i, :len(ids)] = torch.tensor(ids)
        return out

    @torch.no_grad()
    def forward(self, text):
        tokens = self._tokens(text).to(self.model.ln_final.weight.device)
        if self._packed is None:
            self._packed = _PackedTower.from_open_clip(self.model, self.arch)
        n = self.arch["layers"]
        run = _TowerRun(self._packed, tokens, self._pool)
        if self.legacy:                                   # modules.py:572-575: ln_final(x[layer]) and nothing else
            assert not self.return_pooled
            run.advance(n - self.layer_idx)
            z = run.final_norm()
            run.release()
            return z
        run.advance(n - 1)
        penultimate = run.snapshot() if self.layer == "penultimate" else None
        run.advance(1)
        z = penultimate if penultimate is not None else run.snapshot()
        pooled = None
        if self.return_pooled:
            rows = run.pooled_rows()
            pooled = torch.empty(rows.shape[0], self._packed.proj.shape[0], dtype=torch.float32, device=rows.device)
            ops.linear_small_m(rows, self._packed.proj, None, pooled)
        run.release()
        return (z, pooled) if self.return_pooled else z


class ConcatTimestepEmbedderND(AbstractEmbModel):
    """embeds each dimension independently and concatenates them (modules.py:1027-1043; Timestep = sinusoidal
    timestep_embedding, openaimodel.py:69-75)."""

    def __init__(self, outdim):
        super().__init__()
        self.outdim = outdim

    @torch.no_grad()
    def forward(self, x):
        if x.ndim == 1:
            x = x[:, None]
        assert len(x.shape) == 2
        b, dims = x.shape
        t = x.reshape(-1).to(torch.float32).contiguous()
        emb = torch.empty(b * dims, self.outdim, dtype=torch.float32, device=x.device)
        ops.timestep_embedding(t, emb)
        return emb.view(b, dims * self.outdim)


# ----------------------------------------------------------------------------------------------------------------------
# GeneralConditioner (modules.py:81-243)
# ----------------------------------------------------------------------------------------------------------------------
def _cfg_get(cfg, key, default=None):
    return cfg.get(key, default) if hasattr(cfg, "get") else getattr(cfg, key, default)


class GeneralConditioner(nn.Module):
    OUTPUT_DIM2KEYS = {2: "vector", 3: "crossattn", 4: "concat", 5: "concat"}
    KEY2CATDIM = {"vector": 1, "crossattn": 2, "concat": 1, "control_vector": 1}

    def __init__(self, emb_models):
        super().__init__()
        embedders = []
        for embconfig in emb_models:
            embedder = instantiate_from_config(embconfig)
            assert isinstance(embedder, AbstractEmbModel), f"embedder model {embedder.__class__.__name__} has to inherit from AbstractEmbModel"
            embedder.is_trainable = _cfg_get(embconfig, "is_trainable", False)
            embedder.ucg_rate = _cfg_get(embconfig, "ucg_rate", 0.0)
            if embedder.is_trainable:
                raise NotImplementedError("supir_b200 is inference-only: trainable embedders are not supported")
            for param in embedder.parameters():
                param.requires_grad = False
            embedder.eval()
            if "input_key" in embconfig:
                embedder.input_key = embconfig["input_key"]
            elif "input_keys" in embconfig:
                embedder.input_keys = embconfig["input_keys"]
            else:
                raise KeyError(f"need either 'input_key' or 'input_keys' for embedder {embedder.__class__.__name__}")
            embedder.legacy_ucg_val = _cfg_get(embconfig, "legacy_ucg_value", None)
            if embedder.legacy_ucg_val is not None:
                embedder.ucg_prng = np.random.RandomState()
            embedders.append(embedder)
        self.embedders = nn.ModuleList(embedders)

    def possibly_get_ucg_val(self, embedder, batch):
        assert embedder.legacy_ucg_val is not None
        p, val = embedder.ucg_rate, embedder.legacy_ucg_val
        for i in range(len(batch[embedder.input_key])):
            if embedder.ucg_prng.choice(2, p=[1 - p, p]):
                batch[embedder.input_key][i] = val
        return batch

    def _out_key(self, embedder, emb):
        return self.OUTPUT_DIM2KEYS[emb.dim()]

    @torch.no_grad()
    def forward(self, batch, force_zero_embeddings=None):
        output = dict()
        if force_zero_embeddings is None:
            force_zero_embeddings = []
        for embedder in self.embedders:
            if getattr(embedder, "input_key", None) is not None:
                if embedder.legacy_ucg_val is not None:
                    batch = self.possibly_get_ucg_val(embedder, batch)
                emb_out = embedder(batch[embedder.input_key])
            elif hasattr(embedder, "input_keys"):
                emb_out = embedder(*[batch[k] for k in embedder.input_keys])
            assert isinstance(emb_out, (torch.Tensor, list, tuple)), f"encoder outputs must be tensors or a sequence, but got {type(emb_out)}"
            if not isinstance(emb_out, (list, tuple)):
                emb_out = [emb_out]
            for emb in emb_out:
                out_key = self._out_key(embedder, emb)
                if embedder.ucg_rate > 0.0 and embedder.legacy_ucg_val is None:
                    keep = torch.bernoulli((1.0 - embedder.ucg_rate) * torch.ones(emb.shape[0], device=emb.device))
                    emb = keep.view(-1, *([1] * (emb.dim() - 1))) * emb
                if getattr(embedder, "input_key", None) is not None and embedder.input_key in force_zero_embeddings:
                    emb = torch.zeros_like(emb)
                if out_key in output:
                    output[out_key] = torch.cat((output[out_key], emb), self.KEY2CATDIM[out_key])
                else:
                    output[out_key] = emb
        return output

    def get_unconditional_conditioning(self, batch_c, batch_uc=None, force_uc_zero_embeddings=None):
        if force_uc_zero_embeddings is None:
            force_uc_zero_embeddings = []
        ucg_rates = []
        for embedder in self.embedders:
            ucg_rates.append(embedder.ucg_rate)
            embedder.ucg_rate = 0.0
        c = self(batch_c)
        uc = self(batch_c if batch_uc is None else batch_uc, force_uc_zero_embeddings)
        for embedder, rate in zip(self.embedders, ucg_rates):
            embedder.ucg_rate = rate
        return c, uc


class GeneralConditionerWithControl(GeneralConditioner):
    """modules.py:193-243: embeddings of keys containing 'control_vector' are collected separately, and the control latent
    rides along untouched."""

    def _out_key(self, embedder, emb):
        if "control_vector" in (getattr(embedder, "input_key", None) or ""):
            return "control_vector"
        return self.OUTPUT_DIM2KEYS[emb.dim()]

    @torch.no_grad()
    def forward(self, batch, force_zero_embeddings=None):
        output = super().forward(batch, force_zero_embeddings)
        output["control"] = batch["control"]
        return output


class PreparedConditioner(nn.Module):
    """modules.py:246-290: conditioning tensors prepared offline (torch.save'd dicts) instead of text towers; rows repeated to the
    batch of the control latent."""

    def __init__(self, cond_pth, un_cond_pth=None):
        super().__init__()
        for k, v in torch.load(cond_pth).items():
            self.register_buffer(k, v)
        self.un_cond_pth = un_cond_pth
        if un_cond_pth is not None:
            for k, v in torch.load(un_cond_pth).items():
                self.register_buffer(k + "_uc", v)

    @torch.no_grad()
    def forward(self, batch, return_uc=False):
        n = batch["control"].shape[0]
        output = {}
        for k, v in self.state_dict().items():
            if k.endswith("_uc") == bool(return_uc):
                output[k[:-3] if return_uc else k] = v.detach().clone().repeat(n, *[1 for _ in range(v.ndim - 1)])
        output["control"] = batch["control"]
        return output

    def get_unconditional_conditioning(self, batch_c, batch_uc=None, force_uc_zero_embeddings=None):
        return self(batch_c), (self(batch_c, return_uc=True) if self.un_cond_pth is not None else None)
