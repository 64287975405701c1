"""Host-side logic of the FP8 linears mode (no GPU): e4m3 weight packing with per-row scales, the rest of the pack unchanged,
resident bytes, ControlWrapper.dtype invalidation, the dtype names, routing of the ops to the FP8 entry points, and argument
validation of those entry points through the C ABI."""
import ctypes

import pytest
import torch

from weights import make_state_dict, shapes_of

BF, FP8 = torch.bfloat16, torch.float8_e4m3fn

SMALL = dict(in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1, attention_resolutions=[2], channel_mult=[1, 2],
             num_head_channels=64, transformer_depth=1, context_dim=64, adm_in_channels=16, num_classes="sequential",
             use_spatial_transformer=True, use_linear_in_transformer=True, legacy=False, use_checkpoint=False)


def _small_wrapper(dtype):
    from supir_b200 import nets, wrappers
    unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=0.2, **SMALL)
    ctrl = nets.GLVControl(input_upscale=1, **SMALL)
    w = wrappers.ControlWrapper(unet, dtype=dtype)
    w.load_control_model(ctrl)
    w.load_state_dict(make_state_dict(shapes_of(w), seed=5), strict=True)
    return w


def _torch_quant(w):
    """(W * inv).to(float8_e4m3fn) * s with s = amax / 448 per row of the bf16 matrix (1 for a zero row)."""
    wf = w.detach().to(BF).float()
    amax = wf.abs().amax(1)
    f, one = torch.full_like(amax, 448.0), torch.ones_like(amax)          # IEEE divisions (tensor / tensor)
    s = torch.where(amax > 0, amax / f, one)
    inv = torch.where(amax > 0, f / torch.where(amax > 0, amax, one), one)
    return (wf * inv[:, None]).to(FP8), s


@pytest.fixture(scope="module")
def packs():
    wb = _small_wrapper(BF)
    wb.pack()
    w8 = _small_wrapper(FP8)
    w8.pack()
    return wb, w8


def _in_blocks(net):
    from supir_b200 import nets
    ids = set()
    for m in net.modules():
        if isinstance(m, nets.BasicTransformerBlock):
            ids |= {id(m.attn1), id(m.attn2), id(m.ff)}
    return ids


def test_fp8_pack_quantizes_the_transformer_linears(packs):
    from supir_b200 import nets
    _, w8 = packs
    n = 0
    for net in (w8.diffusion_model, w8.control_model):
        assert net._fp8_linears and net._packed_dtype == BF
        inside = _in_blocks(net)
        for m in net.modules():
            if id(m) not in inside:
                continue
            if isinstance(m, nets.CrossAttention):
                if m.is_self:
                    src = {"_wqkv": torch.cat([m.to_q.weight, m.to_k.weight, m.to_v.weight], 0)}
                else:
                    src = {"_wq": m.to_q.weight}
                    assert m._wkv.dtype == BF and torch.equal(m._wkv, torch.cat([m.to_k.weight, m.to_v.weight], 0).to(BF))
                src["_wo"] = m.to_out[0].weight
                assert m._c1 is None and m._bq is None          # no folded LayerNorm in FP8
            else:
                w = m.net[0].proj.weight
                idx = torch.arange(m.inner).view(-1, 16)
                perm = torch.cat([idx, idx + m.inner], 1).reshape(-1)
                src = {"_w1": w[perm], "_w2": m.net[2].weight}
            for k, wt in src.items():
                q, s = getattr(m, k)
                assert q.dtype == FP8 and s.dtype == torch.float32 and s.shape == (wt.shape[0],)
                rq, rs = _torch_quant(wt)
                assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(s, rs), (type(m).__name__, k)
                assert torch.equal(q.float() * s[:, None], rq.float() * rs[:, None])
                n += 1
    assert n >= 10


def test_geglu_interleave_keeps_rows_and_scales_together(packs):
    """Row r of the packed GEGLU matrix dequantizes to row perm[r] of the weight, with that row's own scale."""
    _, w8 = packs
    from supir_b200 import nets
    ff = next(m for m in w8.diffusion_model.modules() if isinstance(m, nets.FeedForward))
    q, s = ff._w1
    w = ff.net[0].proj.weight.detach().to(BF).float()
    inner = ff.inner
    for r in (0, 15, 16, 31, 2 * inner - 1):
        g, c = divmod(r, 32)
        src = g * 16 + c if c < 16 else inner + g * 16 + c - 16
        deq = q[r].float() * s[r]
        assert torch.allclose(deq, w[src], rtol=2 ** -3, atol=float(s[r]) * 2 ** -6)
        assert float(s[r]) == float(w[src].abs().max() / torch.tensor([448.0]))


def _packed_tensors(net):
    out = {}
    for name, m in net.named_modules():
        for k, v in vars(m).items():
            if k.startswith("_") and k != "_ln" and (torch.is_tensor(v) or (isinstance(v, tuple) and v and all(torch.is_tensor(t) or t is None for t in v))):
                out[(name, k)] = v
    return out


def test_every_other_packed_tensor_is_the_bf16_pack(packs):
    wb, w8 = packs
    for nb, n8 in ((wb.diffusion_model, w8.diffusion_model), (wb.control_model, w8.control_model)):
        inside = {name for name, m in n8.named_modules() if id(m) in _in_blocks(n8)}
        tb, t8 = _packed_tensors(nb), _packed_tensors(n8)
        checked = 0
        for key, v in tb.items():
            if key[0] in inside and key[1] in ("_wqkv", "_wq", "_wo", "_w1", "_w2", "_c1", "_bq", "_ln"):
                continue
            v8 = t8[key]
            for a, b in zip(v if isinstance(v, tuple) else (v,), v8 if isinstance(v8, tuple) else (v8,)):
                assert (a is None and b is None) or (a.dtype == b.dtype and torch.equal(a, b)), key
            checked += 1
        assert checked > 50


def _bytes(net):
    seen, n = set(), 0
    for v in _packed_tensors(net).values():
        for t in (v if isinstance(v, tuple) else (v,)):
            if torch.is_tensor(t) and id(t) not in seen:
                seen.add(id(t))
                n += t.numel() * t.element_size()
    return n


def test_packed_bytes_shrink_by_the_quantized_matrices(packs):
    """bf16 [N, K] (2 N K bytes) + fp32 colsum of the folded LayerNorm + fp32 folded bias -> e4m3 [N, K] (N K) + fp32 [N]."""
    from supir_b200 import nets
    wb, w8 = packs
    for nb, n8 in ((wb.diffusion_model, w8.diffusion_model), (wb.control_model, w8.control_model)):
        want = 0
        for m in nb.modules():
            if not isinstance(m, nets.BasicTransformerBlock):
                continue
            C = m.attn1.inner
            dim = m.norm1.normalized_shape[0]
            mats = [(3 * C, dim), (dim, C), (C, dim), (dim, C), (2 * m.ff.inner, dim), (dim, m.ff.inner)]
            want += sum(N * K - 4 * N for N, K in mats)                  # 2NK -> NK bytes, + 4N of scales
            if m.fuse_ln:                                                 # the bf16 pack's folded-LayerNorm colsum + bias
                want += 2 * (4 * 3 * C) + 2 * (4 * C)
        assert _bytes(nb) - _bytes(n8) == want


def test_dtype_switch_bf16_fp8_bf16_invalidates_only_on_a_change():
    from supir_b200 import nets, wrappers
    w = wrappers.ControlWrapper(nets.LightGLVUNet.__new__(nets.LightGLVUNet), dtype=BF)

    def arm():
        w._packed, w._plans = True, {"k": object()}

    arm()
    w.dtype = FP8
    assert not w._packed and not w._plans and w.compute_dtype == BF and w.dtype == FP8
    arm()
    w.dtype = FP8
    assert w._packed and w._plans
    w.dtype = BF
    assert not w._packed and not w._plans
    arm()
    w.dtype = torch.float32                  # fp32 computes bf16: same packs
    assert w._packed and w._plans
    w.dtype = FP8
    assert not w._packed


def test_dtype_names():
    from supir_b200 import util
    assert util.convert_dtype("fp8") is FP8
    assert util.convert_dtype("fp16") is torch.float16 and util.convert_dtype("bf16") is BF and util.convert_dtype("fp32") is torch.float32
    with pytest.raises(NotImplementedError):
        util.convert_dtype("e5m2")


def test_supir_model_accepts_fp8(monkeypatch):
    """diffusion_dtype='fp8' sets the wrapper's dtype; the other values are unchanged (the constructor's config plumbing is
    replaced by stubs: only the dtype mapping is under test)."""
    from supir_b200 import model as smodel

    class Wrapper(torch.nn.Module):
        def __init__(self, net):
            super().__init__()
            self.dtype = None

        def load_control_model(self, m):
            pass

    class FirstStage(torch.nn.Module):
        encoder = torch.nn.Identity()

    def inst(cfg):
        return FirstStage() if cfg == "fs" else object()

    monkeypatch.setattr(smodel, "get_obj_from_str", lambda s: Wrapper)
    monkeypatch.setattr(smodel, "instantiate_from_config", inst)
    want = {"fp8": FP8, "bf16": BF, "fp16": torch.float16, "fp32": torch.float32}
    for name, dt in want.items():
        m = smodel.SUPIRModel("c", "n", "d", "fs", ae_dtype="bf16", diffusion_dtype=name)
        assert m.model.dtype is dt and m.ae_dtype is BF
    with pytest.raises(AssertionError):
        smodel.SUPIRModel("c", "n", "d", "fs", diffusion_dtype="fp4")


def _record(monkeypatch):
    from supir_b200 import _native, ops
    calls = []
    monkeypatch.setattr(_native, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(ops, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    return ops, calls


def test_ops_route_fp8_calls_to_the_fp8_entry_points(monkeypatch):
    ops, calls = _record(monkeypatch)
    q = lambda *s: torch.zeros(*s, dtype=FP8)             # noqa: E731
    f = lambda *s: torch.zeros(*s)                        # noqa: E731
    b = lambda *s: torch.zeros(*s, dtype=BF)              # noqa: E731
    ops.gemm_fp8(q(16, 32), f(16), q(64, 32), f(64), b(16, 32), bias=f(64), act=2)
    ops.gemm_fp8(q(16, 32), f(16), q(8, 32), f(8), b(16, 8), residual=b(16, 8))
    ops.quantize_rows(b(16, 32), q(16, 32), f(16))
    ops.layernorm_quant(b(16, 32), f(32), f(32), q(16, 32), f(16))
    assert calls == ["supir_gemm_fp8", "supir_gemm_fp8", "supir_quantize_rows", "supir_layernorm_quant"]


def test_ops_reject_bad_fp8_calls_before_any_call(monkeypatch):
    ops, calls = _record(monkeypatch)
    q, f = torch.zeros(16, 32, dtype=FP8), torch.zeros(16)
    w, ws = torch.zeros(8, 32, dtype=FP8), torch.zeros(8)
    out = torch.zeros(16, 8, dtype=BF)
    with pytest.raises(ValueError):
        ops.gemm_fp8(q, f, w, ws, out, ln=(torch.zeros(16, 2), torch.zeros(8)))
    with pytest.raises(TypeError):
        ops.gemm_fp8(q.to(torch.float16), f, w, ws, out)                          # fp16 operand
    with pytest.raises(TypeError):
        ops.gemm_fp8(q, f, w.to(BF), ws, out)                                     # mixed operand dtypes
    with pytest.raises(TypeError):
        ops.gemm_fp8(q, f, w, ws, out.to(torch.float16))                          # fp16 output
    with pytest.raises(TypeError):
        ops.gemm_fp8(q, f, w, ws, out, residual=torch.zeros(16, 8, dtype=torch.float16))
    with pytest.raises(TypeError):
        ops.quantize_rows(torch.zeros(16, 32, dtype=torch.float16), q, f)
    with pytest.raises(TypeError):
        ops.layernorm_quant(torch.zeros(16, 32, dtype=BF), torch.zeros(32), torch.zeros(32), q.to(BF), f)
    assert calls == []


def test_fp8_entry_points_reject_bad_arguments_before_any_launch():
    """Negative return code + message, before the device is touched (this runs without a GPU)."""
    from supir_b200 import _native
    lib = _native.load()
    P = lambda a: ctypes.c_void_p(a)                      # noqa: E731
    ok, ok_s = P(1 << 20), P(1 << 21)

    def gemm(A=ok, lda=64, sa=ok_s, W=ok, ldw=64, sw=ok_s, out=ok, ldc=64, M=16, N=64, K=64, ep=None):
        rc = lib.supir_gemm_fp8(A, lda, sa, W, ldw, sw, out, ldc, M, N, K, ep, None)
        return rc, lib.supir_last_error()

    rc, msg = gemm(A=P((1 << 20) + 8))
    assert rc < 0 and b"supir_gemm_fp8" in msg and b"aligned" in msg
    rc, msg = gemm(sa=P((1 << 21) + 2))
    assert rc < 0 and b"aligned" in msg
    rc, msg = gemm(K=40, lda=48, ldw=48)
    assert rc < 0 and b"multiples of 16" in msg
    rc, msg = gemm(lda=72)
    assert rc < 0 and b"multiples of 16" in msg
    rc, msg = gemm(M=0)
    assert rc < 0 and b"bad shape" in msg
    rc, msg = gemm(sw=None)
    assert rc < 0 and b"null" in msg
    for field, val in (("ln_stats", 1 << 22), ("out_f32", 1), ("rowvec", 1 << 22)):
        ep = _native.Epilogue()
        setattr(ep, field, val)
        rc, msg = gemm(ep=ctypes.byref(ep))
        assert rc < 0 and b"FP8 epilogue" in msg, field
    ep = _native.Epilogue()
    ep.act = 2
    rc, msg = gemm(N=40, ep=ctypes.byref(ep))                 # GEGLU needs N % 32 == 0, as in bf16
    assert rc < 0 and b"GEGLU" in msg

    assert lib.supir_quantize_rows(ok, 64, ok, 64, ok_s, 16, 60, None) < 0          # cols % 8
    assert b"supir_quantize_rows" in lib.supir_last_error()
    assert lib.supir_quantize_rows(P((1 << 20) + 8), 64, ok, 64, ok_s, 16, 64, None) < 0
    assert b"misaligned" in lib.supir_last_error()
    assert lib.supir_layernorm_quant(ok, 64, ok, 64, ok_s, 16, 40, ok, ok, 1e-5, None) < 0     # C % 16
    assert b"supir_layernorm_quant" in lib.supir_last_error()
    assert lib.supir_layernorm_quant(ok, 64, ok, 72, ok_s, 16, 64, ok, ok, 1e-5, None) < 0     # ldq % 16
    assert lib.supir_layernorm_quant(ok, 64, P((1 << 20) + 4), 64, ok_s, 16, 64, ok, ok, 1e-5, None) < 0
    assert b"misaligned" in lib.supir_last_error()
