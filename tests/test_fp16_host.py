"""Host-side logic of the fp16 compute mode (no GPU): fp16 weight packing, ControlWrapper.dtype invalidation, routing of the
ops to the `_f16` entry points, and argument validation of those entry points."""
import ctypes

import pytest
import torch

from weights import make_state_dict, shapes_of

H16, BF = torch.float16, torch.bfloat16

SMALL = dict(in_channels=4, model_channels=32, out_channels=4, num_res_blocks=1, attention_resolutions=[2], channel_mult=[1, 2],
             num_head_channels=64, transformer_depth=1, context_dim=64, adm_in_channels=16, num_classes="sequential",
             use_spatial_transformer=True, use_linear_in_transformer=True, legacy=False, use_checkpoint=False)


def _small_wrapper(dtype):
    from supir_b200 import nets, wrappers
    unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=0.2, **dict(SMALL, model_channels=64))
    ctrl = nets.GLVControl(input_upscale=1, **dict(SMALL, model_channels=64))
    w = wrappers.ControlWrapper(unet, dtype=dtype)
    w.load_control_model(ctrl)
    w.load_state_dict(make_state_dict(shapes_of(w), seed=5), strict=True)
    return w


@pytest.fixture(scope="module")
def packed16():
    try:
        w = _small_wrapper(H16)
    except NotImplementedError as e:        # pragma: no cover - configuration outside what the networks accept
        pytest.skip(str(e))
    w.pack()
    return w


def test_fp16_pack_rounds_the_bf16_expressions_to_fp16(packed16):
    """Every packed matrix is fp16 and equals the fp16 rounding of the expression the bf16 pack uses."""
    from supir_b200 import nets
    w = packed16
    mats = 0
    for net in (w.diffusion_model, w.control_model):
        assert net._packed_dtype == H16 and net._emb_w.dtype == H16 and net._ctx_w.dtype == H16
        for m in net.modules():
            for k, v in vars(m).items():
                if k.startswith("_w") and torch.is_tensor(v) and v.dim() == 2 and k not in ("_w", "_wout"):
                    assert v.dtype == H16, (type(m).__name__, k, v.dtype)
                    mats += 1
            if isinstance(m, nets.ResBlock):
                assert torch.equal(m._w1, m.in_layers[2].weight.detach().permute(0, 2, 3, 1).reshape(m.out_channels, -1).half())
                assert torch.equal(m._b1, m.in_layers[2].bias.detach().half().float())
            if isinstance(m, nets.CrossAttention) and m.is_self and m._ln is not None:
                wqkv = torch.cat([m.to_q.weight, m.to_k.weight, m.to_v.weight], 0).detach()
                wg = (wqkv.half().float() * m._ln[0].detach().float()[None, :]).half()     # fp32 product rounded once
                assert torch.equal(m._wqkv, wg)
                assert torch.equal(m._c1, wg.float().sum(1))
            if isinstance(m, nets.Upsample) and hasattr(m, "_wfold"):
                wf = m.conv.weight.detach().half().float()
                tap00 = wf[:, :, 1, 1] + wf[:, :, 1, 2] + wf[:, :, 2, 1] + wf[:, :, 2, 2]     # parity (0, 0), tap (1, 1)
                got = m._wfold[0].view(m.out_channels, 4, -1)[:, 3]
                assert m._wfold[0].dtype == H16 and torch.equal(got, tap00.half())
            if isinstance(m, nets.ConvIn):
                assert m._wp.dtype == H16 and torch.equal(m._w, m.weight.detach().half().float())
    assert mats > 20
    u = w.diffusion_model
    assert u._out_packed[0].dtype == H16 and torch.equal(u._wout, u.out[2].weight.detach().half().float().permute(0, 2, 3, 1))
    assert all(t.dtype == H16 for t in (u._te[0], u._te[2], u._le[0], u._le[2]))


def test_bf16_pack_unchanged_by_the_dtype_parameter():
    from supir_b200 import nets, ops
    g = torch.Generator().manual_seed(1)
    wt = torch.randn(16, 8, 3, 3, generator=g)
    assert torch.equal(nets.pack_conv3x3(wt), nets.pack_conv3x3(wt, BF)) and nets.pack_conv3x3(wt).dtype == BF
    assert nets.pack_conv3x3(wt, H16).dtype == H16
    gamma, beta = torch.rand(8, generator=g) + 0.5, torch.randn(8, generator=g)
    a, b = ops.fold_layernorm(wt[:, :, 0, 0], None, gamma, beta), ops.fold_layernorm(wt[:, :, 0, 0], None, gamma, beta, dtype=BF)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert ops.pack_small_cin_weight(wt[:, :4], H16).dtype == H16 and ops.pack_small_cout_weight(wt[:4], None, H16)[0].dtype == H16
    assert all(t.dtype == H16 for t in ops.fold_upsample_weights(wt, H16))


def test_dtype_switch_invalidates_packs_and_plans_only_on_a_change():
    from supir_b200 import nets, wrappers
    w = wrappers.ControlWrapper(nets.LightGLVUNet.__new__(nets.LightGLVUNet), dtype=BF)
    assert w.dtype == BF and w.compute_dtype == BF

    def arm():
        w._packed, w._plans = True, {"k": object()}

    arm()
    w.dtype = BF
    assert w._packed and w._plans
    w.dtype = H16
    assert not w._packed and not w._plans and w.compute_dtype == H16
    arm()
    w.dtype = H16
    assert w._packed and w._plans
    w.dtype = BF
    assert not w._packed and not w._plans
    arm()
    w.dtype = torch.float32                 # fp32 computes bf16: same packs
    assert w._packed and w._plans and w.compute_dtype == BF


def _record(monkeypatch):
    from supir_b200 import _native, ops
    calls = []
    monkeypatch.setattr(_native, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(ops, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    return ops, calls


def _cases(dt):
    from supir_b200 import ops
    z = lambda *s: torch.zeros(*s, dtype=dt)              # noqa: E731
    f = lambda *s: torch.zeros(*s)                        # noqa: E731
    return [
        ("supir_gemm_bf16", lambda: ops.gemm(z(16, 32), z(8, 32), z(16, 8))),
        ("supir_gemm_bf16", lambda: ops.gemm(z(16, 32), z(8, 32), f(16, 8))),
        ("supir_conv3x3_bf16", lambda: ops.conv3x3(z(2 * 4 * 4, 8), 2, 4, 4, z(16, 72), z(32, 16))),
        ("supir_conv_geom_bf16", lambda: ops.conv3x3_stride2(z(2 * 4 * 4, 8), 2, 4, 4, z(16, 72), z(2 * 2 * 2, 16), 1)),
        ("supir_attention_bf16", lambda: ops.attention(z(10, 64), z(6, 64), z(6, 64), z(10, 64), 2, 1, 5, 3)),
        ("supir_groupnorm_stats", lambda: ops.groupnorm_stats(z(8, 64), 2, 4, torch.zeros(64, dtype=torch.float64))),
        ("supir_groupnorm_apply", lambda: ops.groupnorm_apply(z(8, 64), 2, 4, z(8, 64), f(64), f(64), 1e-5, True, sums=f(8))),
        ("supir_zerosft_apply", lambda: ops.zerosft_apply(z(8, 64), z(8, 32), 32, z(8, 128), z(8, 64), 2, 4, f(8), f(64), f(64), 1e-5, f(1))),
        ("supir_layernorm_bf16", lambda: ops.layernorm(z(8, 64), z(8, 64), f(64), f(64))),
        ("supir_layernorm_stats", lambda: ops.layernorm_stats(z(8, 64), f(8, 2))),
        ("supir_conv3x3_small_cin", lambda: ops.conv3x3_small_cin(f(2, 4, 4, 4), f(16, 4, 3, 3), f(16), z(32, 16))),
        ("supir_conv3x3_small_cout", lambda: ops.conv3x3_small_cout(z(32, 16), 2, 4, 4, f(4, 3, 3, 16), f(4), f(2, 4, 4, 4))),
        ("supir_axpy_bf16", lambda: ops.axpy(z(8, 16), z(8, 16), z(8, 16), f(1))),
        ("supir_f32_to_bf16", lambda: (ops.f32_to_f16 if dt == H16 else ops.f32_to_bf16)(f(64), z(64))),
        ("supir_linear_small_m", lambda: ops.linear_small_m(f(2, 32), z(8, 32), f(8), f(2, 8))),
    ]


def test_ops_route_each_dtype_to_its_entry_point(monkeypatch):
    from supir_b200 import _native
    ops, calls = _record(monkeypatch)
    for dt in (BF, H16):
        for name, fn in _cases(dt):
            calls.clear()
            fn()
            want = name if dt == BF else _native.F16_TWINS[name]
            assert calls == [want], (name, dt, calls)


def test_ops_reject_mixed_16bit_operands_before_any_call(monkeypatch):
    ops, calls = _record(monkeypatch)
    b, h = torch.zeros(16, 32, dtype=BF), torch.zeros(8, 32, dtype=H16)
    with pytest.raises(TypeError):
        ops.gemm(b, h, torch.zeros(16, 8, dtype=BF))
    with pytest.raises(TypeError):
        ops.gemm(b, b[:8], torch.zeros(16, 8, dtype=BF), residual=torch.zeros(16, 8, dtype=H16))
    with pytest.raises(TypeError):
        ops.attention(b[:, :64 // 2 * 2], b, b, torch.zeros(16, 32, dtype=H16), 1, 1, 16, 16)
    with pytest.raises(TypeError):
        ops.layernorm(torch.zeros(8, 64, dtype=BF), torch.zeros(8, 64, dtype=H16), torch.zeros(64), torch.zeros(64))
    assert calls == []


def test_f16_entry_points_reject_bad_arguments_before_any_launch():
    """Negative return code + message for a bad shape, before the device is touched."""
    from supir_b200 import _native
    lib = _native.load()
    p = ctypes.c_void_p(16)
    assert lib.supir_gemm_f16(p, 8, p, 8, p, 8, 0, 8, 8, None, None) < 0
    assert b"supir_gemm_f16" in lib.supir_last_error() and b"bad shape" in lib.supir_last_error()
    assert lib.supir_attention_f16(p, 64, p, 64, p, 64, p, 64, 1, 1, 8, 8, 128, 0.125, None) < 0
    assert b"supir_attention_f16" in lib.supir_last_error()
    assert lib.supir_layernorm_f16(p, 12, p, 12, 4, 12, p, p, 1e-5, None) < 0
    assert b"supir_layernorm_f16" in lib.supir_last_error()
    assert lib.supir_conv3x3_small_cout_f16(p, 16, p, p, p, 1, 1, 1, 1, 4, 4, 16, 5, 0, 0, 4, 4, None) < 0
    assert b"supir_conv3x3_small_cout_f16" in lib.supir_last_error()
    assert lib.supir_linear_small_m_f16(p, 8, p, p, p, 8, 17, 8, 8, 0, 0, None, 0, None) < 0
    assert b"supir_linear_small_m_f16" in lib.supir_last_error()
    for name in _native.F16_TWINS.values():
        assert hasattr(lib, name)
