"""SDXL VAE (encoder / decoder / AutoencoderKL wrapper) and the tiled VAE for the H100 backend.

Reference: sgm/modules/diffusionmodules/model.py:49-148,158-262,482-743 (Encoder/Decoder/ResnetBlock/AttnBlock),
sgm/models/autoencoder.py:282-321 (AutoencoderKL[InferenceWrapper]), sgm/modules/distributions/distributions.py:24-41,
SUPIR/utils/tilevae.py:374-970 (task queue, cross-tile GroupNorm, split/crop bookkeeping, VAEHook).

Parameters carry the reference's names; compute is the C-ABI kernels. The network is flattened once into a step list
(the reference's "task queue"). Untiled: the steps run on one NHWC bf16 tensor. Tiled: every padded tile advances through
the same steps with ALL tiles resident in HBM (the reference parks them on the CPU between GroupNorm layers); at each
GroupNorm the per-tile (mean, biased var) are merged with the reference's pixel-weighted rule (tilevae.py:629-648) by a
kernel and applied to every tile. Tile bboxes / crops are integer host code, bit-identical to the reference.
Opt-in (`VAEHook.shard = True`) the tiles are sharded over torch.distributed ranks: per GroupNorm layer one all-gather of
per-tile statistics (a few KB), and one all-gather of the cropped output tiles at the end.
"""
import math

import torch
import torch.nn as nn

from . import ops
from .nets import Act, _bf, _bias_bf16_values, _f32, pack_conv3x3
from .ops import BF16


# cached scratch above this is handed back to torch's caching allocator between resolutions and after a pass. The three VAE
# networks of a restore (denoise encoder, decoder, encoder) each own a pool, and on an 80 GB H100 they cannot each keep the
# ~26 GB a 4096^2 pass uses: above 8 GB the buffers go back to torch's allocator, where the next network's pass reuses them.
POOL_TRIM_BYTES = 8 << 30


def Normalize(in_channels, num_groups=32):
    return nn.GroupNorm(num_groups=num_groups, num_channels=in_channels, eps=1e-6, affine=True)


class _Up(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, 1, 1)


class _Down(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, 2, 0)


class ResnetBlock(nn.Module):
    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout=0.0, temb_channels=0):
        super().__init__()
        if conv_shortcut or temb_channels:
            raise NotImplementedError("ResnetBlock option outside the SDXL VAE")
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = Normalize(in_channels)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, 1, 1)
        self.norm2 = Normalize(out_channels)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        if in_channels != out_channels:
            self.nin_shortcut = nn.Conv2d(in_channels, out_channels, 1, 1, 0)


class AttnBlock(nn.Module):
    """Single-head attention over all pixels of the (tile's) lowest resolution, head_dim = channels (512)."""

    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = nn.Conv2d(in_channels, in_channels, 1)
        self.k = nn.Conv2d(in_channels, in_channels, 1)
        self.v = nn.Conv2d(in_channels, in_channels, 1)
        self.proj_out = nn.Conv2d(in_channels, in_channels, 1)


MemoryEfficientAttnBlock = AttnBlock  # identical parameters ("vanilla-xformers" in the SUPIR yaml)


class _Level(nn.Module):
    pass


class _VAENet(nn.Module):
    is_decoder = False

    def __init__(self):
        super().__init__()
        self._packed, self._pool = False, None
        # kernel-layout weights are derived data: a later load_state_dict (gradio_demo*.py switch the Q / F checkpoints at
        # run time) or .to() must re-pack them, like ControlWrapper does for the diffusion networks
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate())

    def invalidate(self):
        self._packed, self._pool = False, None

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self.invalidate()
        return r

    # ---- packing: per-step kernel-layout weights ----
    def pack(self):
        self._steps = []
        add = self._steps.append

        def conv3(m):
            return ("conv", pack_conv3x3(m.weight), _bias_bf16_values(m.bias), m.out_channels)

        def norm(m):
            return ("norm", _f32(m.weight), _f32(m.bias), m.num_channels)

        def resblock(b):
            if hasattr(b, "nin_shortcut"):
                s = b.nin_shortcut
                add(("store_res", _bf(s.weight.reshape(s.out_channels, s.in_channels)), _bias_bf16_values(s.bias), s.out_channels))
            else:
                add(("store_res", None, None, b.out_channels))
            add(norm(b.norm1)), add(("silu",)), add(conv3(b.conv1))
            add(norm(b.norm2)), add(("silu",)), add(conv3(b.conv2))
            add(("add_res",))

        def attn(a):
            C = a.in_channels
            add(("store_res", None, None, C))
            add(norm(a.norm))
            wqkv = _bf(torch.cat([a.q.weight.reshape(C, C), a.k.weight.reshape(C, C), a.v.weight.reshape(C, C)], 0))
            bqkv = torch.cat([_bias_bf16_values(a.q.bias), _bias_bf16_values(a.k.bias), _bias_bf16_values(a.v.bias)], 0).contiguous()
            add(("attn", wqkv, bqkv, _bf(a.proj_out.weight.reshape(C, C)), _bias_bf16_values(a.proj_out.bias), C))
            add(("add_res",))

        ci = self.conv_in
        self._conv_in = (ci.weight.detach().to(BF16).to(torch.float32).contiguous(), _bias_bf16_values(ci.bias), ci.out_channels)
        self._conv_in_packed = ops.pack_small_cin_weight(ci.weight)
        mid = lambda: (resblock(self.mid.block_1), attn(self.mid.attn_1), resblock(self.mid.block_2))  # noqa: E731
        if self.is_decoder:
            mid()
            for lvl in reversed(range(self.num_resolutions)):
                for blk in self.up[lvl].block:
                    resblock(blk)
                if lvl != 0:
                    c = self.up[lvl].upsample.conv
                    add(("upsample", ops.fold_upsample_weights(c.weight) if ops.CONV_GEOM else pack_conv3x3(c.weight),
                         _bias_bf16_values(c.bias), c.out_channels))
        else:
            for lvl in range(self.num_resolutions):
                for blk in self.down[lvl].block:
                    resblock(blk)
                if lvl != self.num_resolutions - 1:
                    c = self.down[lvl].downsample.conv
                    add(("downsample", pack_conv3x3(c.weight), _bias_bf16_values(c.bias), c.out_channels))
            mid()
        add(norm(self.norm_out)), add(("silu",))
        co = self.conv_out
        self._conv_out = (co.weight.detach().to(BF16).to(torch.float32).permute(0, 2, 3, 1).contiguous(),
                          _bias_bf16_values(co.bias), co.out_channels)
        self._conv_out_packed = ops.pack_small_cout_weight(co.weight, co.bias)
        self._packed = True
        return self

    # ---- step execution on one tile (in place on the tile record) ----
    def _apply_step(self, pool, step, tile, add_res=False):
        """`add_res`: the step is followed by the block's skip connection, folded into this step's GEMM epilogue."""
        kind = step[0]
        a: Act = tile["h"]
        if kind == "conv":
            out = pool.get((a.rows, step[3]))
            r = tile["res"].pop() if add_res else None
            ops.conv3x3(a.t, a.B, a.H, a.W, step[1], out, bias=step[2], residual=r)
            pool.put(a.t, r)
            tile["h"] = Act(out, a.B, a.H, a.W)
        elif kind == "store_res":
            if step[1] is None:
                r = a.t                     # identity skip: hold the tensor itself; the norm that follows must not recycle it
                tile["keep"] = r
            else:
                r = pool.get((a.rows, step[3]))
                ops.gemm(a.t, step[1], r, bias=step[2])
            tile["res"].append(r)
        elif kind == "add_res":
            r = tile["res"].pop()
            one = tile["one"]
            out = pool.get((a.rows, a.C))
            ops.axpy(r, a.t, out, one)          # res + h * 1
            pool.put(a.t, r)
            tile["h"] = Act(out, a.B, a.H, a.W)
        elif kind == "upsample":
            out = pool.get((4 * a.rows, step[3]))
            if ops.CONV_GEOM:
                ops.upsample2x_conv3x3(a.t, a.B, a.H, a.W, step[1], out, bias=step[2])
            else:
                up = pool.get((4 * a.rows, a.C))
                ops.upsample2x(a.t, a.B, a.H, a.W, up)
                ops.conv3x3(up, a.B, 2 * a.H, 2 * a.W, step[1], out, bias=step[2])
                pool.put(up)
            pool.put(a.t)
            tile["h"] = Act(out, a.B, 2 * a.H, 2 * a.W)
        elif kind == "downsample":       # pad (0,1,0,1), stride 2, no conv padding (model.py:81-85)
            Ho, Wo = (a.H + 1 - 3) // 2 + 1, (a.W + 1 - 3) // 2 + 1
            out = pool.get((a.B * Ho * Wo, step[3]))
            if ops.CONV_GEOM:
                ops.conv3x3_stride2(a.t, a.B, a.H, a.W, step[1], out, 0, bias=step[2])
            else:
                cols = pool.get((a.B * Ho * Wo, 9 * a.C))
                ops.im2col_s2(a.t, a.B, a.H, a.W, cols, Ho, Wo, 0)
                ops.gemm(cols, step[1], out, bias=step[2])
                pool.put(cols)
            pool.put(a.t)
            tile["h"] = Act(out, a.B, Ho, Wo)
        elif kind == "attn":
            self._attn(pool, step, tile, add_res)
        else:
            raise ValueError(kind)

    def _attn(self, pool, step, tile, add_res=False):
        """softmax(q k^T c^-0.5) v with one 512-wide head (model.py:187-189, tilevae.py:292-336): fused Q|K|V projection, the
        flash-style head_dim-512 kernel (no score matrix in HBM), output projection with the block's skip in its epilogue."""
        _, wqkv, bqkv, wo, bo, C = step
        a: Act = tile["h"]
        L = a.HW
        r = tile["res"].pop() if add_res else None
        qkv = pool.get((a.rows, 3 * C))
        ops.gemm(a.t, wqkv, qkv, bias=bqkv)
        o = pool.get((a.rows, C))
        ops.attention_1head(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], o, a.B, L, float(int(C) ** (-0.5)))
        out = pool.get((a.rows, C))
        ops.gemm(o, wo, out, bias=bo, residual=r)
        pool.put(qkv, o, a.t, r)
        tile["h"] = Act(out, a.B, a.H, a.W)

    def _norm_apply(self, pool, step, tile, sums=None, mean=None, var=None):
        a: Act = tile["h"]
        out = pool.get((a.rows, a.C))
        ops.groupnorm_apply(a.t, a.B, a.HW, out, step[1], step[2], 1e-6, tile.get("fuse_silu", False), sums=sums, mean=mean, var=var)
        if tile.get("keep") is a.t:
            tile["keep"] = None             # held as a skip connection (see store_res)
        else:
            pool.put(a.t)
        tile["h"] = Act(out, a.B, a.H, a.W)

    # ---- drivers ----
    def _scratch(self):
        """Scratch pool that lives with the network: a second pass reuses the first one's buffers instead of going back to
        the allocator (a cold tiled pass spent more time in cudaMalloc than in kernels). `release_scratch()` drops it."""
        pool = getattr(self, "_pool", None)
        if pool is None:
            pool = self._pool = ops.Pool()
        return pool

    def release_scratch(self):
        self._pool = None

    def _check(self, x):
        if not x.is_cuda:
            raise RuntimeError("supir_b200 VAE needs CUDA tensors: the backend has no CPU path")
        if not getattr(self, "_packed", False) or self._conv_in[0].device != x.device:
            self.pack()
            self._pool = None

    def _start_tile(self, pool, x_view):
        """conv_in on an fp32 NCHW view (a tile of the input, zero padded at its own border like the reference's per-tile conv)."""
        B, _, H, W = x_view.shape
        w, b, cout = self._conv_in
        out = pool.get((B * H * W, cout))
        ops.conv3x3_small_cin(x_view, w, b, out, w_packed=self._conv_in_packed, pool=pool)
        return {"h": Act(out, B, H, W), "res": [], "one": self._one}

    def _finish_tile(self, pool, tile, out_view, crop=None):
        a: Act = tile["h"]
        w, b, cout = self._conv_out
        ops.conv3x3_small_cout(a.t, a.B, a.H, a.W, w, b, out_view, crop=crop, packed=self._conv_out_packed, pool=pool)
        pool.put(a.t)

    def _fused_steps(self):
        """(step, fused) pairs: a 'silu' right after a 'norm' is folded into the norm-apply kernel, and an 'add_res' right
        after a conv / attention into that step's GEMM epilogue (`fused` is True for the absorbing step)."""
        steps, out, i = self._steps, [], 0
        while i < len(steps):
            nxt = steps[i + 1][0] if i + 1 < len(steps) else None
            if (steps[i][0] == "norm" and nxt == "silu") or (steps[i][0] in ("conv", "attn") and nxt == "add_res"):
                out.append((steps[i], True))
                i += 2
            else:
                out.append((steps[i], False))
                i += 1
        return out

    @torch.no_grad()
    def original_forward(self, x):
        """Untiled Encoder.forward / Decoder.forward. x fp32 NCHW -> fp32 NCHW (values rounded to bf16 like autocast)."""
        self._check(x)
        x = x.float()
        pool = self._scratch()
        self._one = torch.ones(1, dtype=torch.float32, device=x.device)
        tile = self._start_tile(pool, x)
        for step, fuse in self._fused_steps():
            if step[0] == "norm":
                a = tile["h"]
                ws = pool.get((ops.groupnorm_ws_size(a.B, a.HW, a.C),), torch.float64)
                ops.groupnorm_stats(a.t, a.B, a.HW, ws)
                tile["fuse_silu"] = fuse
                self._norm_apply(pool, step, tile, sums=ws)
                pool.put(ws)
            else:
                self._apply_step(pool, step, tile, fuse)
        a = tile["h"]
        out = torch.empty((a.B, self._conv_out[2], a.H, a.W), dtype=torch.float32, device=x.device)
        self._finish_tile(pool, tile, out)
        return out

    forward = original_forward

    @torch.no_grad()
    def estimate_group_norm(self, z, tile_size, color_fix=False):
        """Fast mode of the tiled VAE (tilevae.py:855-876 + estimate_group_norm :776-817): the whole input, nearest-exact
        downsampled to about one tile with its per-channel mean / std restored and clamped to the input's range, runs through
        the layers as ONE tile; the (mean, biased var) every GroupNorm sees there replace the cross-tile merge. Returns one
        (mean, var) pair per norm layer — None for the layers after the first downsample when `color_fix` (the reference then
        estimates only the full-resolution layers and keeps the exact merge for the rest)."""
        N, C, H, W = z.shape
        scale = tile_size / max(H, W)
        iy = nearest_exact_indices(H, scale).to(z.device)
        ix = nearest_exact_indices(W, scale).to(z.device)
        small = z.index_select(2, iy).index_select(3, ix).contiguous()          # F.interpolate(mode='nearest-exact'): a gather
        std_old, mean_old = ops.channel_std_mean(z)
        std_new, mean_new = ops.channel_std_mean(small)
        lo, hi = torch.aminmax(z)
        small = torch.clamp((small - mean_new) / std_new * std_old + mean_old, min=lo, max=hi).contiguous()   # thumbnail-sized
        pool = self._scratch()
        self._one = torch.ones(1, dtype=torch.float32, device=z.device)
        tile = self._start_tile(pool, small)
        steps = self._fused_steps()
        n_norm = sum(1 for s_, _ in steps if s_[0] == "norm")
        fixed = []
        for step, fuse in steps:
            if step[0] == "norm":
                a = tile["h"]
                n = a.B * 32
                ws = pool.get((ops.groupnorm_ws_size(a.B, a.HW, a.C),), torch.float64)
                ops.groupnorm_stats(a.t, a.B, a.HW, ws)
                mean = torch.empty(n, dtype=torch.float32, device=z.device)
                var = torch.empty(n, dtype=torch.float32, device=z.device)
                ops.groupnorm_finalize(ws, n, a.HW * (a.C // 32), mean, var)
                fixed.append((mean, var))
                if len(fixed) < n_norm:
                    tile["fuse_silu"] = fuse
                    self._norm_apply(pool, step, tile, sums=ws)
                pool.put(ws)
                if len(fixed) == n_norm:
                    break
            elif color_fix and step[0] == "downsample":
                break
            else:
                self._apply_step(pool, step, tile, fuse)
        held = [tile["h"].t] + [r for r in tile["res"] if r is not tile["h"].t]
        pool.put(*held)
        return fixed + [None] * (n_norm - len(fixed))

    @torch.no_grad()
    def tiled_forward(self, z, tile_size, shard=False, group=None, fast=False, color_fix=False):
        """VAEHook.vae_tile_forward (tilevae.py:819-970), tiles resident in HBM. `fast`: the reference's fast mode — GroupNorm
        statistics estimated once on a thumbnail (estimate_group_norm), every tile then runs independently (no cross-tile
        merge and, when sharded, no statistics exchange: every rank computes the same estimate).

        `shard=True` (opt-in; torch.distributed initialised, identical input on every rank) deals the tiles round-robin over
        the ranks of `group`. Exchanges: per GroupNorm layer ONE all-gather of the per-tile (mean, var) rows (a few KB),
        and at the end ONE all-gather of the cropped output tiles (each rank contributes its crops, packed back to back:
        the canvas crosses NVLink once, nothing is zero-filled or summed)."""
        import torch.distributed as dist
        self._check(z)
        z = z.float().contiguous()
        N, _, height, width = z.shape
        dec = self.is_decoder
        in_bboxes, out_bboxes = split_tiles(height, width, tile_size, dec)
        T = len(in_bboxes)
        world, rank = ((dist.get_world_size(group), dist.get_rank(group))
                       if shard and dist.is_available() and dist.is_initialized() else (1, 0))
        mine = [i for i in range(T) if i % world == rank]
        per = (T + world - 1) // world                 # tile i lives in slot i // world of rank i % world
        pool = self._scratch()
        dev = z.device
        self._one = torch.ones(1, dtype=torch.float32, device=dev)
        tiles = {i: self._start_tile(pool, z[:, :, in_bboxes[i][2]:in_bboxes[i][3], in_bboxes[i][0]:in_bboxes[i][1]]) for i in mine}
        # spatial size of EVERY tile at the current depth (host integers; every rank needs all pixel counts for the merge)
        dims = [(b[3] - b[2], b[1] - b[0]) for b in in_bboxes]
        # pixel-count weights of the cross-tile merge for EVERY GroupNorm layer, from host integers, uploaded ONCE: a
        # host -> device copy inside the layer loop drains the launch queue at each of the ~26 layers (at 2 tiles per rank the
        # pass was CPU-bound on exactly that: 289 ms for 4 passes on 8 GPUs against ~100 ms of kernels)
        plan_steps = self._fused_steps()
        wrows, d2 = [], list(dims)
        for step, _ in plan_steps:
            if step[0] == "upsample":
                d2 = [(2 * h, 2 * w) for h, w in d2]
            elif step[0] == "downsample":
                d2 = [((h + 1 - 3) // 2 + 1, (w + 1 - 3) // 2 + 1) for h, w in d2]
            elif step[0] == "norm":
                pixels = torch.tensor([float(h * w) for h, w in d2], dtype=torch.float32)
                wts = pixels / pixels.max()
                wrows.append(wts / wts.sum())            # GroupNormParam.summary (tilevae.py:629-648)
        wts_all = torch.stack(wrows, 0).to(dev, non_blocking=True) if wrows else None
        fixed = self.estimate_group_norm(z, tile_size, color_fix and not dec) if fast else None
        norm_idx = 0
        for step, fuse in plan_steps:
            if step[0] == "norm" and fixed is not None and fixed[norm_idx] is not None:
                mean, var = fixed[norm_idx]
                norm_idx += 1
                for i in mine:
                    tiles[i]["fuse_silu"] = fuse
                    self._norm_apply(pool, step, tiles[i], mean=mean, var=var)
                continue
            if step[0] != "norm":
                for i in mine:
                    self._apply_step(pool, step, tiles[i], fuse)
                if step[0] == "upsample":
                    dims = [(2 * h, 2 * w) for h, w in dims]
                elif step[0] == "downsample":
                    dims = [((h + 1 - 3) // 2 + 1, (w + 1 - 3) // 2 + 1) for h, w in dims]
                if step[0] in ("upsample", "downsample") and pool.free_bytes() > POOL_TRIM_BYTES:
                    pool.trim()          # scratch of the resolution just left: its sizes do not recur in this pass
                continue
            # cross-tile GroupNorm: per-tile (mean, biased var) -> pixel-weighted merge -> shared apply
            C = step[3]
            n = N * 32
            stats = torch.zeros((per, 2, n), dtype=torch.float32, device=dev)      # this rank's tiles, slot-major
            for i in mine:
                a = tiles[i]["h"]
                ws = pool.get((ops.groupnorm_ws_size(a.B, a.HW, a.C),), torch.float64)
                ops.groupnorm_stats(a.t, a.B, a.HW, ws)
                ops.groupnorm_finalize(ws, n, a.HW * (C // 32), stats[i // world, 0], stats[i // world, 1])
                pool.put(ws)
            if world > 1:
                allst = torch.empty((world, per, 2, n), dtype=torch.float32, device=dev)
                dist.all_gather_into_tensor(allst.view(-1), stats.view(-1), group=group)
                stats = allst.transpose(0, 1).reshape(per * world, 2, n)            # row slot * world + rank == tile index
            t_mean, t_var = stats[:T, 0].contiguous(), stats[:T, 1].contiguous()
            wts = wts_all[norm_idx]
            norm_idx += 1
            mean = torch.empty(n, dtype=torch.float32, device=dev)
            var = torch.empty(n, dtype=torch.float32, device=dev)
            ops.groupnorm_merge_tiles(t_mean, t_var, wts, mean, var)
            for i in mine:
                tiles[i]["fuse_silu"] = fuse
                self._norm_apply(pool, step, tiles[i], mean=mean, var=var)
        s_out = (height * 8, width * 8) if dec else (height // 8, width // 8)
        Cout = self._conv_out[2]
        result = torch.empty((N, Cout) + s_out, dtype=torch.float32, device=dev)
        # crop geometry of every tile from the tracked tile sizes (host integers, identical on all ranks)
        crops = [crop_margins(dims[i][0], dims[i][1], in_bboxes[i], out_bboxes[i], dec) for i in range(T)]
        if world == 1:
            for i in mine:
                ob = out_bboxes[i]
                y0, y1, x0, x1 = crops[i]
                self._finish_tile(pool, tiles[i], result[:, :, ob[2]:ob[3], ob[0]:ob[1]], crop=(y0, x0, y1 - y0, x1 - x0))
            if pool.free_bytes() > POOL_TRIM_BYTES:
                pool.trim()
            return result
        # sharded: every rank packs its cropped tiles back to back; one all-gather; paste
        numel, offs, slot = plan_packed_crops(crops, N * Cout, world)
        packed = torch.empty((world, slot), dtype=torch.float32, device=dev)
        for i in mine:
            y0, y1, x0, x1 = crops[i]
            view = packed[rank, offs[i]:offs[i] + numel[i]].view(N, Cout, y1 - y0, x1 - x0)
            self._finish_tile(pool, tiles[i], view, crop=(y0, x0, y1 - y0, x1 - x0))
        dist.all_gather_into_tensor(packed.view(-1), packed[rank].clone(), group=group)
        paste_packed_crops(result, packed, crops, out_bboxes, numel, offs, world)
        if pool.free_bytes() > POOL_TRIM_BYTES:
            pool.trim()
        return result


def nearest_exact_indices(in_size, scale_factor):
    """Source index of every output pixel of F.interpolate(x, scale_factor=s, mode='nearest-exact') along one axis, computed
    like ATen does (output size floor(in * s); index min(floor((dst + 0.5) * float32(1 / s)), in - 1))."""
    import numpy as np
    out_size = int(math.floor(float(in_size) * scale_factor))
    scale = np.float32(1.0 / scale_factor)
    idx = np.floor((np.arange(out_size, dtype=np.float32) + np.float32(0.5)) * scale).astype(np.int64)
    return torch.from_numpy(np.minimum(idx, in_size - 1))


def plan_packed_crops(crops, planes, world):
    """Layout of the sharded tiled VAE's output exchange: tile i (owner i % world) stores its cropped output, `planes` x
    (y1-y0) x (x1-x0) floats, back to back in its owner's slot. Returns (numel per tile, offset per tile, slot length)."""
    numel = [planes * (c[1] - c[0]) * (c[3] - c[2]) for c in crops]
    offs, fill = [0] * len(crops), [0] * world
    for i in range(len(crops)):
        offs[i] = fill[i % world]
        fill[i % world] += numel[i]
    return numel, offs, max(fill)


def paste_packed_crops(result, packed, crops, out_bboxes, numel, offs, world):
    """Inverse of the packing: result[:, :, output box of tile i] = tile i's crop (tilevae.py:946-948 pastes the same boxes)."""
    N, Cout = result.shape[:2]
    for i, (y0, y1, x0, x1) in enumerate(crops):
        ob = out_bboxes[i]
        result[:, :, ob[2]:ob[3], ob[0]:ob[1]].copy_(packed[i % world, offs[i]:offs[i] + numel[i]].view(N, Cout, y1 - y0, x1 - x0))
    return result


def get_best_tile_size(lowerbound, upperbound):
    """VAEHook.get_best_tile_size (tilevae.py:702-715)."""
    divider = 32
    while divider >= 2:
        remainer = lowerbound % divider
        if remainer == 0:
            return lowerbound
        candidate = lowerbound - remainer + divider
        if candidate <= upperbound:
            return candidate
        divider //= 2
    return lowerbound


def split_tiles(h, w, tile_size, is_decoder):
    """VAEHook.split_tiles (tilevae.py:717-774). Returns (input bboxes, output bboxes), each [x1, x2, y1, y2]."""
    pad = 11 if is_decoder else 32
    num_h = max(math.ceil((h - 2 * pad) / tile_size), 1)
    num_w = max(math.ceil((w - 2 * pad) / tile_size), 1)
    real_h = get_best_tile_size(math.ceil((h - 2 * pad) / num_h), tile_size)
    real_w = get_best_tile_size(math.ceil((w - 2 * pad) / num_w), tile_size)
    tin, tout = [], []
    for i in range(num_h):
        for j in range(num_w):
            box = [pad + j * real_w, min(pad + (j + 1) * real_w, w), pad + i * real_h, min(pad + (i + 1) * real_h, h)]
            o = [box[0] if box[0] > pad else 0, box[1] if box[1] < w - pad else w,
                 box[2] if box[2] > pad else 0, box[3] if box[3] < h - pad else h]
            tout.append([v * 8 if is_decoder else v // 8 for v in o])
            tin.append([max(0, box[0] - pad), min(w, box[1] + pad), max(0, box[2] - pad), min(h, box[3] + pad)])
    return tin, tout


def crop_margins(tile_h, tile_w, input_bbox, target_bbox, is_decoder):
    """crop_valid_region (tilevae.py:556-567) as (y0, y1, x0, x1) index ranges of the tile's output."""
    padded = [i * 8 if is_decoder else i // 8 for i in input_bbox]
    m = [target_bbox[i] - padded[i] for i in range(4)]
    return m[2], tile_h + m[3], m[0], tile_w + m[1]


class Encoder(_VAENet):
    is_decoder = False

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="vanilla", **ignore_kwargs):
        super().__init__()
        if list(attn_resolutions) or use_linear_attn or not resamp_with_conv or attn_type not in ("vanilla", "vanilla-xformers"):
            raise NotImplementedError("Encoder option outside the SDXL VAE config")
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        self.in_channels = in_channels
        self.conv_in = nn.Conv2d(in_channels, ch, 3, 1, 1)
        in_ch_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        for lvl in range(self.num_resolutions):
            block_in, block_out = ch * in_ch_mult[lvl], ch * ch_mult[lvl]
            level = _Level()
            level.block = nn.ModuleList()
            level.attn = nn.ModuleList()
            for _ in range(num_res_blocks):
                level.block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, dropout=dropout))
                block_in = block_out
            if lvl != self.num_resolutions - 1:
                level.downsample = _Down(block_in)
            self.down.append(level)
        self.mid = _Level()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, dropout=dropout)
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, 2 * z_channels if double_z else z_channels, 3, 1, 1)


class Decoder(_VAENet):
    is_decoder = True

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, give_pre_end=False, tanh_out=False,
                 use_linear_attn=False, attn_type="vanilla", **ignorekwargs):
        super().__init__()
        if list(attn_resolutions) or use_linear_attn or not resamp_with_conv or give_pre_end or tanh_out \
                or attn_type not in ("vanilla", "vanilla-xformers"):
            raise NotImplementedError("Decoder option outside the SDXL VAE config")
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        block_in = ch * ch_mult[self.num_resolutions - 1]
        self.conv_in = nn.Conv2d(z_channels, block_in, 3, 1, 1)
        self.mid = _Level()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, dropout=dropout)
        self.up = nn.ModuleList()
        for lvl in reversed(range(self.num_resolutions)):
            block_out = ch * ch_mult[lvl]
            level = _Level()
            level.block = nn.ModuleList()
            level.attn = nn.ModuleList()
            for _ in range(num_res_blocks + 1):
                level.block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, dropout=dropout))
                block_in = block_out
            if lvl != 0:
                level.upsample = _Up(block_in)
            self.up.insert(0, level)
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, 3, 1, 1)


class VAEHook:
    """Drop-in for SUPIR.utils.tilevae.VAEHook (tilevae.py:677-700): bound as `net.forward` by init_tile_vae."""

    def __init__(self, net, tile_size, is_decoder, fast_decoder=False, fast_encoder=False, color_fix=False, to_gpu=False):
        self.net, self.tile_size, self.is_decoder = net, tile_size, is_decoder
        self.fast_mode = (fast_encoder and not is_decoder) or (fast_decoder and is_decoder)      # tilevae.py:682-683
        self.color_fix = color_fix and not is_decoder
        self.pad = 11 if is_decoder else 32
        self.shard, self.process_group = False, None      # tile sharding over torch.distributed ranks is opt-in

    def __call__(self, x):
        B, C, H, W = x.shape
        if max(H, W) <= self.pad * 2 + self.tile_size:
            return self.net.original_forward(x)
        return self.net.tiled_forward(x, self.tile_size, shard=self.shard, group=self.process_group, fast=self.fast_mode,
                                      color_fix=self.color_fix)

    def split_tiles(self, h, w):
        return split_tiles(h, w, self.tile_size, self.is_decoder)

    def get_best_tile_size(self, lowerbound, upperbound):
        return get_best_tile_size(lowerbound, upperbound)


class DiagonalGaussianDistribution:
    """distributions.py:24-41; sample() draws eps on the CPU generator like the reference, the arithmetic is a kernel."""

    def __init__(self, parameters):
        self.parameters = parameters.float().contiguous()

    def _latent(self, eps):
        B, C2 = self.parameters.shape[:2]
        z = torch.empty((B, C2 // 2) + tuple(self.parameters.shape[2:]), dtype=torch.float32, device=self.parameters.device)
        return ops.gaussian_latent(self.parameters, eps, 1.0, z)

    def sample(self):
        shape = (self.parameters.shape[0], self.parameters.shape[1] // 2) + tuple(self.parameters.shape[2:])
        return self._latent(torch.randn(shape).to(device=self.parameters.device))

    def mode(self):
        return self._latent(None)


class _Conv1x1Small(nn.Conv2d):
    """quant_conv / post_quant_conv: <= 8 channels each side, fp32 NCHW (autoencoder.py:297-298)."""

    def forward(self, x, in_scale=1.0):
        if not x.is_cuda:
            raise RuntimeError("supir_b200 VAE needs CUDA tensors: the backend has no CPU path")
        x = x.float().contiguous()
        out = torch.empty((x.shape[0], self.out_channels) + tuple(x.shape[2:]), dtype=torch.float32, device=x.device)
        w = self.weight.detach().reshape(self.out_channels, self.in_channels).to(BF16).float().contiguous()
        return ops.conv1x1_small_nchw(x, w, _bias_bf16_values(self.bias), out, in_scale=in_scale)


class AutoencoderKL(nn.Module):
    def __init__(self, embed_dim, ddconfig, ckpt_path=None, lossconfig=None, monitor=None, ignore_keys=(), **kw):
        super().__init__()
        assert ddconfig["double_z"]
        self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        self.quant_conv = _Conv1x1Small(2 * ddconfig["z_channels"], 2 * embed_dim, 1)
        self.post_quant_conv = _Conv1x1Small(embed_dim, ddconfig["z_channels"], 1)
        self.embed_dim = embed_dim
        if ckpt_path is not None:
            raise NotImplementedError("load weights through the SUPIR checkpoint loader (SUPIR/util.py:15-47)")

    def encode(self, x):
        h = self.encoder(x)
        return DiagonalGaussianDistribution(self.quant_conv(h))

    def decode(self, z, **kw):
        return self.decoder(self.post_quant_conv(z))


class AutoencoderKLInferenceWrapper(AutoencoderKL):
    def encode(self, x):
        return super().encode(x).sample()
