"""ControlNet + ControlledUnetModel forward on the sm_90a kernels.

Replaces ControlLDM.forward (reference model/cldm.py:160-172), i.e. ControlNet.forward
(model/controlnet.py:314-328) and ControlledUnetModel.forward (model/controlnet.py:18-47),
for the SD-2.1 configuration of configs/inference/cldm.yaml (or any channel set that is a
multiple of 64 with 64-wide heads).

Data layout in HBM: activations NHWC; the residual stream / skip tensors / eps are fp32;
every tensor-core operand (normalised activations, Q/K/V, attention output, GEGLU hidden) is
16-bit (lib.operand_dtype()) and exists only between its producer and the GEMM that eats it.

Execution order inside one forward: UNet encoder + middle (produces the skips hs[i]), then
ControlNet, whose zero-conv epilogues write  hs[i] += scale_i * (W h + b)  in place
(fusing cldm.py:164 and controlnet.py:36-43 into the GEMM), then the UNet decoder, which reads
cat([h, hs[i]]) as a *virtual* concat (GroupNorm statistics + operand pass read both sources).

What is hoisted out of the per-step path (constant across sampler steps):
  * text K/V projections of every cross-attention (attention.py:192-193) -> set_context()
  * time-embedding MLP and the per-ResBlock emb_layers (unet.py:616-617, 166-172)
    -> set_timesteps() builds a table indexed by step.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence

import torch

from .. import arch, lib
from .common import Workspace, f32, geglu_tile, op16, pack_conv3x3, pack_geglu, pack_linear

HEAD_DIM = 64


class _Net:
    """Packed weights of one UNet-like network (UNet or ControlNet)."""

    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict, controlnet: bool, device):
        self.cfg = cfg
        self.plan = arch.unet_plan(cfg, controlnet)
        self.controlnet = controlnet
        self.dev = device
        self.w: Dict[str, torch.Tensor] = {}
        shapes = arch.unet_shapes(cfg, controlnet)
        missing = [k for k in shapes if k not in sd]
        if missing:
            raise KeyError(f"checkpoint is missing {len(missing)} keys, e.g. {missing[:3]}")
        for k, shp in shapes.items():
            if tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: checkpoint shape {tuple(sd[k].shape)} != expected {shp}")
        self.res_layers: List[arch.Layer] = []
        self.attn_layers: List[arch.Layer] = []
        for blk in self.plan.input_blocks + [self.plan.middle] + self.plan.output_blocks:
            for l in blk.layers:
                self._pack_layer(sd, l)
        w = self.w
        for nm in ("time_embed.0", "time_embed.2"):
            w[nm + ".weight"] = f32(sd[nm + ".weight"], device)
            w[nm + ".bias"] = f32(sd[nm + ".bias"], device)
        if controlnet:
            for i in range(len(self.plan.input_blocks)):
                w[f"zero_convs.{i}.w"] = pack_linear(sd[f"zero_convs.{i}.0.weight"], device)
                w[f"zero_convs.{i}.b"] = f32(sd[f"zero_convs.{i}.0.bias"], device)
            w["middle_block_out.w"] = pack_linear(sd["middle_block_out.0.weight"], device)
            w["middle_block_out.b"] = f32(sd["middle_block_out.0.bias"], device)
        else:
            w["out.0.weight"] = f32(sd["out.0.weight"], device)
            w["out.0.bias"] = f32(sd["out.0.bias"], device)
            ow = sd["out.2.weight"]
            w["out.2.weight"] = f32(ow.permute(0, 2, 3, 1).reshape(ow.shape[0], -1), device)
            w["out.2.bias"] = f32(sd["out.2.bias"], device)

    def _pack_layer(self, sd, l: arch.Layer):
        w, p, dev = self.w, l.prefix, self.dev
        if l.kind == "conv_in":
            cw = sd[p + "weight"]                           # [Cout, Cin, 3, 3] -> [9*Cin, Cout]
            w[p + "w"] = f32(cw.permute(2, 3, 1, 0).reshape(-1, cw.shape[0]), dev)
            w[p + "b"] = f32(sd[p + "bias"], dev)
        elif l.kind == "res":
            self.res_layers.append(l)
            for nm in ("in_layers.0", "out_layers.0"):
                w[p + nm + ".weight"] = f32(sd[p + nm + ".weight"], dev)
                w[p + nm + ".bias"] = f32(sd[p + nm + ".bias"], dev)
            w[p + "conv1.w"] = pack_conv3x3(sd[p + "in_layers.2.weight"], dev)
            w[p + "conv1.b"] = f32(sd[p + "in_layers.2.bias"], dev)
            w[p + "conv2.w"] = pack_conv3x3(sd[p + "out_layers.3.weight"], dev)
            w[p + "conv2.b"] = f32(sd[p + "out_layers.3.bias"], dev)
            w[p + "emb.w"] = f32(sd[p + "emb_layers.1.weight"], dev)
            w[p + "emb.b"] = f32(sd[p + "emb_layers.1.bias"], dev)
            if l.cin != l.cout:
                w[p + "skip.w"] = pack_linear(sd[p + "skip_connection.weight"], dev)
                w[p + "skip.b"] = f32(sd[p + "skip_connection.bias"], dev)
        elif l.kind == "attn":
            self.attn_layers.append(l)
            c = l.cin
            q = p + "transformer_blocks.0."
            for nm in ("norm",):
                w[p + nm + ".weight"] = f32(sd[p + nm + ".weight"], dev)
                w[p + nm + ".bias"] = f32(sd[p + nm + ".bias"], dev)
            w[p + "proj_in.w"] = pack_linear(sd[p + "proj_in.weight"], dev)
            w[p + "proj_in.b"] = f32(sd[p + "proj_in.bias"], dev)
            w[p + "proj_out.w"] = pack_linear(sd[p + "proj_out.weight"], dev)
            w[p + "proj_out.b"] = f32(sd[p + "proj_out.bias"], dev)
            for nm in ("norm1", "norm2", "norm3"):
                w[q + nm + ".weight"] = f32(sd[q + nm + ".weight"], dev)
                w[q + nm + ".bias"] = f32(sd[q + nm + ".bias"], dev)
            w[q + "qkv.w"] = op16(torch.cat([sd[q + "attn1.to_q.weight"], sd[q + "attn1.to_k.weight"],
                                             sd[q + "attn1.to_v.weight"]], 0), dev)
            w[q + "o1.w"] = pack_linear(sd[q + "attn1.to_out.0.weight"], dev)
            w[q + "o1.b"] = f32(sd[q + "attn1.to_out.0.bias"], dev)
            w[q + "q2.w"] = pack_linear(sd[q + "attn2.to_q.weight"], dev)
            w[q + "kv2.w"] = op16(torch.cat([sd[q + "attn2.to_k.weight"], sd[q + "attn2.to_v.weight"]], 0), dev)
            w[q + "o2.w"] = pack_linear(sd[q + "attn2.to_out.0.weight"], dev)
            w[q + "o2.b"] = f32(sd[q + "attn2.to_out.0.bias"], dev)
            bn = geglu_tile(c)
            w[q + "ff1.w"], w[q + "ff1.b"] = pack_geglu(sd[q + "ff.net.0.proj.weight"],
                                                        sd[q + "ff.net.0.proj.bias"], bn, dev)
            w[q + "ff2.w"] = pack_linear(sd[q + "ff.net.2.weight"], dev)
            w[q + "ff2.b"] = f32(sd[q + "ff.net.2.bias"], dev)
        elif l.kind == "down":
            w[p + "w"] = pack_conv3x3(sd[p + "op.weight"], dev)
            w[p + "b"] = f32(sd[p + "op.bias"], dev)
        elif l.kind == "up":
            w[p + "w"] = pack_conv3x3(sd[p + "conv.weight"], dev)
            w[p + "b"] = f32(sd[p + "conv.bias"], dev)


class CldmEngine:
    def __init__(self, unet_sd, controlnet_sd, unet_cfg: dict = None, controlnet_cfg: dict = None,
                 device="cuda"):
        self.dev = torch.device(device)
        unet_cfg = dict(arch.UNET_CFG if unet_cfg is None else unet_cfg)
        controlnet_cfg = dict(arch.CONTROLNET_CFG if controlnet_cfg is None else controlnet_cfg)
        self.unet = _Net(unet_sd, unet_cfg, False, self.dev)
        self.cnet = _Net(controlnet_sd, controlnet_cfg, True, self.dev)
        self.mc = unet_cfg["model_channels"]
        self.ctx_dim = unet_cfg["context_dim"]
        # Twin layers: the ControlNet is a copy of the UNet encoder + middle block (controlnet.py:50-312), so
        # every layer past the stem has a same-shape twin. Their packed weights are stacked along N
        # ([W_unet ; W_controlnet]) so that both twins run as ONE grouped launch (dbir_gemm groups = 2) on
        # activations stacked along the batch ([UNet images ; ControlNet images]); the per-net entries
        # become views of the stacked tensors (no copy).
        self.twin_w: Dict[str, torch.Tensor] = {}
        self.twin_prefixes = set()
        cn_layers = {l.prefix: l for blk in self.cnet.plan.input_blocks + [self.cnet.plan.middle] for l in blk.layers}
        for blk in self.unet.plan.input_blocks + [self.unet.plan.middle]:
            for l in blk.layers:
                lc = cn_layers.get(l.prefix)
                if l.kind == "conv_in" or lc is None or (lc.kind, lc.cin, lc.cout) != (l.kind, l.cin, l.cout):
                    continue
                self.twin_prefixes.add(l.prefix)
                for k in [k for k in self.unet.w if k.startswith(l.prefix)]:
                    wu, wc = self.unet.w[k], self.cnet.w[k]
                    assert wu.shape == wc.shape and wu.dtype == wc.dtype, k
                    cat = torch.cat([wu, wc], 0).contiguous()
                    self.twin_w[k] = cat
                    self.unet.w[k], self.cnet.w[k] = cat[: wu.shape[0]], cat[wu.shape[0]:]
        self.group_twins = os.environ.get("DBIR_GROUP_TWINS", "1") != "0"
        self.ws = Workspace(self.dev)
        self.op_dtype = lib.operand_dtype()
        self.kv: Dict[str, torch.Tensor] = {}      # per attention layer: op16 [nb*77, 2C]
        self.ctx_len = 0
        self.emb_table: Optional[torch.Tensor] = None
        self.emb_offsets: Dict[str, int] = {}
        self._nb = 0
        self.two_streams = True          # ControlNet || UNet encoder
        self._side = None
        self._ts_key = None
        self._part = {}                  # fp32 activation data_ptr -> (GN partial-sum buffer, slots)
        self._wseq, self._wpos = {}, {}  # per-stream weight sequence of the forward (L2 prefetch lookahead)
        self.prefetch_weights = False    # opt-in: L2 prefetch of the next layers' weights during a GEMM
        self.fuse_gn_stats = True
        # Batch-invariant kernel plans: no split-K, whole attention tiles per CTA. Every sample's result
        # then has the same bits whatever batch it runs in (tiled sampling: sharded == single rank) and
        # whatever plan the timing-based tuner picked (run-to-run / process-to-process reproducible).
        # DBIR_DETERMINISTIC=1 pins it for every forward; the samplers set it for tiled sampling.
        self.deterministic = os.environ.get("DBIR_DETERMINISTIC", "0") == "1"
        self.batch_invariant = self.deterministic
        self.emb_cur = None
        self._graphs = {}                # (shape, scales) -> (CUDAGraph, x_in, c_img, eps, launches)
        self.ws.on_grow = self._graphs.clear

    # ------------------------------------------------------------------ hoisted work
    def set_context(self, c_txt: torch.Tensor):
        """c_txt fp32 [nb, L, ctx_dim] -> K/V of every cross-attention, op16 [nb*L, 2C]."""
        nb, L, d = c_txt.shape
        ctx16 = c_txt.to(self.dev).reshape(nb * L, d).to(self.op_dtype).contiguous()
        self.ctx_len = L
        self._nb = nb
        for l in self.unet.attn_layers:
            q = l.prefix + "transformer_blocks.0."
            twin = l.prefix in self.twin_prefixes
            rows = nb * L
            buf = self.kv.get("g" + l.prefix)
            if buf is None or buf.shape[0] != (2 if twin else 1) * rows:
                # twin layers: [UNet K/V ; ControlNet K/V] back to back (one batched cross-attention)
                buf = torch.empty((2 if twin else 1) * rows, 2 * l.cin, dtype=self.op_dtype, device=self.dev)
                self.kv["g" + l.prefix] = buf
                self.kv["u" + l.prefix] = buf[:rows]
                if twin:
                    self.kv["c" + l.prefix] = buf[rows:]
                self._graphs.clear()
            lib.gemm(ctx16, self.unet.w[q + "kv2.w"], self.kv["u" + l.prefix], M=rows, N=2 * l.cin, K=d)
            if twin:
                lib.gemm(ctx16, self.cnet.w[q + "kv2.w"], self.kv["c" + l.prefix], M=rows, N=2 * l.cin, K=d)

    def set_timesteps(self, timesteps: Sequence[int], nb: int):
        """Time-embedding MLP + emb_layers of every ResBlock for every sampler step.
        Table layout: [steps][ per ResBlock r: nb x Cout_r ] fp32 (rows replicated over the
        batch so each step needs a single device-to-device copy). Cached per (schedule, batch)."""
        key = (tuple(int(t) for t in timesteps), nb)
        if key == self._ts_key:
            return
        S = len(timesteps)
        t = torch.tensor([float(x) for x in timesteps], dtype=torch.float32, device=self.dev)
        offs, total = {}, 0
        for l in self.unet.res_layers:                 # twins adjacent: [UNet rows ; ControlNet rows]
            offs["u" + l.prefix] = total
            total += nb * l.cout
            if l.prefix in self.twin_prefixes:
                offs["c" + l.prefix] = total
                total += nb * l.cout
        for l in self.cnet.res_layers:
            if "c" + l.prefix not in offs:
                offs["c" + l.prefix] = total
                total += nb * l.cout
        table = torch.empty(S, total, dtype=torch.float32, device=self.dev)
        emb_dim = 4 * self.mc
        for net, tag in ((self.unet, "u"), (self.cnet, "c")):
            te = torch.empty(S, self.mc, dtype=torch.float32, device=self.dev)
            lib.timestep_embedding(t, S, self.mc, te)
            h1 = torch.empty(S, emb_dim, dtype=torch.float32, device=self.dev)
            lib.linear_f32(te, self.mc, S, self.mc, net.w["time_embed.0.weight"],
                           net.w["time_embed.0.bias"], emb_dim, h1, emb_dim, silu_out=True)
            # every consumer is emb_layers = SiLU -> Linear (unet.py:166-172): apply the SiLU once
            emb_act = torch.empty(S, emb_dim, dtype=torch.float32, device=self.dev)
            lib.linear_f32(h1, emb_dim, S, emb_dim, net.w["time_embed.2.weight"],
                           net.w["time_embed.2.bias"], emb_dim, emb_act, emb_dim, silu_out=True)
            tmp = torch.empty(S, max(l.cout for l in net.res_layers), dtype=torch.float32, device=self.dev)
            for l in net.res_layers:
                o = offs[tag + l.prefix]
                y = tmp[:, : l.cout]
                lib.linear_f32(emb_act, emb_dim, S, emb_dim, net.w[l.prefix + "emb.w"],
                               net.w[l.prefix + "emb.b"], l.cout, y, tmp.shape[1])
                table[:, o:o + nb * l.cout] = y.repeat(1, nb)
        self.emb_table = table
        self.emb_offsets = offs
        self.emb_nb = nb
        if self.emb_cur is None or self.emb_cur.numel() != total:
            self.emb_cur = torch.empty(total, dtype=torch.float32, device=self.dev)
            self._graphs.clear()            # graphs hold the old buffer's address
        self.timesteps = list(timesteps)
        self._ts_key = key

    def load_step(self, step_idx: int):
        """Selects the time embedding of sampler step `step_idx` (one D2D copy, outside graphs)."""
        self.emb_cur.copy_(self.emb_table[step_idx])

    def _gemm(self, tag: str, a, b, *args, **kw):
        """dbir_gemm with this stream's split-K scratch (64 MiB, zero-initialised once) and an L2
        prefetch of the weights of the GEMM that follows on the same stream (weights are the only
        cold operand of a forward: 2.5 GB streamed from HBM per step, activations are L2-resident).
        The weight sequence is learnt on the previous forward (it never changes)."""
        ws = self.ws.get(tag + ":splitk", (16 * 1024 * 1024 + 16384,), torch.float32, zero=True)
        seq = self._wseq.setdefault(tag, [])
        i = self._wpos.get(tag, 0)
        wbytes = b.numel() * b.element_size()
        if i < len(seq):
            if seq[i][0] != b.data_ptr():          # sequence changed (other shapes): relearn
                del seq[i:]
        if i >= len(seq):
            seq.append((b.data_ptr(), wbytes))
        self._wpos[tag] = i + 1
        pf = None
        if self.prefetch_weights and i + 1 < len(seq):
            pf = seq[i + 1]
        if self.batch_invariant:
            kw.setdefault("split_k", 1)
        lib.gemm(a, b, *args, splitk_ws=ws, prefetch=pf, **kw)

    def _emb(self, tag: str, l: arch.Layer, nb: int) -> torch.Tensor:
        """Time-embedding rows of ResBlock l for this call's images; tag "g" = both twins ([UNet ; ControlNet])."""
        if tag == "g":
            o = self.emb_offsets["u" + l.prefix]
            assert self.emb_offsets["c" + l.prefix] == o + (nb // 2) * l.cout
            return self.emb_cur[o:o + nb * l.cout]
        o = self.emb_offsets[tag + l.prefix]
        return self.emb_cur[o:o + nb * l.cout]

    # ------------------------------------------------------------------ blocks
    # Every block method takes the weight table W (a net's, or self.twin_w for grouped twin launches),
    # the workspace / stream tag ("u", "c", or "g" for the twins), the TOTAL number of images nb of the
    # call and G = problems stacked along the batch (1, or 2: first nb/2 images are the UNet's, the rest
    # the ControlNet's; weights / norm parameters of problem g sit at offset g in the stacked tensors).
    def _gn(self, tag, src1, src2, c1, c2, nb, h, w, eps, gamma, beta, out16, silu, out_raw=None, G=1):
        """GroupNorm(+SiLU) of the virtual concat [src1 | src2] -> 16-bit operand. Statistics come
        from the partial sums the producing GEMM epilogues emitted (dbir_gn_finalize); tensors
        without partials (the stem conv output) take the stand-alone statistics kernel."""
        ws = self.ws
        stats = ws.get(tag + ":gn_stats", (nb * 64,), torch.float32)
        p1 = self._part.get(src1.data_ptr())
        p2 = self._part.get(src2.data_ptr()) if src2 is not None else None
        if self.fuse_gn_stats and p1 is not None and (src2 is None or p2 is not None):
            lib.gn_finalize(p1[0], p1[1], c1, p2[0] if p2 else None, p2[1] if p2 else 0, c2, nb, h * w, eps, stats)
        else:
            wsp = ws.get(tag + ":gn_ws", (lib.gn_workspace_floats(nb, h * w, c1 + c2),), torch.float32, zero=True)
            lib.gn_stats(src1, src2, c1, c2, nb, h * w, eps, stats, wsp)
        lib.gn_apply(src1, src2, c1, c2, nb, h, w, stats, gamma, beta, out16, norm=True, silu=silu,
                     out_raw=out_raw, imgs_per_group=nb // G if G > 1 else 0)

    def _stats_kw(self, out: torch.Tensor, nb: int, n_cols: int, conv_hw=None, rows_per_img: int = 0) -> dict:
        """kwargs that make dbir_gemm emit GroupNorm partial sums for its output tensor `out`."""
        if not self.fuse_gn_stats:
            return {}
        slots = lib.gemm_gn_slots(*conv_hw) if conv_hw else lib.gemm_gn_slots(0, 0, rows_per_img)
        if slots <= 0:
            self._part.pop(out.data_ptr(), None)
            return {}
        buf = self.ws.get(f"part:{out.data_ptr()}", (nb * slots * n_cols * 2,), torch.float32)
        self._part[out.data_ptr()] = (buf, slots)
        return dict(gn_partials=buf) if conv_hw else dict(gn_partials=buf, gn_rows_per_img=rows_per_img)

    def _res(self, W, tag: str, l: arch.Layer, src1, src2, c1, c2, nb, h, w, out, G=1):
        """ResBlock._forward (unet.py:203-223): out may alias src1 when c2 == 0."""
        ws, p = self.ws, l.prefix
        cin, cout, M = c1 + c2, l.cout, nb * h * w
        a16 = ws.get(tag + ":res_a16", (M, cin), self.op_dtype)
        raw16 = ws.get(tag + ":res_raw16", (M, cin), self.op_dtype) if cin != cout else None
        self._gn(tag, src1, src2, c1, c2, nb, h, w, 1e-5, W[p + "in_layers.0.weight"],
                 W[p + "in_layers.0.bias"], a16, True, out_raw=raw16, G=G)
        h1 = ws.get(tag + ":res_h1", (M, cout), torch.float32)
        self._gemm(tag, a16, W[p + "conv1.w"], h1, M=M, N=cout, K=9 * cin, bias=W[p + "conv1.b"],
                   rowvec=self._emb(tag, l, nb), conv=(nb, h, w, cin, 3), groups=G,
                   **self._stats_kw(h1, nb, cout, conv_hw=(h, w)))
        b16 = ws.get(tag + ":res_b16", (M, cout), self.op_dtype)
        self._gn(tag, h1, None, cout, 0, nb, h, w, 1e-5, W[p + "out_layers.0.weight"],
                 W[p + "out_layers.0.bias"], b16, True, G=G)
        if cin != cout:
            skip = ws.get(tag + ":res_skip", (M, cout), torch.float32)
            self._gemm(tag, raw16, W[p + "skip.w"], skip, M=M, N=cout, K=cin, bias=W[p + "skip.b"], groups=G)
            res = skip
        else:
            res = src1
        self._gemm(tag, b16, W[p + "conv2.w"], out, M=M, N=cout, K=9 * cout, bias=W[p + "conv2.b"],
                   residual=res, conv=(nb, h, w, cout, 3), groups=G, **self._stats_kw(out, nb, cout, conv_hw=(h, w)))

    def _attn(self, W, tag: str, l: arch.Layer, x, nb, h, w, G=1):
        """SpatialTransformer.forward, in place on x (fp32 NHWC [nb,h,w,C]) — attention.py:334-353."""
        ws, p = self.ws, l.prefix
        q = p + "transformer_blocks.0."
        c, M, hw = l.cin, nb * h * w, h * w
        heads = c // HEAD_DIM
        rpg = M // G if G > 1 else 0                  # LayerNorm rows per stacked problem
        a16 = ws.get(tag + ":at_a16", (M, c), self.op_dtype)
        self._gn(tag, x, None, c, 0, nb, h, w, 1e-6, W[p + "norm.weight"], W[p + "norm.bias"], a16, False, G=G)
        t = ws.get(tag + ":at_t", (M, c), torch.float32)
        self._gemm(tag, a16, W[p + "proj_in.w"], t, M=M, N=c, K=c, bias=W[p + "proj_in.b"], groups=G)
        # self-attention
        lib.layernorm(t, c, M, c, W[q + "norm1.weight"], W[q + "norm1.bias"], a16, c, rows_per_group=rpg)
        qkv = ws.get(tag + ":at_qkv", (M, 3 * c), self.op_dtype)
        self._gemm(tag, a16, W[q + "qkv.w"], qkv, M=M, N=3 * c, K=c, groups=G)
        att = ws.get(tag + ":at_o16", (M, c), self.op_dtype)
        nws = lib.attention_ws_bytes(nb, heads, hw, hw)
        aws = ws.get(tag + ":at_sk", (nws // 4,), torch.float32, zero=True) if nws and not self.batch_invariant else None
        lib.attention(qkv, qkv[:, c:], qkv[:, 2 * c:], att, batch=nb, heads=heads, sq=hw, skv=hw,
                      ldq=3 * c, ldk=3 * c, ldv=3 * c, ldo=c, ws=aws)
        self._gemm(tag, att, W[q + "o1.w"], t, M=M, N=c, K=c, bias=W[q + "o1.b"], residual=t, groups=G)
        # cross-attention on the (pre-projected) text context
        lib.layernorm(t, c, M, c, W[q + "norm2.weight"], W[q + "norm2.bias"], a16, c, rows_per_group=rpg)
        q16 = ws.get(tag + ":at_q16", (M, c), self.op_dtype)
        self._gemm(tag, a16, W[q + "q2.w"], q16, M=M, N=c, K=c, groups=G)
        kv = self.kv[tag + l.prefix]
        lib.attention(q16, kv, kv[:, c:], att, batch=nb, heads=heads, sq=hw, skv=self.ctx_len,
                      ldq=c, ldk=2 * c, ldv=2 * c, ldo=c)
        self._gemm(tag, att, W[q + "o2.w"], t, M=M, N=c, K=c, bias=W[q + "o2.b"], residual=t, groups=G)
        # GEGLU feed-forward
        lib.layernorm(t, c, M, c, W[q + "norm3.weight"], W[q + "norm3.bias"], a16, c, rows_per_group=rpg)
        ffh = ws.get(tag + ":at_ffh", (M, 4 * c), self.op_dtype)
        self._gemm(tag, a16, W[q + "ff1.w"], ffh, M=M, N=8 * c, K=c, bias=W[q + "ff1.b"], geglu=True,
                   force_bn=geglu_tile(c), groups=G)
        self._gemm(tag, ffh, W[q + "ff2.w"], a16, M=M, N=c, K=4 * c, bias=W[q + "ff2.b"], residual=t, groups=G)
        self._gemm(tag, a16, W[p + "proj_out.w"], x, M=M, N=c, K=c, bias=W[p + "proj_out.b"], residual=x,
                   groups=G, **self._stats_kw(x, nb, c, rows_per_img=hw))

    def _down(self, W, tag: str, l: arch.Layer, x, nb, h, w, out, G=1):
        c, ho, wo = l.cin, h // 2, w // 2
        col = self.ws.get(tag + ":down_col", (nb * ho * wo, 9 * c), self.op_dtype)
        lib.im2col_s2(x, nb, h, w, c, 1, col)
        self._gemm(tag, col, W[l.prefix + "w"], out, M=nb * ho * wo, N=l.cout, K=9 * c,
                   bias=W[l.prefix + "b"], groups=G, **self._stats_kw(out, nb, l.cout, rows_per_img=ho * wo))

    def _up(self, W, tag: str, l: arch.Layer, x, nb, h, w, out):
        c = l.cin
        up16 = self.ws.get("up_a16", (nb * 4 * h * w, c), self.op_dtype)
        lib.gn_apply(x, None, c, 0, nb, h, w, None, None, None, up16, norm=False, silu=False, upsample=2)
        self._gemm(tag, up16, W[l.prefix + "w"], out, M=nb * 4 * h * w, N=l.cout, K=9 * c,
                   bias=W[l.prefix + "b"], conv=(nb, 2 * h, 2 * w, c, 3),
                   **self._stats_kw(out, nb, l.cout, conv_hw=(2 * h, 2 * w)))

    def _encoder(self, net: _Net, tag: str, x_in, hint, nb, h, w):
        """Input blocks + middle of ONE net. Returns (list of (tensor, c, h, w) per input block, middle)."""
        ws, W = self.ws, net.w
        outs = []
        cur, ch, cw, cc = None, h, w, 0
        for bi, blk in enumerate(net.plan.input_blocks):
            for l in blk.layers:
                if l.kind == "conv_in":
                    o = ws.get(f"{tag}_hs{bi}", (nb * h * w, l.cout), torch.float32)
                    c1 = x_in.shape[1]
                    c2 = hint.shape[1] if hint is not None else 0
                    lib.conv3x3_small_cin(x_in, hint, c1, c2, nb, h, w, W[l.prefix + "w"],
                                          W[l.prefix + "b"], l.cout, o)
                    self._part.pop(o.data_ptr(), None)      # written without GEMM partials
                    cur, cc = o, l.cout
                elif l.kind == "res":
                    o = ws.get(f"{tag}_hs{bi}", (nb * ch * cw, l.cout), torch.float32)
                    self._res(W, tag, l, cur, None, cc, 0, nb, ch, cw, o)
                    cur, cc = o, l.cout
                elif l.kind == "attn":
                    self._attn(W, tag, l, cur, nb, ch, cw)
                elif l.kind == "down":
                    o = ws.get(f"{tag}_hs{bi}", (nb * (ch // 2) * (cw // 2), l.cout), torch.float32)
                    self._down(W, tag, l, cur, nb, ch, cw, o)
                    cur, cc, ch, cw = o, l.cout, ch // 2, cw // 2
            outs.append((cur, cc, ch, cw))
        mid = ws.get(f"{tag}_mid", (nb * ch * cw, cc), torch.float32)
        m = net.plan.middle.layers
        self._res(W, tag, m[0], cur, None, cc, 0, nb, ch, cw, mid)
        self._attn(W, tag, m[1], mid, nb, ch, cw)
        self._res(W, tag, m[2], mid, None, cc, 0, nb, ch, cw, mid)
        return outs, (mid, cc, ch, cw)

    def twins_feasible(self, nb: int, h: int, w: int) -> bool:
        """Grouped twin launches need every stacked problem to start on a 128-row tile boundary (plain
        GEMMs) and conv tiles not to straddle the two nets: true for even nb with >= 64 pixels at the
        coarsest level (the 512^2 / tiled production shapes); reduced test shapes take the two-stream path."""
        if not self.group_twins or set(l.prefix for blk in self.cnet.plan.input_blocks[1:] + [self.cnet.plan.middle]
                                       for l in blk.layers) - self.twin_prefixes:
            return False
        ch, cw = h, w
        for blk in self.unet.plan.input_blocks:
            for l in blk.layers:
                if l.kind == "down":
                    ch, cw = ch // 2, cw // 2
        px = ch * cw                                   # pixels per image at the coarsest level
        if (nb * px) % 128 != 0:
            return False
        imgs_per_tile = max(1, 128 // px)              # conv tiles of 128 pixels span this many images
        return nb % imgs_per_tile == 0

    def _encoder_twins(self, x_in, hint, nb, h, w):
        """UNet encoder + middle and ControlNet as ONE stream of grouped launches: activations are stacked
        along the batch ([nb UNet images ; nb ControlNet images]), every twin layer is one dbir_gemm with
        groups = 2 (norm kernels pick the gamma / beta set by image). Halves the launch count of the
        encoder half of the forward and doubles the wave fill of its single-wave grids.
        Returns (UNet skips, UNet middle, ControlNet outputs, ControlNet middle) as views of the stacked buffers."""
        ws, U, Cn, W, tag = self.ws, self.unet, self.cnet, self.twin_w, "g"
        n2 = 2 * nb
        outs = []
        cur, ch, cw, cc = None, h, w, 0
        for bi, blk in enumerate(U.plan.input_blocks):
            for l in blk.layers:
                if l.kind == "conv_in":                     # the stems differ (4 vs 4 + 4 input channels)
                    o = ws.get(f"g_hs{bi}", (n2 * h * w, l.cout), torch.float32)
                    half = nb * h * w
                    lib.conv3x3_small_cin(x_in, None, x_in.shape[1], 0, nb, h, w, U.w[l.prefix + "w"],
                                          U.w[l.prefix + "b"], l.cout, o[:half])
                    lib.conv3x3_small_cin(x_in, hint, x_in.shape[1], hint.shape[1], nb, h, w, Cn.w[l.prefix + "w"],
                                          Cn.w[l.prefix + "b"], l.cout, o[half:])
                    self._part.pop(o.data_ptr(), None)      # written without GEMM partials
                    cur, cc = o, l.cout
                elif l.kind == "res":
                    o = ws.get(f"g_hs{bi}", (n2 * ch * cw, l.cout), torch.float32)
                    self._res(W, tag, l, cur, None, cc, 0, n2, ch, cw, o, G=2)
                    cur, cc = o, l.cout
                elif l.kind == "attn":
                    self._attn(W, tag, l, cur, n2, ch, cw, G=2)
                elif l.kind == "down":
                    o = ws.get(f"g_hs{bi}", (n2 * (ch // 2) * (cw // 2), l.cout), torch.float32)
                    self._down(W, tag, l, cur, n2, ch, cw, o, G=2)
                    cur, cc, ch, cw = o, l.cout, ch // 2, cw // 2
            outs.append((cur, cc, ch, cw))
        mid = ws.get("g_mid", (n2 * ch * cw, cc), torch.float32)
        m = U.plan.middle.layers
        self._res(W, tag, m[0], cur, None, cc, 0, n2, ch, cw, mid, G=2)
        self._attn(W, tag, m[1], mid, n2, ch, cw, G=2)
        self._res(W, tag, m[2], mid, None, cc, 0, n2, ch, cw, mid, G=2)

        def halves(t, c, th, tw):
            r = nb * th * tw
            return (t[:r], c, th, tw), (t[r:], c, th, tw)
        hs, chs = zip(*(halves(*o) for o in outs))
        umid, cmid = halves(mid, cc, ch, cw)
        return list(hs), umid, list(chs), cmid

    # ------------------------------------------------------------------ CUDA graph of one forward
    def graphed_forward(self, nb: int, c: int, h: int, w: int, control_scales: Sequence[float]):
        """Returns (graph, x_in, c_img, eps, kernels_per_replay): static input/output buffers and
        a CUDA graph of forward(x_in, c_img) -> eps, captured once per (shape, strength) and
        reused across images (set_context / load_step only rewrite buffers the graph reads)."""
        key = (nb, c, h, w, tuple(float(s) for s in control_scales), self.two_streams, self.batch_invariant,
               self.group_twins)
        hit = self._graphs.get(key)
        if hit is not None:
            return hit
        x_in = torch.zeros(nb, c, h, w, device=self.dev)
        c_img = torch.zeros(nb, c, h, w, device=self.dev)
        eps = torch.empty(nb, c, h, w, device=self.dev)
        # warm-up: sizes every workspace buffer; on one stream first, so that the GEMM plans tuned on
        # first use (dbir_gemm) are timed without a concurrent branch
        two, self.two_streams = self.two_streams, False
        self.forward(x_in, c_img, control_scales, out=eps)
        self.two_streams = two
        if two:
            self.forward(x_in, c_img, control_scales, out=eps)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        n0 = lib.launches()
        with torch.cuda.graph(graph):
            self.forward(x_in, c_img, control_scales, out=eps)
        n = lib.launches() - n0
        lib.count_launch(-n)                                       # capture executes nothing
        self._graphs[key] = (graph, x_in, c_img, eps, n)
        return self._graphs[key]

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor, c_img: torch.Tensor, control_scales: Sequence[float],
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """eps/v = ControlLDM.forward(x, t, {c_txt, c_img}) for the step loaded with load_step()
        and the context given to set_context(). x, c_img: fp32 NCHW [nb, 4, h, w] on the device.
        Returns fp32 NCHW [nb, 4, h, w]."""
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        assert c_img.is_cuda and c_img.dtype == torch.float32 and c_img.is_contiguous()
        nb, _, h, w = x.shape
        assert nb == self._nb == self.emb_nb, "set_context / set_timesteps batch mismatch"
        self._wpos = {}
        ws, U, Cn = self.ws, self.unet, self.cnet
        # 1+2. UNet encoder + middle and the ControlNet. Production shapes: their twin layers run as ONE
        #      stream of grouped launches on batch-stacked activations (_encoder_twins). Otherwise: UNet
        #      on the current stream, ControlNet concurrently on a side stream (fork/join with events so
        #      the pair is also captured as parallel graph branches).
        main = torch.cuda.current_stream()
        if self.twins_feasible(nb, h, w):
            hs, (mid, mc_, mh, mw), chs, (cmid, cmc, cmh, cmw) = self._encoder_twins(x, c_img, nb, h, w)
        elif self.two_streams:
            if self._side is None:
                self._side = torch.cuda.Stream(device=self.dev)
                self._ev_fork, self._ev_join = torch.cuda.Event(), torch.cuda.Event()
            self._ev_fork.record(main)
            self._side.wait_event(self._ev_fork)
            with torch.cuda.stream(self._side):
                chs, (cmid, cmc, cmh, cmw) = self._encoder(Cn, "c", x, c_img, nb, h, w)
                self._ev_join.record(self._side)
            hs, (mid, mc_, mh, mw) = self._encoder(U, "u", x, None, nb, h, w)
            main.wait_event(self._ev_join)
        else:
            hs, (mid, mc_, mh, mw) = self._encoder(U, "u", x, None, nb, h, w)
            chs, (cmid, cmc, cmh, cmw) = self._encoder(Cn, "c", x, c_img, nb, h, w)
        # zero-convs accumulate scale_i * (W h + b) into the UNet skips / middle in place
        for i, (t, c, th, tw) in enumerate(chs):
            M = nb * th * tw
            a16 = ws.get("zc_a16", (M, c), self.op_dtype)
            lib.gn_apply(t, None, c, 0, nb, th, tw, None, None, None, a16, norm=False, silu=False)
            tgt = hs[i][0]
            self._gemm("u", a16, Cn.w[f"zero_convs.{i}.w"], tgt, M=M, N=c, K=c, bias=Cn.w[f"zero_convs.{i}.b"],
                       alpha=float(control_scales[i]), residual=tgt, **self._stats_kw(tgt, nb, c, rows_per_img=th * tw))
        M = nb * cmh * cmw
        a16 = ws.get("zc_a16", (M, cmc), self.op_dtype)
        lib.gn_apply(cmid, None, cmc, 0, nb, cmh, cmw, None, None, None, a16, norm=False, silu=False)
        self._gemm("u", a16, Cn.w["middle_block_out.w"], mid, M=M, N=cmc, K=cmc, bias=Cn.w["middle_block_out.b"],
                   alpha=float(control_scales[len(chs)]), residual=mid, **self._stats_kw(mid, nb, cmc, rows_per_img=cmh * cmw))
        # 3. UNet decoder over virtual concats
        cur, cc, ch, cw = mid, mc_, mh, mw
        stack = list(hs)
        for bi, blk in enumerate(U.plan.output_blocks):
            for l in blk.layers:
                if l.kind == "res":
                    skip, sc, sh, sw = stack.pop()
                    assert (sh, sw) == (ch, cw) and cc + sc == l.cin
                    o = ws.get(f"u_out{bi % 2}", (nb * ch * cw, l.cout), torch.float32)
                    self._res(U.w, "u", l, cur, skip, cc, sc, nb, ch, cw, o)
                    cur, cc = o, l.cout
                elif l.kind == "attn":
                    self._attn(U.w, "u", l, cur, nb, ch, cw)
                elif l.kind == "up":
                    o = ws.get(f"u_up{bi % 2}", (nb * 4 * ch * cw, l.cout), torch.float32)
                    self._up(U.w, "u", l, cur, nb, ch, cw, o)
                    cur, cc, ch, cw = o, l.cout, ch * 2, cw * 2
        # 4. out = conv(silu(gn(h)))  (unet.py:675-679)
        a16 = ws.get("u:res_a16", (nb * ch * cw, cc), self.op_dtype)
        self._gn("u", cur, None, cc, 0, nb, ch, cw, 1e-5, U.w["out.0.weight"], U.w["out.0.bias"], a16, True)
        oc = U.cfg["out_channels"]
        if out is None:
            out = torch.empty(nb, oc, ch, cw, dtype=torch.float32, device=self.dev)
        lib.conv3x3_small_cout(a16, nb, ch, cw, cc, U.w["out.2.weight"], U.w["out.2.bias"], oc, out,
                               nchw=True)
        return out
