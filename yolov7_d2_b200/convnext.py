"""ConvNeXt backbone on the H100 kernels: execution plan (ConvNeXtEngine) and the reference-facing module.

Reference: yolov7/modeling/backbone/convnext.py -- `Block` :25-60, `ConvNeXt` :62-180 (forward_features :149-159), `LayerNorm` :182-206,
`build_convnext_backbone` :209-230.  Parameter names / shapes are the reference's state_dict; parameters and gradients live in flat
fp32 buffers (same contract as engine.YoloxEngine, so optim.FlatOptimizer and the single gradient all-reduce apply unchanged).

Data layout: NHWC bf16 activations.  Per block the plan keeps x (input), d (depthwise output), per-pixel LayerNorm statistics, y (normalised),
u (pwconv1 pre-activation), h = GELU(u) and the block output; the 4C-wide du gradient and the C-wide temporaries are shared per stage.
Kernel sequence of one block (forward 4 launches, backward 11):
  dwconv7 -> layernorm_fwd -> linear_gelu_fwd (wgmma GEMM, bias+GELU epilogue) -> conv2d_affine_fwd (GEMM, gamma*b2 shift + residual epilogue)
  colsum(dOut) | linear_dgrad_gelu (GEMM, GELU' epilogue, db1 column sums) | wgrad(h, dOut) + layer_scale_grad | dgrad(du) | wgrad(y, du)
  | layernorm_bwd | dwconv7(flip, + dOut) | dwconv7_wgrad
There is no CPU implementation: every method needs the CUDA library.
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import capi

LN_EPS = 1e-6


class _T:
    """NHWC bf16 tensor + cached yb200_act view"""

    def __init__(self, n, h, w, c, dev):
        self.t = torch.zeros(n, h, w, c, dtype=torch.bfloat16, device=dev)
        self._a = capi.act(self.t)

    @property
    def a(self):
        return ctypes.byref(self._a)


class ConvNeXtEngine:
    def __init__(self, batch, height, width, depths=(3, 3, 9, 3), dims=(96, 192, 384, 768), layer_scale_init_value=1e-6, out_indices=(0, 1, 2, 3),
                 device="cuda", share_params_of=None):
        if height % 32 or width % 32:
            raise ValueError("ConvNeXt input must be a multiple of 32 (size_divisibility, convnext.py:170-180)")
        if any(d % 32 for d in dims):
            raise capi.Yb200Error("ConvNeXtEngine: stage widths must be multiples of 32 (depthwise kernel channel slices)")
        self.L = capi.lib()
        self.dev = torch.device(device)
        self.n, self.h, self.w = batch, height, width
        self.depths, self.dims = tuple(depths), tuple(dims)
        self.layer_scale = layer_scale_init_value
        self.out_indices = tuple(out_indices)
        # the reference runs all four stages even when the last ones are not returned (convnext.py:149-159); their outputs are discarded,
        # so the plan stops after the last returned stage (their parameters receive zero gradients, as in the reference)
        self.n_stages = max(self.out_indices) + 1
        self.kernel_launches = 0
        self.trace = None
        self._alloc_params(share_params_of)
        self._alloc_runtime()

    # ------------------------------------------------------------------ parameters
    def _specs(self):
        d = self.dims
        specs = [("downsample_layers.0.0.weight", (d[0], 3, 4, 4)), ("downsample_layers.0.0.bias", (d[0],)),
                 ("downsample_layers.0.1.weight", (d[0],)), ("downsample_layers.0.1.bias", (d[0],))]
        for i in range(3):
            p = f"downsample_layers.{i + 1}."
            specs += [(p + "0.weight", (d[i],)), (p + "0.bias", (d[i],)), (p + "1.weight", (d[i + 1], d[i], 2, 2)), (p + "1.bias", (d[i + 1],))]
        for i in range(4):
            c = d[i]
            for j in range(self.depths[i]):
                p = f"stages.{i}.{j}."
                specs += [(p + "dwconv.weight", (c, 1, 7, 7)), (p + "dwconv.bias", (c,)), (p + "norm.weight", (c,)), (p + "norm.bias", (c,)),
                          (p + "pwconv1.weight", (4 * c, c)), (p + "pwconv1.bias", (4 * c,)), (p + "pwconv2.weight", (c, 4 * c)), (p + "pwconv2.bias", (c,))]
                if self.layer_scale > 0:
                    specs.append((p + "gamma", (c,)))
        for i in range(4):
            specs += [(f"norm{i}.weight", (d[i],)), (f"norm{i}.bias", (d[i],))]
        return specs

    def _alloc_params(self, share):
        specs = self._specs()
        offs, total = {}, 0
        for name, shape in specs:
            offs[name] = total
            total = (total + math.prod(shape) + 3) // 4 * 4  # 16-byte alignment of every tensor
        if share is not None:
            assert share.param_names == [n for n, _ in specs], "architectures differ"
        dev = self.dev
        self.flat_param = share.flat_param if share is not None else torch.zeros(total, device=dev)
        self.flat_grad = share.flat_grad if share is not None else torch.zeros(total, device=dev)
        self.params, self.grads = {}, {}
        for name, shape in specs:
            n = math.prod(shape)
            self.params[name] = self.flat_param[offs[name]:offs[name] + n].view(shape)
            self.grads[name] = self.flat_grad[offs[name]:offs[name] + n].view(shape)
        self.param_names = [n for n, _ in specs]
        self.param_specs = specs
        self.param_layout = [(n, offs[n], math.prod(s)) for n, s in specs]
        if self.layer_scale <= 0:  # gamma is None in the reference: identity scale, no gradient
            self._ones = {c: torch.ones(c, device=dev) for c in set(self.dims)}

    def init_weights(self, seed=0):
        """ConvNeXt._init_weights (convnext.py:119-122): trunc_normal(std .02) conv / linear weights, zero biases, LN 1 / 0, gamma = init value"""
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, shape in self.param_specs:
                p = self.params[name]
                if name.endswith("gamma"):
                    p.fill_(self.layer_scale)
                elif name.endswith(".bias"):
                    p.zero_()
                elif len(shape) == 1:
                    p.fill_(1.0)
                else:
                    t = torch.empty(shape)
                    torch.nn.init.trunc_normal_(t, std=0.02, generator=g)
                    p.copy_(t)

    def load_state_dict(self, sd, prefix=""):
        with torch.no_grad():
            for name in self.param_names:
                self.params[name].copy_(sd[prefix + name].to(self.dev))

    def state_dict(self):
        return {n: self.params[n].detach().clone() for n in self.param_names}

    # ------------------------------------------------------------------ plan
    def _alloc_runtime(self):
        dev, n = self.dev, self.n
        L = self.L
        self.images = None  # set by the caller: uint8 or fp32 [N,3,H,W] on the device
        self.images_u8 = torch.zeros(n, 3, self.h, self.w, dtype=torch.uint8, device=dev)
        self.stage = []
        self.packed = {}
        ws_need = [16]
        h, w = self.h // 4, self.w // 4
        self.patches = _T(n, h, w, 48, dev)
        for i, c in enumerate(self.dims):
            st = type("Stage", (), {})()
            st.c, st.h, st.w = c, h, w
            st.npix = n * h * w
            if i == 0:
                st.ds_conv = _T(n, h, w, c, dev)       # stem conv output (input of the stem LayerNorm)
            else:
                st.ds_ln = _T(n, 2 * h, 2 * w, self.dims[i - 1], dev)  # LayerNorm output feeding the 2x2 convolution
            st.ds_stats = torch.zeros(n * (h if i == 0 else 2 * h) * (w if i == 0 else 2 * w), 2, device=dev)
            st.x0 = _T(n, h, w, c, dev)                 # stage input (downsample output)
            st.blocks = []
            for _ in range(self.depths[i]):
                b = type("Block", (), {})()
                b.d, b.y, b.out = _T(n, h, w, c, dev), _T(n, h, w, c, dev), _T(n, h, w, c, dev)
                b.u, b.hh = _T(n, h, w, 4 * c, dev), _T(n, h, w, 4 * c, dev)
                b.stats = torch.zeros(st.npix, 2, device=dev)
                st.blocks.append(b)
            st.out = _T(n, h, w, c, dev)                # norm{i} output (returned feature)
            st.out_stats = torch.zeros(st.npix, 2, device=dev)
            # gradient temporaries shared by the blocks of the stage
            st.g = [_T(n, h, w, c, dev), _T(n, h, w, c, dev)]   # ping-pong: gradient w.r.t. a block's output / input
            st.gout = _T(n, h, w, c, dev)                        # gradient of the returned feature (filled by the caller)
            st.dy = _T(n, h, w, c, dev)
            # double buffered: the weight-gradient kernels of block j (side stream) read them while block j-1 is being processed
            st.dd = [_T(n, h, w, c, dev), _T(n, h, w, c, dev)]
            st.du = [_T(n, h, w, 4 * c, dev), _T(n, h, w, 4 * c, dev)]
            st.bias_acc = torch.zeros(4 * c, dtype=torch.float64, device=dev)
            st.colsum = torch.zeros(c, device=dev)
            st.gamma_scratch = torch.zeros(c, device=dev)
            st.raw = torch.zeros(c, 4 * c, device=dev)
            if i > 0:
                st.g_ds = _T(n, 2 * h, 2 * w, self.dims[i - 1], dev)  # gradient w.r.t. the downsample LayerNorm output
            ws_need += [L.yb200_conv2d_wgrad_workspace(st.blocks[0].hh.a, st.g[0].a, 1, 1) if st.blocks else 16,
                        L.yb200_conv2d_wgrad_workspace(st.blocks[0].y.a, st.du[0].a, 1, 1) if st.blocks else 16,
                        L.yb200_dwconv7_wgrad_workspace(st.x0.a), L.yb200_layernorm_bwd_workspace(st.x0.a), L.yb200_colsum_workspace(st.x0.a)]
            if i == 0:
                ws_need.append(L.yb200_conv2d_wgrad_workspace(self.patches.a, st.ds_conv.a, 1, 1))
            else:
                ws_need += [L.yb200_conv2d_wgrad_workspace(st.ds_ln.a, st.x0.a, 2, 2), L.yb200_layernorm_bwd_workspace(st.ds_ln.a)]
            self.stage.append(st)
            h, w = h // 2, w // 2
        assert min(ws_need) > 0, self.L.yb200_last_error()
        self.ws = torch.empty(max(ws_need), dtype=torch.uint8, device=dev)        # main stream
        self.ws_side = torch.empty(max(ws_need), dtype=torch.uint8, device=dev)   # weight-gradient stream
        self.overlap_wgrad = True
        self._side = torch.cuda.Stream(device=dev)
        self._fork = [[torch.cuda.Event() for _ in st.blocks] for st in self.stage]
        self._done = [[torch.cuda.Event() for _ in st.blocks] for st in self.stage]
        # packed bf16 weights
        d = self.dims
        bf = dict(dtype=torch.bfloat16, device=dev)
        self.packed["stem"] = torch.empty(d[0], 1, 48, **bf)
        for i in range(1, 4):
            self.packed[f"ds{i}"] = (torch.empty(d[i], 4, d[i - 1], **bf), torch.empty(d[i - 1], 4, d[i], **bf))
        for i in range(4):
            c = d[i]
            for j in range(self.depths[i]):
                self.packed[f"b{i}.{j}"] = (torch.empty(4 * c, 1, c, **bf), torch.empty(c, 1, 4 * c, **bf),   # pwconv1 fwd / dgrad
                                            torch.empty(c, 1, 4 * c, **bf), torch.empty(4 * c, 1, c, **bf),   # gamma*pwconv2 fwd / dgrad
                                            torch.empty(c, device=dev))                                        # gamma * b2

    def _count(self, k=1, label=None):
        self.kernel_launches += k
        if self.trace is not None:
            self.trace.append((label or "?", k))

    def _gamma(self, i, j):
        p = self.params.get(f"stages.{i}.{j}.gamma")
        return p if p is not None else self._ones[self.dims[i]]

    def pack_weights(self):
        L, sp, P, d = self.L, capi.stream_ptr(), self.params, self.dims
        capi.check(L.yb200_pack_conv_weight(capi.ptr(P["downsample_layers.0.0.weight"]), d[0], 48, 1, d[0], 48, capi.ptr(self.packed["stem"]), None, sp), "pack stem")
        for i in range(1, 4):
            wf, wd = self.packed[f"ds{i}"]
            capi.check(L.yb200_pack_conv_weight(capi.ptr(P[f"downsample_layers.{i}.1.weight"]), d[i], d[i - 1], 2, d[i], d[i - 1], capi.ptr(wf), capi.ptr(wd), sp),
                       "pack downsample")
        self._count(4, "pack stem+downsample")
        for i in range(4):
            c = d[i]
            for j in range(self.depths[i]):
                p = f"stages.{i}.{j}."
                w1f, w1d, w2f, w2d, sb = self.packed[f"b{i}.{j}"]
                capi.check(L.yb200_pack_conv_weight(capi.ptr(P[p + "pwconv1.weight"]), 4 * c, c, 1, 4 * c, c, capi.ptr(w1f), capi.ptr(w1d), sp), "pack pwconv1")
                capi.check(L.yb200_pack_conv_weight_scaled(capi.ptr(P[p + "pwconv2.weight"]), capi.ptr(self._gamma(i, j)), capi.ptr(P[p + "pwconv2.bias"]), c, 4 * c, 1,
                                                           c, 4 * c, capi.ptr(w2f), capi.ptr(w2d), capi.ptr(sb), sp), "pack pwconv2")
                self._count(3, "pack " + p)

    # ------------------------------------------------------------------ forward
    def forward_features(self, images=None):
        """images: uint8 or fp32 [N,3,H,W] on the device (default: self.images_u8).  Returns the NHWC bf16 feature tensors of out_indices."""
        L, sp, P = self.L, capi.stream_ptr(), self.params
        img = self.images_u8 if images is None else images
        assert img.is_cuda and img.is_contiguous() and img.shape == (self.n, 3, self.h, self.w) and img.dtype in (torch.uint8, torch.float32)
        eps = ctypes.c_float(LN_EPS)
        capi.check(L.yb200_patchify4(capi.ptr(img), int(img.dtype == torch.float32), self.n, self.h, self.w, self.patches.a, sp), "patchify4")
        self._count(1, "patchify")
        x = None
        for i, st in enumerate(self.stage[:self.n_stages]):
            if i == 0:
                capi.check(L.yb200_conv2d_affine_fwd(self.patches.a, capi.ptr(self.packed["stem"]), None, capi.ptr(P["downsample_layers.0.0.bias"]), None,
                                                     st.ds_conv.a, 1, 1, sp), "stem conv")
                capi.check(L.yb200_layernorm_fwd(st.ds_conv.a, capi.ptr(P["downsample_layers.0.1.weight"]), capi.ptr(P["downsample_layers.0.1.bias"]), eps, st.x0.a,
                                                 capi.ptr(st.ds_stats), sp), "stem norm")
            else:
                pre = f"downsample_layers.{i}."
                capi.check(L.yb200_layernorm_fwd(x.a, capi.ptr(P[pre + "0.weight"]), capi.ptr(P[pre + "0.bias"]), eps, st.ds_ln.a, capi.ptr(st.ds_stats), sp),
                           "downsample norm")
                capi.check(L.yb200_conv2d_affine_fwd(st.ds_ln.a, capi.ptr(self.packed[f"ds{i}"][0]), None, capi.ptr(P[pre + "1.bias"]), None, st.x0.a, 2, 2, sp),
                           "downsample conv")
            self._count(2, f"downsample {i}")
            x = st.x0
            for j, b in enumerate(st.blocks):
                p = f"stages.{i}.{j}."
                w1f, _, w2f, _, sb = self.packed[f"b{i}.{j}"]
                capi.check(L.yb200_dwconv7(x.a, capi.ptr(P[p + "dwconv.weight"]), capi.ptr(P[p + "dwconv.bias"]), None, b.d.a, 0, sp), "dwconv7")
                self._count(1, f"dwconv7 s{i}")
                capi.check(L.yb200_layernorm_fwd(b.d.a, capi.ptr(P[p + "norm.weight"]), capi.ptr(P[p + "norm.bias"]), eps, b.y.a, capi.ptr(b.stats), sp), "block norm")
                self._count(1, f"layernorm s{i}")
                capi.check(L.yb200_linear_gelu_fwd(b.y.a, capi.ptr(w1f), capi.ptr(P[p + "pwconv1.bias"]), b.u.a, b.hh.a, sp), "pwconv1+gelu")
                self._count(1, f"pwconv1+gelu s{i}")
                capi.check(L.yb200_conv2d_affine_fwd(b.hh.a, capi.ptr(w2f), None, capi.ptr(sb), x.a, b.out.a, 1, 1, sp), "pwconv2+scale+residual")
                self._count(1, f"pwconv2+res s{i}")
                x = b.out
            st.last = x
            if i in self.out_indices:
                capi.check(L.yb200_layernorm_fwd(x.a, capi.ptr(P[f"norm{i}.weight"]), capi.ptr(P[f"norm{i}.bias"]), eps, st.out.a, capi.ptr(st.out_stats), sp), "out norm")
                self._count(1, f"out norm {i}")
        return tuple(self.stage[i].out.t for i in self.out_indices)

    # ------------------------------------------------------------------ backward
    def _wgrad(self, x_a, dz_a, k, s, cin_real, dst, acc, label, ws=None):
        ws = self.ws if ws is None else ws
        capi.check(self.L.yb200_conv2d_wgrad(x_a, dz_a, k, s, cin_real, capi.ptr(dst), acc, capi.ptr(ws), ctypes.c_int64(ws.numel()), capi.stream_ptr()),
                   "wgrad " + label)
        self._count(2, "wgrad " + label)

    def _block_param_grads(self, i, j, st, b, gout, du, dd, xin, acc):
        """every parameter gradient of one block that needs a reduction over pixels; nothing downstream reads them, so they run on the side
        stream (own workspace) while the main stream continues with the data-gradient chain of the next block"""
        L, sp, P, G = self.L, capi.stream_ptr(), self.params, self.grads
        p, c = f"stages.{i}.{j}.", st.c
        ws = self.ws_side
        capi.check(L.yb200_colsum(gout.a, ctypes.c_float(1.0), capi.ptr(st.colsum), 0, capi.ptr(ws), sp), "colsum")
        self._count(2, f"colsum s{i}")
        self._wgrad(b.hh.a, gout.a, 1, 1, 4 * c, st.raw, 0, f"pwconv2 s{i}", ws)
        has_gamma = (p + "gamma") in G
        gg = G[p + "gamma"] if has_gamma else st.gamma_scratch
        capi.check(L.yb200_layer_scale_grad(capi.ptr(st.raw), capi.ptr(P[p + "pwconv2.weight"]), capi.ptr(P[p + "pwconv2.bias"]), capi.ptr(self._gamma(i, j)),
                                            capi.ptr(st.colsum), c, 4 * c, capi.ptr(G[p + "pwconv2.weight"]), capi.ptr(gg), capi.ptr(G[p + "pwconv2.bias"]),
                                            acc if has_gamma else 0, sp), "layer scale grad")
        self._count(1, "layer_scale_grad")
        self._wgrad(b.y.a, du.a, 1, 1, c, G[p + "pwconv1.weight"], acc, f"pwconv1 s{i}", ws)
        capi.check(L.yb200_dwconv7_wgrad(xin.a, dd.a, capi.ptr(G[p + "dwconv.weight"]), capi.ptr(G[p + "dwconv.bias"]), acc, capi.ptr(ws), sp), "dwconv7 wgrad")
        self._count(2, f"dwconv7 wgrad s{i}")

    def backward(self, accumulate=False):
        """gradients of sum_i <out_i, gout_i> w.r.t. every parameter; the caller has filled stage[i].gout.t for i in out_indices"""
        L, sp, P, G = self.L, capi.stream_ptr(), self.params, self.grads
        acc = 1 if accumulate else 0
        ws = capi.ptr(self.ws)
        carry = None  # gradient w.r.t. the last block output of the current stage coming from the next stage's downsample layer
        if not accumulate:
            for name in self.param_names:  # stages behind the last returned feature
                if any(name.startswith(f"stages.{i}.") or name.startswith(f"downsample_layers.{i}.") or name.startswith(f"norm{i}.") for i in range(self.n_stages, 4)):
                    G[name].zero_()
        for i in reversed(range(self.n_stages)):
            st = self.stage[i]
            g = st.g[0]
            cur = 0
            have = False
            if carry is not None:
                # carry was written into st.g[0] by the next stage's downsample backward
                have = True
            if i in self.out_indices:
                capi.check(L.yb200_layernorm_bwd(st.gout.a, st.last.a, capi.ptr(st.out_stats), capi.ptr(P[f"norm{i}.weight"]), g.a if have else None, g.a,
                                                 capi.ptr(G[f"norm{i}.weight"]), capi.ptr(G[f"norm{i}.bias"]), acc, ws, sp), "out norm bwd")
                self._count(2, f"out norm bwd {i}")
                have = True
            elif not accumulate:
                G[f"norm{i}.weight"].zero_()
                G[f"norm{i}.bias"].zero_()
            assert have, "no gradient reaches stage %d" % i
            c = st.c
            main = torch.cuda.current_stream()
            t, last_done = 0, None
            for j in reversed(range(len(st.blocks))):
                b = st.blocks[j]
                p = f"stages.{i}.{j}."
                xin = st.blocks[j - 1].out if j > 0 else st.x0
                _, w1d, _, w2d, _ = self.packed[f"b{i}.{j}"]
                gout, gin = st.g[cur], st.g[1 - cur]
                du, dd = st.du[t & 1], st.dd[t & 1]
                capi.check(L.yb200_linear_dgrad_gelu(gout.a, capi.ptr(w2d), b.u.a, du.a, capi.ptr(st.bias_acc), sp), "dgrad pwconv2 + gelu bwd")
                self._count(1, f"dgrad2+gelu' s{i}")
                capi.check(L.yb200_f64_to_f32(capi.ptr(st.bias_acc), 4 * c, capi.ptr(G[p + "pwconv1.bias"]), acc, 1, sp), "db1")
                self._count(1, "db1")
                capi.check(L.yb200_conv2d_dgrad(du.a, capi.ptr(w1d), st.dy.a, None, 1, 1, sp), "dgrad pwconv1")
                self._count(1, f"dgrad1 s{i}")
                capi.check(L.yb200_layernorm_bwd(st.dy.a, b.d.a, capi.ptr(b.stats), capi.ptr(P[p + "norm.weight"]), None, dd.a, capi.ptr(G[p + "norm.weight"]),
                                                 capi.ptr(G[p + "norm.bias"]), acc, ws, sp), "block norm bwd")
                self._count(2, f"layernorm bwd s{i}")
                if self.overlap_wgrad:
                    self._fork[i][j].record(main)
                    with torch.cuda.stream(self._side):
                        self._side.wait_event(self._fork[i][j])
                        self._block_param_grads(i, j, st, b, gout, du, dd, xin, acc)
                        self._done[i][j].record(self._side)
                    # the next kernel overwrites gin = the output-gradient buffer of the previous iteration, which that iteration's
                    # weight-gradient kernels read (this also protects du / dd of two iterations ago)
                    if last_done is not None:
                        main.wait_event(last_done)
                    last_done = self._done[i][j]
                else:
                    self._block_param_grads(i, j, st, b, gout, du, dd, xin, acc)
                capi.check(L.yb200_dwconv7(dd.a, capi.ptr(P[p + "dwconv.weight"]), None, gout.a, gin.a, 1, sp), "dwconv7 dgrad")
                self._count(1, f"dwconv7 dgrad s{i}")
                cur = 1 - cur
                t += 1
            if last_done is not None:
                main.wait_event(last_done)  # join before the downsample layer reuses the stage's buffers and the workspace
            g = st.g[cur]  # gradient w.r.t. the stage input x0
            if i == 0:
                pre = "downsample_layers.0."
                capi.check(L.yb200_layernorm_bwd(g.a, st.ds_conv.a, capi.ptr(st.ds_stats), capi.ptr(P[pre + "1.weight"]), None, st.dd[0].a, capi.ptr(G[pre + "1.weight"]),
                                                 capi.ptr(G[pre + "1.bias"]), acc, ws, sp), "stem norm bwd")
                capi.check(L.yb200_colsum(st.dd[0].a, ctypes.c_float(1.0), capi.ptr(G[pre + "0.bias"]), acc, ws, sp), "stem bias grad")
                self._count(4, "stem norm bwd + bias")
                self._wgrad(self.patches.a, st.dd[0].a, 1, 1, 48, G[pre + "0.weight"], acc, "stem")
            else:
                pre = f"downsample_layers.{i}."
                prev = self.stage[i - 1]
                capi.check(L.yb200_colsum(g.a, ctypes.c_float(1.0), capi.ptr(G[pre + "1.bias"]), acc, ws, sp), "downsample bias grad")
                self._wgrad(st.ds_ln.a, g.a, 2, 2, self.dims[i - 1], G[pre + "1.weight"], acc, f"downsample {i}")
                capi.check(L.yb200_conv2d_dgrad(g.a, capi.ptr(self.packed[f"ds{i}"][1]), st.g_ds.a, None, 2, 2, sp), "downsample dgrad")
                capi.check(L.yb200_layernorm_bwd(st.g_ds.a, prev.last.a, capi.ptr(st.ds_stats), capi.ptr(P[pre + "0.weight"]), None, prev.g[0].a,
                                                 capi.ptr(G[pre + "0.weight"]), capi.ptr(G[pre + "0.bias"]), acc, ws, sp), "downsample norm bwd")
                self._count(8, f"downsample {i} bwd")
                carry = prev.g[0]

    def train_step(self, accumulate=False):
        """forward + backward with the output gradients currently stored in stage[i].gout (benchmark / test driver)"""
        self.pack_weights()
        self.forward_features()
        self.backward(accumulate)


class _ConvNeXtFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, engine, x, *params):
        engine.pack_weights()
        outs = engine.forward_features(x.contiguous())
        ctx.engine = engine
        # the module boundary is the reference's: NCHW fp32 features
        return tuple(o.permute(0, 3, 1, 2).float() for o in outs)

    @staticmethod
    def backward(ctx, *gouts):
        eng = ctx.engine
        for i, g in zip(eng.out_indices, gouts):
            st = eng.stage[i]
            if g is None:
                st.gout.t.zero_()
            else:
                st.gout.t.copy_(g.permute(0, 2, 3, 1))
        eng.backward()
        return (None, None) + tuple(eng.grads[n].clone() for n in eng.param_names)


class ConvNeXt(nn.Module):
    """Drop-in for the reference `ConvNeXt(Backbone)` (convnext.py:62-180): same constructor arguments, parameter names and
    `forward(x) -> tuple of NCHW features`; `output_shape()` returns {index: ShapeSpec(channels)}.  drop_path_rate must be 0 for parity
    (stochastic depth is an RNG-driven training regulariser: SURVEY.md par.8a row C1) and is ignored otherwise."""

    def __init__(self, in_chans=3, depths=[3, 3, 9, 3], dims=[96, 192, 384, 768], drop_path_rate=0.0, layer_scale_init_value=1e-6, out_indices=[0, 1, 2, 3],
                 device="cuda"):
        super().__init__()
        if in_chans != 3:
            raise capi.Yb200Error("ConvNeXt stem kernel is specialised for 3 input channels")
        self.depths, self.dims, self.out_indices = list(depths), list(dims), list(out_indices)
        self.layer_scale_init_value = layer_scale_init_value
        self.device_ = torch.device(device)
        self._root = ConvNeXtEngine(1, 32, 32, depths, dims, layer_scale_init_value, out_indices, self.device_)
        self._root.init_weights(0)
        self._plans = {}
        for name in self._root.param_names:  # register the flat-buffer views under the reference's names
            mod = self
            *path, leaf = name.split(".")
            for part in path:
                if not hasattr(mod, part):
                    mod.add_module(part, nn.Module())
                mod = getattr(mod, part)
            mod.register_parameter(leaf, nn.Parameter(self._root.params[name]))
        from .modeling import ShapeSpec
        self.output_shape_dict = {i: ShapeSpec(channels=dims[i]) for i in range(4)}

    @property
    def engine(self):
        return self._root

    @property
    def size_divisibility(self):
        return 32

    def output_shape(self):
        return self.output_shape_dict

    def _plan(self, n, h, w):
        key = (n, h, w)
        if key not in self._plans:
            self._plans[key] = ConvNeXtEngine(n, h, w, self.depths, self.dims, self.layer_scale_init_value, self.out_indices, self.device_, share_params_of=self._root)
        return self._plans[key]

    def forward_features(self, x):
        if not x.is_cuda:
            raise capi.Yb200Error("ConvNeXt: input must be a CUDA tensor (no CPU path)")
        if x.dtype not in (torch.uint8, torch.float32):
            x = x.float()
        eng = self._plan(*[x.shape[0], x.shape[2], x.shape[3]])
        by_name = dict(self.named_parameters())
        return _ConvNeXtFn.apply(eng, x, *[by_name[n] for n in eng.param_names])

    def forward(self, x):
        return self.forward_features(x)


def build_convnext_backbone(cfg, input_shape=None):
    """convnext.py:209-230 (registered in BACKBONE_REGISTRY below): ConvNeXt-T, out_indices from cfg.MODEL.CONVNEXT.OUT_FEATURES"""
    n_out = len(cfg.MODEL.CONVNEXT.OUT_FEATURES)
    out_indices = [0, 1, 2] if n_out == 3 else [0, 1, 2, 3]
    return ConvNeXt(in_chans=3, depths=[3, 3, 9, 3], dims=[96, 192, 384, 768], drop_path_rate=0.2, layer_scale_init_value=1e-6, out_indices=out_indices)


def _register():
    from .modeling import BACKBONE_REGISTRY
    try:
        BACKBONE_REGISTRY.register(build_convnext_backbone)
    except Exception:  # already registered (module reloaded)
        pass


_register()
