"""Host runtime of the H100 detection path: a tiny static-graph builder whose
ops are launches of the C-ABI kernels (include/odt_b200.h) on torch-owned
device buffers.  PyTorch is plumbing only (allocation, streams, CUDA graphs).

A model file (nets.py) describes its layers once through `Builder`; the builder
  * names variables the way TF1 variable scopes do (SURVEY.md App. D) so the
    same weight dict drives this path and the CPU oracle,
  * pads fp16 activations to 64-channel multiples (TMA / wgmma K-chunk),
  * fuses what the reference expresses as separate TF ops into conv epilogues:
    bias / folded inference BN / ReLU / LeakyReLU / residual add / the
    consumer's pre-activation BN+ReLU (second output) / direct scatter of the
    head convolutions into the [B, N, Tail.row] candidate-row buffer.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import torch

from . import lib as L

BN_EPS = 1e-3   # tf.layers.batch_normalization default (SURVEY App. A.3)
GN_EPS = 1e-6   # tf.contrib.layers.group_norm default (App. A.5)
ACT = {None: L.ACT_NONE, "relu": L.ACT_RELU, "leaky": L.ACT_LEAKY}


def _round_up(x, m):
    return (x + m - 1) // m * m


def slice_store_width(cout, tensor_cores):
    """Channels per output pixel a convolution may store into an extra output (out1 / out2) from its first channel:
    the tensor-core kernels store whole 32-channel chunks up to Cout_pad (zero past Cout), the CUDA-core kernels
    exactly Cout.  Net.concat relies on it: a part must not reach the next part's channels."""
    return _round_up(cout, 32) if tensor_cores else cout


def same_pad(size, k, stride, dil=1):
    """TF SAME geometry (SURVEY App. A.1); host twin of odt_same_pad."""
    out = -(-size // stride)
    total = max((out - 1) * stride + (k - 1) * dil + 1 - size, 0)
    return out, total // 2, total - total // 2


class Namer:
    """TF1-style variable scopes: default layer names are uniquified per scope."""

    def __init__(self):
        self.stack, self.counts = [], {}

    def push(self, name):
        self.stack.append(name)

    def pop(self):
        self.stack.pop()

    def prefix(self):
        return "/".join(self.stack)

    def unique(self, base):
        key = (self.prefix(), base)
        k = self.counts.get(key, 0)
        self.counts[key] = k + 1
        name = base if k == 0 else "%s_%d" % (base, k)
        return (self.prefix() + "/" + name) if self.stack else name

    def named(self, name):
        return (self.prefix() + "/" + name) if self.stack else name

    def reset_under(self, prefix):
        self.counts = {k: v for k, v in self.counts.items() if not k[0].startswith(prefix)}


class Act:
    """An activation tensor [B,H,W,C] with channel stride ld."""

    def __init__(self, name, B, H, W, C, ld, dtype):
        self.name, self.B, self.H, self.W, self.C, self.ld, self.dtype = name, B, H, W, C, ld, dtype
        self.buf = None
        self.needed = True  # False when only a fused second output is consumed
        self.halo = 0       # 1: stored as [B, H+2, W+2, ld] with a zero border (halo-flat 3x3 convs)
        self.base, self.c0 = None, 0  # a channel slice [c0, c0 + C) of the tensor `base` (Net.concat)
        self.parts = ()               # Net.concat: the slices that make up this tensor
        self.chan_map = None          # Net.padded_concat: stored channel of every real channel (None: the identity)

    @property
    def real_channels(self):
        return self.C if self.chan_map is None else len(self.chan_map)

    @property
    def img_stride(self):
        return (self.H + 2 * self.halo) * (self.W + 2 * self.halo) * self.ld

    @property
    def pixels(self):
        return self.B * self.H * self.W

    def ptr(self):
        return self.buf.data_ptr() if self.buf is not None else None


class Op:
    reads = ()
    writes = ()

    def prepare(self, net):
        pass

    def launch(self, net, stream):
        raise NotImplementedError


class ConvOp(Op):
    def __init__(self, x, y, k, stride, dil, kernel, bias, bn, act, residual, head, is_image):
        self.x, self.y = x, y
        self.k, self.stride, self.dil = k, stride, dil
        self.kernel, self.bias, self.bn, self.act = kernel, bias, bn, act
        self.residual, self.head, self.is_image = residual, head, is_image
        self.pre = None     # fused consumer pre-activation: (bn_scope, act, Act)
        self.pre2 = None    # a second one (tensor-core path): RetinaNet block inputs feed two BNs
        self.pool = 0       # 2: the 2x2/2 max-pool that follows is done in the epilogue (y is the pooled tensor)
        # a concatenated input is read through its slices: their producers are what the op waits for
        self.reads = tuple(t for t in (x, residual) if t is not None) + (x.parts if x is not None else ())
        self.writes = (y,) if y is not None else ()
        self.flops = 0

    def on_tensor_cores(self, net):
        """odt_conv2d_f16_tc runs this layer (conv_tc and the kernels its planner picks); otherwise the CUDA-core
        direct convolution or the stem."""
        return net.precision == "fp16" and net.allow_tc and not self.is_image and self.x.ld % 64 == 0

    def slice_channels(self, net):
        """Channels of each output pixel this layer may store into an extra output (slice_store_width)."""
        return slice_store_width(self.y.C, self.on_tensor_cores(net))

    def host_weights(self, net):
        """HWIO kernel and bias of the convolution the kernels run.  The filter rows of an input stored with gaps
        between its parts (Net.padded_concat) are scattered to the stored channels, zero at the gaps."""
        kern = np.asarray(net.weights[self.kernel], dtype=np.float32)
        bias = (np.asarray(net.weights[self.bias], dtype=np.float32) if self.bias
                else np.zeros(kern.shape[3], np.float32))
        x = self.x
        if self.is_image and net.in_scale is not None:
            # a per-channel input scale folds exactly into the input-channel rows: SAME padding pads with zeros
            kern = (kern * np.asarray(net.in_scale, np.float32).reshape(1, 1, 3, 1)).astype(np.float32)
        if x is not None and x.chan_map is not None:
            full = np.zeros(kern.shape[:2] + (x.C, kern.shape[3]), np.float32)
            full[:, :, x.chan_map, :] = kern
            kern = full
        return kern, bias

    def host_bn(self, net):
        """(scale, shift) of the folded inference BN, per output channel of the convolution the kernels run."""
        return net.bn_fold(self.bn)

    def prepare(self, net):
        x = self.x
        dev = net.device
        kern, bias = self.host_weights(net)  # HWIO
        R, S, cin, cout = kern.shape
        assert cin == (3 if self.is_image else x.C), (self.kernel, cin, x.C)
        self.cout = cout
        f16 = net.precision == "fp16"
        adt = torch.float16 if f16 else torch.float32
        self.use_tc = self.on_tensor_cores(net)
        ohwi = np.transpose(kern, (3, 0, 1, 2))  # [Cout,R,S,Cin]
        if self.use_tc:
            cpad = _round_up(cout, 32)
            wp = np.zeros((cpad, R, S, x.ld), dtype=np.float32)
            wp[:cout, :, :, :cin] = ohwi
            self.w_ld, self.cout_pad = x.ld, cpad
        else:
            wp = np.ascontiguousarray(ohwi)
            self.w_ld, self.cout_pad = cin, cout
        self.wdev = torch.from_numpy(wp).to(dev).to(adt).contiguous()
        if self.bn:
            sc, sh = self.host_bn(net)
            shift = sh + bias * sc
            scale = sc
        else:
            scale, shift = None, bias
        self.scale = torch.from_numpy(scale).to(dev) if scale is not None else None
        self.shift = torch.from_numpy(np.ascontiguousarray(shift)).to(dev)
        H, Wd = (net.in_h, net.in_w) if self.is_image else (x.H, x.W)
        B = net.batch
        OH, pt, _ = same_pad(H, R, self.stride, self.dil)
        OW, pl, _ = same_pad(Wd, S, self.stride, self.dil)
        p = L.ConvParams()
        p.B, p.H, p.W, p.Cin = B, H, Wd, cin
        p.in_ld = 3 if self.is_image else x.ld
        p.OH, p.OW, p.Cout = OH, OW, cout
        p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = R, S, self.stride, self.dil, pt, pl
        p.w_ld, p.Cout_pad = self.w_ld, self.cout_pad
        p.scale = self.scale.data_ptr() if self.scale is not None else None
        p.shift = self.shift.data_ptr()
        p.act = ACT[self.act]
        p.residual = self.residual.ptr() if self.residual is not None else None
        p.in_halo = 0 if self.is_image else x.halo
        p.out0_halo = 0
        if self.head is not None:
            hb, row = net.head_buf, net.tail.row
            lvl_off, col, group, gstride, A = self.head
            p.out0 = hb.data_ptr() + 4 * (lvl_off * row + col)
            p.out0_dtype = L.ODT_F32
            p.out0_img_stride = net.N * row
            p.out0_pix_stride = A * row
            p.out0_group, p.out0_group_stride = group, gstride
        else:
            y = self.y
            if self.pool:
                assert (y.H, y.W, y.C) == (OH // 2, OW // 2, cout) and OH % 2 == 0 and OW % 2 == 0
            else:
                assert (y.H, y.W, y.C) == (OH, OW, cout)
            p.out0_pool = self.pool
            p.out0 = y.ptr() if y.needed else None
            p.out0_dtype = L.ODT_F16 if f16 else L.ODT_F32
            p.out0_img_stride = y.img_stride
            p.out0_pix_stride = y.ld
            p.out0_halo = y.halo
            assert self.residual is None or self.residual.halo == y.halo
            p.out0_group = p.out0_group_stride = 0
        if self.pre is not None:
            scope, act2, t = self.pre
            if scope is not None:
                s2, h2 = net.bn_fold(scope)
                self.scale2 = torch.from_numpy(s2).to(dev)
                self.shift2 = torch.from_numpy(h2).to(dev)
                p.scale2, p.shift2 = self.scale2.data_ptr(), self.shift2.data_ptr()
            p.act2 = ACT[act2]
            p.out1 = t.ptr()
            p.out1_img_stride = t.img_stride
            p.out1_pix_stride = t.ld
            p.out1_halo = t.halo
        if self.pre2 is not None:
            scope, act3, t = self.pre2
            if scope is not None:
                s3, h3 = net.bn_fold(scope)
                self.scale3 = torch.from_numpy(s3).to(dev)
                self.shift3 = torch.from_numpy(h3).to(dev)
                p.scale3, p.shift3 = self.scale3.data_ptr(), self.shift3.data_ptr()
            p.act3 = ACT[act3]
            p.out2 = t.ptr()
            p.out2_img_stride = t.img_stride
            p.out2_pix_stride = t.ld
            p.out2_halo = t.halo
        self.p = p
        self.flops = 2 * B * OH * OW * cout * R * S * cin
        # the 7x7 / stride-2 stem reads a packed fp16 RGBX copy of the image (mean subtracted, zero border of `rgbx`
        # pixels) so that every filter row is one aligned span -- see csrc/conv_stem_tc.cu
        self.rgbx = 0
        if (self.is_image and f16 and net.allow_tc and self.pre is None and self.head is None
                and (R, self.stride) == (7, 2) and cout <= 16 and Wd % 2 == 0 and pl % 2 == 0 and pl <= 4 and pt <= 4):
            self.rgbx = 4
        if self.rgbx == 4 and cout < 16:
            # the packed 7x7 stem computes 16 outputs (RetinaNet's basic variant has 7): filter rows, BN scale and
            # shift are zero past `cout`, so the pad lanes its whole-sector store writes stay zero
            wp = np.zeros((16,) + ohwi.shape[1:], np.float32)
            wp[:cout] = ohwi
            self.wdev = torch.from_numpy(wp).to(dev).to(adt).contiguous()
            sc16, sh16 = np.zeros(16, np.float32), np.zeros(16, np.float32)
            sc16[:cout] = 1.0 if scale is None else scale
            sh16[:cout] = shift
            self.scale, self.shift = torch.from_numpy(sc16).to(dev), torch.from_numpy(sh16).to(dev)
            p.scale, p.shift = self.scale.data_ptr(), self.shift.data_ptr()
            self.cout_pad = p.Cout_pad = 16
        if self.rgbx:
            P = self.rgbx
            net.image_rgbx = torch.zeros((B, H + 2 * P, Wd + 2 * P, 4), dtype=torch.float16, device=dev)

    def params(self, net):
        """The kernel parameter block; head convolutions have a second one that scatters into the candidate-row buffer of
        pipeline slot 1 (Net.capture_pipelined)."""
        return self.p1 if (net.slot == 1 and self.head is not None) else self.p

    def launch(self, net, stream):
        lib = net.lib
        if self.is_image and self.rgbx:
            P = self.rgbx
            L.check(lib.odt_pack_input_rgbx(net.image_buf.data_ptr(), net.image_rgbx.data_ptr(), net.batch,
                                            net.in_h, net.in_w, P, net.mean3, stream), "pack_input_rgbx")
            self.p.in_ld, self.p.in_halo = 4, P
            rc = lib.odt_conv2d_stem_rgbx(net.image_rgbx.data_ptr(), self.wdev.data_ptr(), C.byref(self.p), stream)
            if rc == L.ERR_UNSUPPORTED:  # shape outside the packed variants: the fp32-gather stem from now on
                self.rgbx = 0
                self.p.in_ld, self.p.in_halo = 3, 0
                return self.launch(net, stream)
        elif self.is_image:
            rc = lib.odt_conv2d_stem(net.image_buf.data_ptr(), net.mean3, self.wdev.data_ptr(),
                                     L.ODT_F16 if net.precision == "fp16" else L.ODT_F32,
                                     C.byref(self.p), stream)
        elif self.use_tc:
            rc = lib.odt_conv2d_f16_tc(self.x.ptr(), self.wdev.data_ptr(), C.byref(self.params(net)), stream)
        else:
            rc = lib.odt_conv2d_direct(self.x.ptr(), self.wdev.data_ptr(),
                                       L.ODT_F16 if net.precision == "fp16" else L.ODT_F32,
                                       C.byref(self.params(net)), stream)
        L.check(rc, "conv %s" % self.kernel)


class PoolOp(Op):
    def __init__(self, x, y, k, stride):
        self.x, self.y, self.k, self.stride = x, y, k, stride
        self.pre = None    # fused consumer pre-activations (bn_scope, act, Act): RetinaNet / FCOS pooled stem
        self.pre2 = None
        self.reads, self.writes = (x,), (y,)

    def prepare(self, net):
        self.aff = []
        for pr in (self.pre, self.pre2):
            if pr is None:
                self.aff.append(None)
                continue
            scope, act, t = pr
            sp = np.ones(self.x.ld, np.float32)
            hp = np.zeros(self.x.ld, np.float32)
            if scope is not None:
                sc, sh = net.bn_fold(scope)
                sp[:], hp[:] = 0.0, 0.0
                sp[:self.x.C], hp[:self.x.C] = sc, sh
            self.aff.append((torch.from_numpy(sp).to(net.device), torch.from_numpy(hp).to(net.device), ACT[act], t))

    def launch(self, net, stream):
        x = self.x
        # Only the 16-byte sectors that hold real channels are pooled: every activation owns a zero-initialised
        # buffer (Net.allocate), so the padding lanes of y that are never written stay zero, and the ones inside
        # the last sector are maxima of zeros.  (RetinaNet's 16-channel stem output is stored 64 wide.)
        c = min(x.ld, _round_up(x.C, 8))
        if self.pre is None and self.pre2 is None:
            L.check(net.lib.odt_maxpool(x.ptr(), self.y.ptr(), net.dt, x.B, x.H, x.W, c, x.ld,
                                        self.k, self.stride, x.halo, self.y.halo, stream), "maxpool")
            return
        a1, a2 = self.aff
        L.check(net.lib.odt_maxpool_affine(
            x.ptr(), self.y.ptr() if self.y.needed else None, net.dt, x.B, x.H, x.W, c, x.ld, self.k, self.stride,
            x.halo, self.y.halo,
            a1[0].data_ptr() if a1 else None, a1[1].data_ptr() if a1 else None, a1[2] if a1 else 0,
            a1[3].ptr() if a1 else None, a1[3].halo if a1 else 0,
            a2[0].data_ptr() if a2 else None, a2[1].data_ptr() if a2 else None, a2[2] if a2 else 0,
            a2[3].ptr() if a2 else None, a2[3].halo if a2 else 0, stream), "maxpool_affine")


class L2NormOp(Op):
    def __init__(self, x, y, var):
        self.x, self.y, self.var = x, y, var
        self.reads, self.writes = (x,) + x.parts, (y,)

    def prepare(self, net):
        self.gamma = float(np.asarray(net.weights[self.var], dtype=np.float32).reshape(-1)[0])

    def launch(self, net, stream):
        x = self.x
        L.check(net.lib.odt_l2norm_scale(x.ptr(), self.y.ptr(), net.dt, x.pixels, x.C, x.ld,
                                         self.gamma, stream), "l2norm")


class AffineActOp(Op):
    """Stand-alone inference BN (+activation): the pre-activation of RetinaNet's
    _bn_activation_conv when it cannot be fused into the producer."""

    def __init__(self, x, y, bn, act):
        self.x, self.y, self.bn, self.act = x, y, bn, act
        self.reads, self.writes = (x,), (y,)

    def prepare(self, net):
        s, h = net.bn_fold(self.bn)
        x = self.x
        sp = np.zeros(x.ld, np.float32)
        hp = np.zeros(x.ld, np.float32)
        sp[:x.C], hp[:x.C] = s, h
        self.scale = torch.from_numpy(sp).to(net.device)
        self.shift = torch.from_numpy(hp).to(net.device)

    def launch(self, net, stream):
        x = self.x
        L.check(net.lib.odt_affine_act(x.ptr(), self.y.ptr(), net.dt, x.pixels, x.ld, x.ld,
                                       self.scale.data_ptr(), self.shift.data_ptr(), ACT[self.act],
                                       stream), "affine_act")


class GroupNormActOp(Op):
    def __init__(self, x, y, gn, act, groups=8):
        self.x, self.y, self.gn, self.act, self.groups = x, y, gn, act, groups
        self.reads, self.writes = (x,), (y,)
        self.acc = None  # slice of the net's arena (zeroed once per forward): the two-launch path's workspace

    def prepare(self, net):
        dev = net.device
        self.gamma = torch.from_numpy(np.asarray(net.weights[self.gn + "/gamma"], np.float32)).to(dev)
        self.beta = torch.from_numpy(np.asarray(net.weights[self.gn + "/beta"], np.float32)).to(dev)
        self.stats = torch.zeros(self.x.B * self.groups * 6, dtype=torch.float32, device=dev)
        n = self.workspace_doubles(net)
        self.two_launch = n > 0
        if self.two_launch:
            self.acc = net.gn_take(n)

    def workspace_doubles(self, net):
        """fp64 words of odt_groupnorm_act's workspace for this op; 0 outside its two-launch path."""
        x = self.x
        nbytes = net.lib.odt_groupnorm_act_workspace_bytes(net.dt, x.B, x.H * x.W, x.C, self.groups)
        return (nbytes + 7) // 8

    def launch(self, net, stream):
        x = self.x
        hw = x.H * x.W
        if self.two_launch:
            rc = net.lib.odt_groupnorm_act(x.ptr(), self.y.ptr(), self.acc, net.dt, x.B, hw, x.C, x.ld,
                                           self.groups, GN_EPS, self.gamma.data_ptr(), self.beta.data_ptr(),
                                           ACT[self.act], stream)
            if rc == 0:
                return
            if rc != L.ERR_UNSUPPORTED:
                L.check(rc, "gn_act")
            self.two_launch = False  # shape outside the fused path: fall through to stats + apply
        L.check(net.lib.odt_groupnorm_stats(x.ptr(), self.stats.data_ptr(), net.dt, x.B, hw, x.C,
                                            x.ld, self.groups, GN_EPS, stream), "gn_stats")
        L.check(net.lib.odt_groupnorm_apply(x.ptr(), self.y.ptr(), self.stats.data_ptr(), net.dt,
                                            x.B, hw, x.C, x.ld, self.groups, self.gamma.data_ptr(),
                                            self.beta.data_ptr(), ACT[self.act], stream), "gn_apply")


class UpsampleAddOp(Op):
    def __init__(self, top, a, y):
        self.top, self.a, self.y = top, a, y
        self.pre = None
        self.reads, self.writes = (top, a), (y,)

    def prepare(self, net):
        self.s2 = self.h2 = None
        if self.pre is not None and self.pre[0] is not None:
            s, h = net.bn_fold(self.pre[0])
            sp = np.zeros(self.y.ld, np.float32)
            hp = np.zeros(self.y.ld, np.float32)
            sp[:self.y.C], hp[:self.y.C] = s, h
            self.s2 = torch.from_numpy(sp).to(net.device)
            self.h2 = torch.from_numpy(hp).to(net.device)

    def launch(self, net, stream):
        t, a, y = self.top, self.a, self.y
        out1 = self.pre[2].ptr() if self.pre is not None else None
        act2 = ACT[self.pre[1]] if self.pre is not None else 0
        L.check(net.lib.odt_upsample_bilinear_add(
            t.ptr(), a.ptr(), y.ptr(), net.dt, y.B, t.H, t.W, y.H, y.W, y.ld, y.ld,
            self.s2.data_ptr() if self.s2 is not None else None,
            self.h2.data_ptr() if self.h2 is not None else None, act2, out1, stream), "upsample_add")


class NearestConcatOp(Op):
    def __init__(self, a, b, y):
        self.a, self.b, self.y = a, b, y
        self.reads, self.writes = (a, b), (y,)

    def launch(self, net, stream):
        a, b, y = self.a, self.b, self.y
        L.check(net.lib.odt_upsample_nearest_concat(a.ptr(), b.ptr(), y.ptr(), net.dt, y.B, y.H, y.W,
                                                    a.C, a.ld, b.H, b.W, b.C, b.ld, y.ld, stream),
                "nearest_concat")


# a tap of TF's 4x4 / stride-2 SAME conv2d_transpose (pad_before = 1) seen from output phase p along one axis, as a
# 3x3 stencil row r on the low-resolution input (input index i + r - 1): output 2i + p takes input i + d through
# kernel tap k = p + 1 - 2d.  None: that stencil row has no tap in this phase
_DECONV_TAP = ((3, 1, None), (None, 2, 0))


class PhaseConvOp(ConvOp):
    """The 4x4 / stride-2 SAME conv2d_transpose (+ bias + BN) as one 3x3 stride-1 convolution with 4 * cout outputs:
    output channel p * cout + c is phase p = 2 * py + px of channel c (PixelShuffleOp places it).  Each phase uses 2x2
    of the 16 taps; the other stencil taps are zero."""

    def __init__(self, x, y, kernel, bias, bn, act=None):
        super().__init__(x, y, 3, 1, 1, kernel, bias, bn, act, None, None, False)

    def host_weights(self, net):
        k4 = np.asarray(net.weights[self.kernel], dtype=np.float32)  # [4, 4, cout, cin]
        cout, cin = k4.shape[2], k4.shape[3]
        kern = np.zeros((3, 3, cin, 4 * cout), np.float32)
        for py in range(2):
            for px in range(2):
                p = 2 * py + px
                for r in range(3):
                    for s in range(3):
                        ky, kx = _DECONV_TAP[py][r], _DECONV_TAP[px][s]
                        if ky is not None and kx is not None:
                            kern[r, s, :, p * cout:(p + 1) * cout] = k4[ky, kx].T
        bias = np.tile(np.asarray(net.weights[self.bias], dtype=np.float32), 4)
        return kern, bias

    def host_bn(self, net):
        sc, sh = net.bn_fold(self.bn)
        return np.tile(sc, 4), np.tile(sh, 4)


class PixelShuffleOp(Op):
    """Phases [B, h, w, 4C] of PhaseConvOp -> act(out [B, 2h, 2w, C] (+ residual))."""

    def __init__(self, x, y, residual, act):
        self.x, self.y, self.residual, self.act = x, y, residual, act
        self.reads = (x,) if residual is None else (x, residual)
        self.writes = (y,)

    def launch(self, net, stream):
        x, y, r = self.x, self.y, self.residual
        assert x.halo == 0 and y.halo == 0 and (r is None or r.halo == 0)
        L.check(net.lib.odt_pixel_shuffle2x(x.ptr(), y.ptr(), r.ptr() if r is not None else None, net.dt, x.B, x.H,
                                            x.W, y.C, x.ld, y.ld, r.ld if r is not None else 0, ACT[self.act],
                                            stream), "pixel_shuffle2x")


class ResizeOp(Op):
    """Align-corners bilinear resize; `out2`: a concat slice that takes a second copy (Net.padded_concat)."""

    def __init__(self, x, y):
        self.x, self.y, self.out2 = x, y, None
        self.reads, self.writes = (x,), (y,)

    def launch(self, net, stream):
        x, y, o2 = self.x, self.y, self.out2
        assert x.halo == 0 and y.halo == 0
        L.check(net.lib.odt_resize_bilinear_ac(x.ptr(), y.ptr() if y.needed else None,
                                               o2.ptr() if o2 is not None else None, net.dt, x.B, x.H, x.W, x.C,
                                               x.ld, y.H, y.W, y.ld, o2.ld if o2 is not None else 0, stream),
                "resize_bilinear_ac")


class AvgPoolOp(Op):
    def __init__(self, x, y):
        self.x, self.y = x, y
        self.reads, self.writes = (x,), (y,)

    def launch(self, net, stream):
        x, y = self.x, self.y
        assert x.halo == 0 and y.halo == 0
        L.check(net.lib.odt_avgpool2x2_same(x.ptr(), y.ptr(), net.dt, x.B, x.H, x.W, x.C, x.ld, y.ld, stream),
                "avgpool2x2_same")


class DlaJoinOp(Op):
    """CenterNet's DLA joins: a + b, or (pooled) 2x2 SAME max pool of a + 2x2 SAME average pool of b."""

    def __init__(self, a, b, y, pooled):
        self.a, self.b, self.y, self.pooled = a, b, y, pooled
        self.reads, self.writes = (a, b), (y,)

    def launch(self, net, stream):
        a, b, y = self.a, self.b, self.y
        assert a.halo == 0 and b.halo == 0 and y.halo == 0
        L.check(net.lib.odt_dla_join(a.ptr(), b.ptr(), y.ptr(), net.dt, a.B, a.H, a.W, a.C, a.ld, b.ld, y.ld,
                                     int(self.pooled), stream), "dla_join")


class Net:
    """A built network: buffers + op list + the decode/NMS tail."""

    spec_only = False  # class-level switch: describe the graph without touching CUDA

    def __init__(self, batch, in_h, in_w, precision="fp16", device="cuda", allow_tc=True):
        assert precision in ("fp16", "fp32")
        self.lib = None if Net.spec_only else L.load()
        self.batch, self.in_h, self.in_w = batch, in_h, in_w
        self.precision, self.device, self.allow_tc = precision, torch.device(device), allow_tc
        self.dt = L.ODT_F16 if precision == "fp16" else L.ODT_F32
        self.tdtype = torch.float16 if precision == "fp16" else torch.float32
        self.namer = Namer()
        self.vars = {}      # name -> (shape, init kind), creation order
        self.ops = []
        self.acts = []
        self.levels = []    # (H, W, A) per head level, in candidate order
        self.tail = None
        self.mean3 = (C.c_float * 3)(123.68, 116.779, 103.979)  # ref SSD300.py:55
        self.in_scale = None  # per-channel multiplier of the mean-subtracted image, folded into the stem's kernel
        # ODT_HALO=0 keeps every tensor dense: the end-to-end reference the halo layouts are tested against
        self.use_halo = os.environ.get("ODT_HALO", "1") != "0"
        self.weights = None
        self.graph = None
        self.slot = 0            # pipeline slot the launches address (capture_pipelined)
        self.body_graphs = None

    # ---------------------------------------------------------- variables ---
    def var(self, name, shape, kind):
        if name not in self.vars:
            self.vars[name] = (tuple(int(s) for s in shape), kind)
        return name

    def bn_fold(self, scope):
        W = self.weights
        g = np.asarray(W[scope + "/gamma"], np.float32)
        b = np.asarray(W[scope + "/beta"], np.float32)
        m = np.asarray(W[scope + "/moving_mean"], np.float32)
        v = np.asarray(W[scope + "/moving_variance"], np.float32)
        sc = (g / np.sqrt(v + np.float32(BN_EPS))).astype(np.float32)
        return sc, (b - m * sc).astype(np.float32)

    # -------------------------------------------------------------- build ---
    def new_act(self, name, H, W, Cc):
        ld = _round_up(Cc, 64) if self.precision == "fp16" else Cc
        t = Act(name, self.batch, H, W, Cc, ld, self.precision)
        self.acts.append(t)
        return t

    def scope(self, name):
        net = self

        class _S:
            def __enter__(self_):
                net.namer.push(name)

            def __exit__(self_, *a):
                net.namer.pop()

        return _S()

    def conv(self, x, cout, k, stride=1, dil=1, name=None, kernel_var=None, bias_var=None,
             bn=False, act=None, residual=None, head=None, bias_init="zeros", bn_scope=None):
        """tf.layers.conv2d (+ BN + activation + residual).  x=None means the image.  bn_scope: the BN variables'
        scope when they were named ahead of this call (TF order differs from op order)."""
        is_image = x is None
        cin = 3 if is_image else x.real_channels
        if kernel_var is None:
            vs = self.namer.named(name) if name else self.namer.unique("conv2d")
            kernel_var, bias_var = vs + "/kernel", vs + "/bias"
        self.var(kernel_var, (k, k, cin, cout), "he")
        if bias_var:
            self.var(bias_var, (cout,), bias_init)
        if bn and bn_scope is None:
            bn_scope = self.bn_vars(cout)
        H, W = (self.in_h, self.in_w) if is_image else (x.H, x.W)
        OH, _, _ = same_pad(H, k, stride, dil)
        OW, _, _ = same_pad(W, k, stride, dil)
        y = None if head is not None else self.new_act(kernel_var, OH, OW, cout)
        op = ConvOp(x, y, k, stride, dil, kernel_var, bias_var, bn_scope, act, residual, head,
                    is_image)
        op.out_hw = (OH, OW)
        self.ops.append(op)
        return y if head is None else op

    def bn_vars(self, c):
        scope = self.namer.unique("batch_normalization")
        self.var(scope + "/gamma", (c,), "bn_gamma")
        self.var(scope + "/beta", (c,), "bn_beta")
        self.var(scope + "/moving_mean", (c,), "bn_mean")
        self.var(scope + "/moving_variance", (c,), "bn_var")
        return scope

    def preact_bn(self, x, act="relu"):
        """inference BN -> activation as its own tensor (fused into the producer later)."""
        scope = self.bn_vars(x.C)
        y = self.new_act(scope + "/out", x.H, x.W, x.C)
        self.ops.append(AffineActOp(x, y, scope, act))
        return y

    def preact_gn(self, x, act="relu"):
        scope = self.namer.unique("GroupNorm")
        self.var(scope + "/beta", (x.C,), "gn_beta")
        self.var(scope + "/gamma", (x.C,), "gn_gamma")
        y = self.new_act(scope + "/out", x.H, x.W, x.C)
        self.ops.append(GroupNormActOp(x, y, scope, act))
        return y

    def maxpool(self, x, k, stride):
        OH, _, _ = same_pad(x.H, k, stride)
        OW, _, _ = same_pad(x.W, k, stride)
        y = self.new_act(x.name + "/pool", OH, OW, x.C)
        self.ops.append(PoolOp(x, y, k, stride))
        return y

    def l2norm(self, x, var, init=20.0):
        """x * rsqrt(sum_c x^2) * factor, with the scalar variable `var` initialised to `init`."""
        self.var(var, (1,), "l2norm" if init == 20.0 else "l2norm_%g" % init)
        y = self.new_act(var + "/out", x.H, x.W, x.C)
        y.chan_map = x.chan_map  # zero gap channels stay zero
        self.ops.append(L2NormOp(x, y, var))
        return y

    def upsample_add(self, top, a):
        y = self.new_act(a.name + "/topdown", a.H, a.W, a.C)
        self.ops.append(UpsampleAddOp(top, a, y))
        return y

    def nearest_concat(self, a, b):
        y = self.new_act(a.name + "/concat", a.H, a.W, a.C + b.C)
        self.ops.append(NearestConcatOp(a, b, y))
        return y

    def concat(self, parts):
        """tf.concat(parts, axis=channels) with no copy (YOLOv2.py:90): one tensor whose channel slices are stored by the
        producers of the parts, each as an extra epilogue output of its convolution (an identity pre-activation that
        fuse() folds in).  A part whose producer cannot take it is an error at finalize, not a copy."""
        y = self.new_act(parts[0].name + "/concat", parts[0].H, parts[0].W, sum(t.C for t in parts))
        c0, views = 0, []
        for t in parts:
            assert (t.B, t.H, t.W) == (y.B, y.H, y.W), (t.name, y.name)
            v = Act(t.name + "/slice", t.B, t.H, t.W, t.C, y.ld, t.dtype)
            v.base, v.c0 = y, c0
            self.acts.append(v)
            self.ops.append(AffineActOp(t, v, None, None))
            views.append(v)
            c0 += t.C
        y.parts = tuple(views)
        return y

    def padded_concat(self, parts):
        """tf.concat(parts, axis=channels) of parts whose widths are not multiples of 32 (PFPNet-R's 85-channel parts,
        PFPNetR.py:364-395), with no copy: each part is stored at a 32-aligned channel offset of one buffer, the channels
        between a part's end and the next offset stay zero, so a tensor-core producer's whole-chunk store stays inside
        its slice.  `chan_map` of the result lists the stored channel of every real channel, and its consumers scatter
        their filter rows to those channels (ConvOp.host_weights).  A part comes from a convolution (an extra
        epilogue output, as in `concat`) or from `resize_ac` (its second output)."""
        offs, c0 = [], 0
        for t in parts:
            assert (t.B, t.H, t.W) == (parts[0].B, parts[0].H, parts[0].W), (t.name, parts[0].name)
            offs.append(c0)
            c0 += _round_up(t.C, 32)
        y = self.new_act(parts[0].name + "/concat", parts[0].H, parts[0].W, c0)
        y.chan_map = np.concatenate([np.arange(o, o + t.C) for o, t in zip(offs, parts)])
        views = []
        for t, o in zip(parts, offs):
            v = Act(t.name + "/slice", t.B, t.H, t.W, t.C, y.ld, t.dtype)
            v.base, v.c0 = y, o
            self.acts.append(v)
            rs = next((op for op in self.ops if isinstance(op, ResizeOp) and op.y is t), None)
            if rs is not None:
                assert rs.out2 is None, t.name
                rs.out2, rs.writes = v, (t, v)
            else:
                self.ops.append(AffineActOp(t, v, None, None))
            views.append(v)
        y.parts = tuple(views)
        return y

    def deconv(self, x, cout, residual=None, act=None):
        """tf.layers.conv2d_transpose(cout, 4, 2, 'same') -> BN (PFPNetR.py:696-709), then `+ residual` and `act`:
        one 3x3 stride-1 convolution of 4 * cout phase-major outputs on the low-resolution grid (PhaseConvOp) and their
        placement on the 2x grid (PixelShuffleOp)."""
        return self.shuffle(self.deconv_phases(x, cout), residual, act)

    def deconv_phases(self, x, cout, act=None):
        """tf.layers.conv2d_transpose(cout, 4, 2, 'same') -> BN (-> act) as the four phases on the low-resolution grid,
        `act` in the phase convolution's epilogue (CenterNet.py:349-361: the ReLU comes before its sums); `shuffle`
        places them."""
        vs = self.namer.unique("conv2d_transpose")
        kernel_var, bias_var = vs + "/kernel", vs + "/bias"
        self.var(kernel_var, (4, 4, cout, x.real_channels), "he")
        self.var(bias_var, (cout,), "zeros")
        bn_scope = self.bn_vars(cout)
        ph = self.new_act(kernel_var + "/phases", x.H, x.W, 4 * cout)
        op = PhaseConvOp(x, ph, kernel_var, bias_var, bn_scope, act)
        op.out_hw = (x.H, x.W)
        self.ops.append(op)
        return ph

    def shuffle(self, ph, residual=None, act=None):
        """act(the phases of `deconv_phases` on the 2x grid (+ residual))."""
        y = self.new_act(ph.name + "/out%d" % len(self.ops), 2 * ph.H, 2 * ph.W, ph.C // 4)
        if residual is not None:
            assert (residual.H, residual.W, residual.C) == (y.H, y.W, y.C), (residual.name, y.name)
        self.ops.append(PixelShuffleOp(ph, y, residual, act))
        return y

    def dla_join(self, a, b, pooled):
        """a + b, or (pooled) max_pool(a, 2, 2, SAME) + average_pool(b, 2, 2, SAME) (CenterNet.py:93-110)."""
        assert (a.H, a.W, a.C) == (b.H, b.W, b.C), (a.name, b.name)
        H, W = ((a.H + 1) // 2, (a.W + 1) // 2) if pooled else (a.H, a.W)
        y = self.new_act(a.name + ("/join_pooled" if pooled else "/join"), H, W, a.C)
        self.ops.append(DlaJoinOp(a, b, y, pooled))
        return y

    def resize_ac(self, x, OH, OW):
        """tf.image.resize_bilinear(x, [OH, OW], align_corners=True) (PFPNetR.py:324-326)."""
        y = self.new_act(x.name + "/resize%dx%d" % (OH, OW), OH, OW, x.C)
        self.ops.append(ResizeOp(x, y))
        return y

    def avgpool(self, x):
        """tf.layers.average_pooling2d(x, 2, 2, 'same') (PFPNetR.py:721-728)."""
        y = self.new_act(x.name + "/avgpool", (x.H + 1) // 2, (x.W + 1) // 2, x.C)
        self.ops.append(AvgPoolOp(x, y))
        return y

    def add_level(self, H, W, A):
        off = sum(h * w * a for h, w, a in self.levels)
        self.levels.append((H, W, A))
        return off

    # ------------------------------------------------------------- fusion ---
    def fuse(self):
        """Fold stand-alone BN+ReLU pre-activations into the epilogue of the op
        that produces their input; drop raw outputs nobody else reads."""
        consumers = {}
        for op in self.ops:
            for t in op.reads:
                consumers.setdefault(id(t), []).append(op)
        producer = {}
        for op in self.ops:
            for t in op.writes:
                producer[id(t)] = op
        kept = []
        for op in self.ops:
            if isinstance(op, AffineActOp):
                q = producer.get(id(op.x))
                if op.y.base is not None:
                    self._check_slice_producer(q, op.y)
                ok = isinstance(q, (ConvOp, UpsampleAddOp, PoolOp)) and q.pre is None
                if ok and isinstance(q, ConvOp):
                    ok = q.head is None
                # second pre-activation of the same tensor: tensor-core convs (third epilogue output) and pools
                second = (not ok and isinstance(q, ConvOp) and q.head is None and q.pre is not None
                          and q.pre2 is None and q.on_tensor_cores(self))
                second = second or (not ok and isinstance(q, PoolOp) and q.pre is not None and q.pre2 is None)
                if ok or second:
                    if ok:
                        q.pre = (op.bn, op.act, op.y)
                    else:
                        q.pre2 = (op.bn, op.act, op.y)
                    producer[id(op.y)] = q
                    consumers[id(op.x)].remove(op)
                    if not consumers[id(op.x)] and isinstance(q, (ConvOp, PoolOp)):
                        op.x.needed = False
                    continue
            if isinstance(op, AffineActOp) and op.y.base is not None:
                raise ValueError("concat: the producer of %s cannot store its channel slice" % op.x.name)
            kept.append(op)
        self.ops = kept

    def _check_slice_producer(self, q, v):
        """A concat part `v` is stored by its producer `q` as an extra epilogue output at the concat's pixel stride.
        Only the convolution kernels take that stride (the pooling and upsampling kernels address their extra output
        with their own), and a producer that stores whole chunks of channels must not reach the next part's first
        channels, or past the concat's row for the last part."""
        if not isinstance(q, ConvOp) or q.head is not None:
            raise ValueError("concat: the producer of %s cannot store its channel slice (%s)"
                             % (v.name, type(q).__name__ if q is not None else "no producer"))
        parts = v.base.parts
        i = next(j for j, t in enumerate(parts) if t is v)
        end = parts[i + 1].c0 if i + 1 < len(parts) else v.base.ld
        stored = q.slice_channels(self)
        if v.c0 + stored > end:
            raise ValueError("concat: the producer of %s cannot store its channel slice (%d channels per pixel from "
                             "channel %d reach past channel %d)" % (v.name, stored, v.c0, end))

    # -------------------------------------------------------------- halos ----
    STEM_TC_VARIANTS = {(3, 1, 64), (3, 1, 32), (7, 2, 16)}

    def assign_halos(self):
        """Give a zero 1-pixel halo to fp16 tensors that feed a flat-eligible 3x3 conv
        (stride 1, dilation 1, padded Cout <= 128) when every producer / consumer of the
        tensor understands the layout (tensor-core convs, the tensor-core stems, max-pool)."""
        if self.precision != "fp16" or not self.allow_tc:
            return
        readers, producer = {}, {}
        for op in self.ops:
            for t in op.reads:
                readers.setdefault(id(t), []).append(op)
            for t in op.writes:
                producer[id(t)] = op
            for pr in (getattr(op, "pre", None), getattr(op, "pre2", None)):
                if pr is not None:
                    # fused second / third outputs: the tensor-core convolutions (conv_tc / conv_tapn / conv_thin
                    # epilogues) and the fused pool write them in the halo layout too; other producers stay dense
                    can = ((isinstance(op, ConvOp) and not op.is_image and op.head is None and op.x.ld % 64 == 0)
                           or isinstance(op, PoolOp))
                    producer[id(pr[2])] = "fused" if can else None
        for t in self.acts:
            prod = producer.get(id(t))
            cons = readers.get(id(t), [])
            if not cons or not t.needed:
                continue
            if prod == "fused":
                pass
            elif isinstance(prod, ConvOp):
                if prod.head is not None or prod.residual is not None:
                    continue
                if prod.is_image and (prod.k, prod.stride, t.C) not in self.STEM_TC_VARIANTS:
                    continue
                if prod.is_image and prod.pre is not None:
                    continue
            elif not isinstance(prod, PoolOp):
                continue
            ok, gain = True, False
            for c in cons:
                if isinstance(c, ConvOp) and c.x is t and c.residual is not t and not c.is_image:
                    cout = self.vars[c.kernel][0][3]
                    if (c.k == 3 and c.stride == 1 and c.dil == 1 and _round_up(cout, 32) <= 128
                            and t.H >= 16 and t.W >= 16):
                        gain = True  # small maps: the halo positions would dominate
                elif isinstance(c, PoolOp):
                    pass
                else:
                    ok = False
            if ok and gain and self.batch * (t.H + 2) * (t.W + 2) < (1 << 31) - 4096:
                t.halo = 1

    def fuse_pools(self):
        """Fold a 2x2/2 max-pool into the epilogue of the halo-flat 3x3 conv that feeds it
        (a4: SSD300.py:539-547 after conv1_2 / conv2_2): the unpooled tensor is never stored."""
        if self.precision != "fp16" or not self.allow_tc:
            return
        readers, producer = {}, {}
        for op in self.ops:
            for t in op.reads:
                readers.setdefault(id(t), []).append(op)
            for t in op.writes:
                producer[id(t)] = op
        kept = []
        for op in self.ops:
            if isinstance(op, PoolOp) and op.k == 2 and op.stride == 2:
                q, t = producer.get(id(op.x)), op.x
                ok = (isinstance(q, ConvOp) and q.y is t and readers.get(id(t)) == [op] and q.pre is None
                      and q.pre2 is None
                      and q.head is None and q.residual is None and not q.is_image and q.pool == 0
                      and q.x.halo == 1 and q.x.ld % 64 == 0 and q.k == 3 and q.stride == 1 and q.dil == 1
                      and _round_up(t.C, 32) <= 128 and t.H % 2 == 0 and t.W % 2 == 0)
                if ok:
                    q.pool, q.y, q.writes = 2, op.y, (op.y,)
                    producer[id(op.y)] = q
                    t.needed, t.fused_away = False, True
                    continue
            kept.append(op)
        self.ops = kept

    # ------------------------------------------------------------ finalize --
    def finalize(self, weights, tail, fuse=True):
        """Allocate buffers, upload weights, build the kernel parameter blocks."""
        self.weights = weights
        missing = [k for k in self.vars if k not in weights]
        if missing:
            raise KeyError("weights missing %d variables, e.g. %s" % (len(missing), missing[:3]))
        if fuse:
            self.fuse()
        if self.use_halo:
            self.assign_halos()
            self.fuse_pools()
        dev = self.device
        self.image_buf = torch.zeros((self.batch, self.in_h, self.in_w, 3), dtype=torch.float32,
                                     device=dev)
        for t in self.acts:
            if getattr(t, "fused_away", False):
                continue  # the pre-pool tensor of a conv with a fused max-pool is never materialised
            if not t.needed or t.base is not None:
                continue  # raw output nobody reads (only its fused pre-activations are consumed); slices below
            t.buf = torch.zeros((t.B, t.H + 2 * t.halo, t.W + 2 * t.halo, t.ld), dtype=self.tdtype, device=dev)
        for t in self.acts:
            if t.base is not None:
                assert t.halo == 0 and t.base.halo == 0
                t.buf = t.base.buf[..., t.c0:t.c0 + t.C]
        self.N = sum(h * w * a for h, w, a in self.levels)
        # candidate rows of a detection tail (a classification tail has no head levels and no rows)
        self.head_buf = torch.zeros((self.batch, self.N, getattr(tail, "row", 0)), dtype=torch.float32, device=dev)
        self.tail = tail
        tail.prepare(self)
        # one fp64 arena for the workspaces of every GroupNorm (per-slice moments, statistics, arrival counters),
        # zeroed once per forward
        n_gn = sum(op.workspace_doubles(self) for op in self.ops if isinstance(op, GroupNormActOp))
        self.gn_arena = torch.zeros(n_gn, dtype=torch.float64, device=dev) if n_gn > 0 else None
        self._gn_used = 0
        for op in self.ops:
            op.prepare(self)
        self.conv_flops = sum(getattr(op, "flops", 0) for op in self.ops)
        return self

    # ---------------------------------------------------------------- run ---
    def gn_take(self, n):
        ptr = self.gn_arena.data_ptr() + 8 * self._gn_used
        self._gn_used += n
        assert self._gn_used <= self.gn_arena.numel()
        return ptr

    def forward(self, stream=None, with_tail=True):
        """Launch backbone + heads (+ tail) on the current torch stream."""
        st = torch.cuda.current_stream().cuda_stream if stream is None else stream
        if self.gn_arena is not None:
            assert stream is None, "the GroupNorm arena is zeroed on the current torch stream"
            self.gn_arena.zero_()
        for op in self.ops:
            op.launch(self, st)
        if with_tail:
            self.tail.launch(self, st)

    # Independent branches of the op list (FPN levels, the two towers, SSD/YOLO heads
    # next to the rest of the backbone) are captured on separate stream lanes so that
    # launches with fewer CTAs than SMs overlap inside the graph.
    def plan_lanes(self, max_lanes=12):
        """Dataflow -> (lane of every op, cross-lane waits).  Pure host logic."""
        producer, deps = {}, []
        for i, op in enumerate(self.ops):
            deps.append(sorted({producer[id(t)] for t in op.reads if id(t) in producer}))
            outs = list(op.writes)
            for pr in (getattr(op, "pre", None), getattr(op, "pre2", None)):
                if pr is not None:
                    outs.append(pr[2])
            for t in outs:
                producer[id(t)] = i
        lane_of, tails, waits = [], [], []   # tails[l] = index of the last op put on lane l
        for i, d in enumerate(deps):
            lane = None
            for p in reversed(d):             # continue the lane of a producer that is still its tail
                if tails[lane_of[p]] == p:
                    lane = lane_of[p]
                    break
            if lane is None:
                if not tails or not d:        # roots stay on the capturing stream
                    lane = 0
                    if not tails:
                        tails.append(-1)
                elif len(tails) < max(1, max_lanes):
                    lane = len(tails)
                    tails.append(-1)
                else:                         # reuse the lane that has been idle longest
                    lane = min(range(len(tails)), key=lambda l: tails[l])
            waits.append([p for p in d if lane_of[p] != lane])
            lane_of.append(lane)
            tails[lane] = i
        return lane_of, waits, tails

    def forward_lanes(self, with_tail=True):
        """Multi-lane launch of the op list (used under graph capture); with_tail=False: backbone + heads only."""
        lane_of, waits, tails = self.plan_lanes()
        main = torch.cuda.current_stream()
        if len(tails) <= 1:
            return self.forward(with_tail=with_tail)
        if self.gn_arena is not None:
            self.gn_arena.zero_()  # on the capturing stream, ahead of every lane
        if getattr(self, "_lanes", None) is None or len(self._lanes) < len(tails):
            self._lanes = [None] + [torch.cuda.Stream(device=self.device) for _ in range(len(tails) - 1)]
        streams = [main] + self._lanes[1:len(tails)]
        need_event = {p for w in waits for p in w} | {t for l, t in enumerate(tails) if l != 0 and t >= 0}
        events = {}
        for i, op in enumerate(self.ops):
            st = streams[lane_of[i]]
            for p in waits[i]:
                st.wait_event(events[p])
            op.launch(self, st.cuda_stream)
            if i in need_event:
                ev = torch.cuda.Event()
                ev.record(st)
                events[i] = ev
        for l, t in enumerate(tails):         # join every lane back before the tail
            if l != 0 and t >= 0:
                main.wait_event(events[t])
        if with_tail:
            self.tail.launch(self, main.cuda_stream)

    def capture(self):
        """Capture the whole forward in a CUDA graph (launch-bound tail + 30-130 convs)."""
        import gc
        self.forward()  # warm-up outside capture (lazy attribute sets, driver entry points)
        # Garbage of earlier engines (CUDA graphs, streams, events) must not be finalised while the capture is
        # open: destroying a graph exec during a capture invalidates it (cudaErrorStreamCaptureInvalidated, seen once
        # when a collection happened to fire on the first launch).  Collect now, keep the collector off inside.
        gc.collect()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        gc_was_on = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                self.forward_lanes()
        finally:
            if gc_was_on:
                gc.enable()
        self.graph = g
        return g

    def run(self):
        if self.graph is not None:
            self.graph.replay()
        else:
            self.forward()

    # ---- two-stage pipeline over a stream of batches -----------------------------------------------------------
    # decode + NMS of batch i (latency-bound, 0.1-0.2 ms) run on a second, high-priority stream under the stem and the
    # first convolutions of batch i+1.  Everything the tail touches exists twice (candidate rows, candidate lists,
    # packed records: pipeline slots 0 / 1), the backbone's activations once (consecutive bodies are stream-ordered).
    def capture_pipelined(self):
        """Capture [body graph, tail graph] per pipeline slot (idempotent)."""
        import copy
        import gc
        if self.body_graphs is not None:
            return
        self.head_buf1 = torch.zeros_like(self.head_buf)
        t1 = copy.copy(self.tail)
        t1.prepare(self, head_buf=self.head_buf1)
        # slot 1 decodes and selects with slot 0's parameter block as it stands, not as the config built it: a score
        # threshold set on `tail.p` after the build (bench.py's dense-threshold RetinaNet) holds for every batch
        C.memmove(C.byref(t1.p), C.byref(self.tail.p), C.sizeof(t1.p))
        self.tails = [self.tail, t1]
        delta = self.head_buf1.data_ptr() - self.head_buf.data_ptr()
        for op in self.ops:
            if isinstance(op, ConvOp) and op.head is not None:
                p1 = L.ConvParams()
                C.memmove(C.byref(p1), C.byref(op.p), C.sizeof(p1))
                p1.out0 = op.p.out0 + delta
                op.p1 = p1
        body, tails = [], []
        gc_was_on = gc.isenabled()
        try:
            for s in (0, 1):
                self.slot = s
                self.forward(with_tail=False)  # warm-up of this slot's launches outside capture
                self.tails[s].launch(self, torch.cuda.current_stream().cuda_stream)
                gc.collect()
                torch.cuda.synchronize()
                gc.disable()
                gb, gt = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                with torch.cuda.graph(gb, capture_error_mode="thread_local"):
                    self.forward_lanes(with_tail=False)
                with torch.cuda.graph(gt, capture_error_mode="thread_local"):
                    self.tails[s].launch(self, torch.cuda.current_stream().cuda_stream)
                if gc_was_on:
                    gc.enable()
                body.append(gb)
                tails.append(gt)
        finally:
            self.slot = 0
            if gc_was_on:
                gc.enable()
        self._tail_stream = torch.cuda.Stream(device=self.device, priority=-1)
        self._body_done = [torch.cuda.Event() for _ in range(2)]
        self._tail_done = [torch.cuda.Event() for _ in range(2)]
        for ev in self._tail_done:
            ev.record(torch.cuda.current_stream())
        self.body_graphs, self.tail_graphs = body, tails

    def run_pipelined(self, slot, after_tail=None):
        """One step on pipeline slot `slot` (alternate 0 / 1 from batch to batch): the body on the current stream, the
        tail (+ `after_tail(tail)`: gather / read-back of its records) on the tail stream.  Returns the slot's Tail; its
        buffers are valid once `_tail_done[slot]` has fired (sync_pipelined waits for both)."""
        main = torch.cuda.current_stream()
        ts = self._tail_stream
        main.wait_event(self._tail_done[slot])  # this slot's rows / records of two batches ago have been consumed
        self.body_graphs[slot].replay()
        self._body_done[slot].record(main)
        ts.wait_event(self._body_done[slot])
        with torch.cuda.stream(ts):
            self.tail_graphs[slot].replay()
            if after_tail is not None:
                after_tail(self.tails[slot])
            self._tail_done[slot].record(ts)
        return self.tails[slot]

    def join_pipelined(self):
        """The current stream waits for the tails of both slots (e.g. before an event that closes a timed region)."""
        main = torch.cuda.current_stream()
        for ev in self._tail_done:
            main.wait_event(ev)

    def sync_pipelined(self):
        for ev in self._tail_done:
            ev.synchronize()

    def num_launches(self):
        n = 0
        for op in self.ops:
            if isinstance(op, GroupNormActOp):
                n += 2 if op.two_launch else 3
            else:
                n += 2 if getattr(op, "rgbx", 0) else 1  # packed-image stems: pack + convolution
        return n + self.tail.num_launches()


class Tail:
    """decode + per-class NMS (+ optional class-major compaction) on [B,N,row] candidate rows."""

    def __init__(self, kind, num_fg, nms_classes, score_thr, iou_thr, max_boxes, level_fn, cap=None):
        self.kind, self.num_fg, self.nms_classes = kind, num_fg, nms_classes
        # floats per candidate row, the one place the host decides it (DESIGN.md section 2): num_fg class scores + 5
        # (SSD / RetinaNet: 20 + background + 4 box; YOLOv3: 4 box + objectness; FCOS: centre-ness + 4 distances);
        # PFPNet-R's two-step rows + 11 (ODM background + 4 box, ARM 2 logits + 4 box)
        # CenterNet's peak rows + 4 (dy, dx, h, w after the keypoint logits)
        self.row = num_fg + 11 if kind == L.DECODE_TWO_STEP else num_fg + 4 if kind == L.DECODE_PEAK else num_fg + 5
        self.score_thr, self.iou_thr, self.max_boxes = score_thr, iou_thr, max_boxes
        self.level_fn, self.cap = level_fn, cap
        self.pool_cap = 8 << 20  # box-pool entries (16 B each) for lists beyond the shared-memory window

    def params(self, levels):
        """odt_tail_params of this tail over the (H, W, A) level table, candidate order: what `prepare` hands the
        decode / NMS / loss kernels, and what the training step hands the loss kernels for the same network."""
        N = sum(h * w * a for h, w, a in levels)
        p = L.TailParams()
        p.kind, p.num_levels, p.N = self.kind, len(levels), N
        p.num_fg, p.nms_classes = self.num_fg, self.nms_classes
        p.score_thr, p.iou_thr, p.max_boxes = self.score_thr, self.iou_thr, self.max_boxes
        p.cap = self.cap or N
        off = 0
        for i, (h, w, a) in enumerate(levels):
            lv = p.level[i]
            lv.H, lv.W, lv.A, lv.offset = h, w, a, off
            self.level_fn(i, h, w, lv)
            off += h * w * a
        return p

    def prepare(self, net, head_buf=None):
        dev = net.device
        B = net.batch
        self.head_buf = net.head_buf if head_buf is None else head_buf  # the candidate rows this tail reads
        self.p = p = self.params(net.levels)
        self.cand_keys = torch.zeros((B, self.num_fg, p.cap), dtype=torch.int64, device=dev)
        self.cand_count = torch.zeros((B, self.num_fg), dtype=torch.int32, device=dev)
        D = self.nms_classes * self.max_boxes
        self.D = D
        # ONE packed fixed-size record per image: D rows (score, y1, x1, y2, x2, class) followed by
        # (count, overflow flag) -- written by the NMS kernel itself; the unit the host read-back and the
        # multi-GPU all-gather ship (no pack kernels).  `dets` is the [B, D, 6] view of the same memory.
        self.rec = torch.zeros((B, D * 6 + 2), dtype=torch.float32, device=dev)
        self.dets = self.rec[:, :D * 6].view(B, D, 6)
        self.det_anchor = torch.zeros((B, D), dtype=torch.int32, device=dev)
        self.det_count = torch.zeros((B,), dtype=torch.int32, device=dev)
        nbytes = net.lib.odt_nms_scratch_bytes(C.byref(p), B)
        self.scratch = torch.zeros(max(1, (nbytes + 3) // 4), dtype=torch.int32, device=dev)  # 0 NMS classes: 0 bytes
        self.work = torch.zeros((B + (B & 1) + 2,), dtype=torch.int32, device=dev)
        self.status = torch.zeros((1,), dtype=torch.int32, device=dev)
        # box cache for candidate lists longer than the NMS shared-memory window
        total = B * self.nms_classes * p.cap
        self.pool_entries = 0 if p.cap <= 1024 else min(total, self.pool_cap)
        self.box_pool = (torch.empty((self.pool_entries, 4), dtype=torch.float32, device=dev)
                         if self.pool_entries else None)

    def launch_decode(self, net, stream):
        L.check(net.lib.odt_decode_candidates(self.head_buf.data_ptr(), C.byref(self.p), net.batch,
                                              self.cand_keys.data_ptr(), self.cand_count.data_ptr(),
                                              stream), "decode_candidates")

    def launch_nms(self, net, stream):
        L.check(net.lib.odt_nms_per_class(self.head_buf.data_ptr(), C.byref(self.p), net.batch,
                                          self.cand_keys.data_ptr(), self.cand_count.data_ptr(),
                                          self.rec.data_ptr(), self.det_anchor.data_ptr(),  # dets: a view at offset 0
                                          self.det_count.data_ptr(), self.scratch.data_ptr(),
                                          self.work.data_ptr(), self.status.data_ptr(),
                                          self.box_pool.data_ptr() if self.box_pool is not None else None,
                                          self.pool_entries, self.rec.shape[1], stream),
                "nms_per_class")

    def launch(self, net, stream):
        self.launch_decode(net, stream)
        self.launch_nms(net, stream)

    # training-loss kind -> the family's scalars of odt_<kind>_loss_fwd, in argument order, with their defaults
    LOSS_SCALARS = {"retina": (("alpha", 0.25), ("gamma", 2.0)), "ssd": (), "fcos": (),
                    "yolo": (("coord_scale", 1.0), ("noobj_scale", 1.0), ("obj_scale", 5.0), ("class_scale", 1.0)),
                    "yolo2": (("coord_scale", 1.0), ("noobj_scale", 1.0), ("obj_scale", 5.0), ("class_scale", 1.0)),
                    "pfpnet": (), "centernet": ()}

    def loss(self, net, kind, ground_truth, return_info=False, **kw):
        """Training-loss forward kernels on the rows this tail reads: kind in 'retina' | 'ssd' | 'fcos' | 'yolo' | 'yolo2' |
        'pfpnet',
        the family's scalars (LOSS_SCALARS) as keywords.  ground_truth [B,G,5] (y,x,h,w,id) padded with -1.
        Returns float32 [B]; for 'ssd' with return_info=True also int32 [B,3] = (#positives, #negatives,
        #mined negatives) per image."""
        return self._loss_call(net, kind, ground_truth, return_info, False, kw)

    def loss_grad(self, net, kind, ground_truth, return_info=False, grad_out=None, **kw):
        """odt_<kind>_loss_grad on the rows this tail reads (arguments as `loss`): (loss float32 [B], gradient
        d loss[b] / d rows[b] float32 [B,N,row]), and for 'ssd' with return_info=True the info as a third item.
        grad_out: the float32 device buffer shaped as the rows to write the gradient into (default: a fresh
        uninitialised one), e.g. one pre-filled with a sentinel to show the kernel writes every element."""
        return self._loss_call(net, kind, ground_truth, return_info, True, kw, grad_out)

    def _loss_call(self, net, kind, ground_truth, return_info, with_grad, kw, grad_out=None):
        if kind not in self.LOSS_SCALARS:
            raise ValueError(kind)
        if return_info and kind != "ssd":
            raise ValueError("return_info: only the SSD loss reports (#pos, #neg, #mined)")
        gt = torch.as_tensor(np.ascontiguousarray(ground_truth, dtype=np.float32)).to(net.device)
        B, G = gt.shape[0], gt.shape[1]
        assert B == net.batch
        p = C.byref(self.p)
        nbytes = getattr(net.lib, "odt_%s_loss_scratch_bytes" % kind)(p, B)
        scratch = torch.zeros((nbytes + 7) // 8, dtype=torch.int64, device=net.device)
        out = torch.zeros(B, dtype=torch.float32, device=net.device)
        info = torch.zeros((B, 3), dtype=torch.int32, device=net.device) if return_info else None
        grad = None
        if with_grad:
            grad = torch.empty_like(self.head_buf) if grad_out is None else grad_out
            if (grad.shape != self.head_buf.shape or grad.dtype != torch.float32 or grad.device != self.head_buf.device
                    or not grad.is_contiguous()):
                raise ValueError("grad_out: a contiguous float32 buffer shaped as the rows, on their device")
        args = [float(kw.get(k, d)) for k, d in self.LOSS_SCALARS[kind]] + [scratch.data_ptr(), out.data_ptr()]
        if kind == "ssd":
            args.append(None if info is None else info.data_ptr())
        if with_grad:
            args.append(grad.data_ptr())
        fn = "odt_%s_loss_%s" % (kind, "grad" if with_grad else "fwd")
        L.check(getattr(net.lib, fn)(self.head_buf.data_ptr(), p, B, gt.data_ptr(), G, *args,
                                     torch.cuda.current_stream().cuda_stream), kind + ("_loss_grad" if with_grad else "_loss"))
        res = [out.cpu().numpy()]
        if with_grad:
            res.append(grad.cpu().numpy())
        if return_info:
            res.append(info.cpu().numpy())
        return res[0] if len(res) == 1 else tuple(res)

    def num_launches(self):
        return 2  # decode + NMS kernels (plus 3 memset nodes)

    def results(self):
        """ONE D2H read of the packed records -> per-image [scores f32[K], bbox f32[K,4] (y1,x1,y2,x2),
        class_id i32[K]] (ref SSD300.py:190)."""
        return unpack_records(self.rec.cpu().numpy(), self.p.cap)


class PeakTail(Tail):
    """CenterNet's tail (CenterNet.py:159-185) on rows [B, H*W, num_fg + 4] of one stride-4 level: the peaks of the
    per-cell best class sigmoid above `score_thr`, the top `max_boxes` of them, boxes around their integer cells --
    odt_peak_topk, two launches, into the packed record every tail writes (D = max_boxes rows)."""

    def __init__(self, num_fg, score_thr, max_boxes):
        super().__init__(L.DECODE_PEAK, num_fg, 1, score_thr, 0.0, max_boxes, lambda i, h, w, lv: None)

    def prepare(self, net, head_buf=None):
        dev = net.device
        B = net.batch
        self.head_buf = net.head_buf if head_buf is None else head_buf
        self.p = p = self.params(net.levels)
        self.D = D = self.max_boxes
        self.rec = torch.zeros((B, D * 6 + 2), dtype=torch.float32, device=dev)
        self.dets = self.rec[:, :D * 6].view(B, D, 6)
        self.det_anchor = torch.zeros((B, D), dtype=torch.int32, device=dev)
        nbytes = net.lib.odt_peak_topk_scratch_bytes(C.byref(p), B)
        if nbytes < 0:
            raise L.OdtError("odt_peak_topk_scratch_bytes: %s" % net.lib.odt_last_error().decode())
        self.scratch = torch.zeros((nbytes + 7) // 8, dtype=torch.int64, device=dev)

    @property
    def det_count(self):
        return self.rec[:, self.D * 6].to(torch.int32)

    def launch(self, net, stream):
        L.check(net.lib.odt_peak_topk(self.head_buf.data_ptr(), C.byref(self.p), net.batch, self.scratch.data_ptr(),
                                      self.rec.data_ptr(), self.rec.shape[1], self.det_anchor.data_ptr(), stream),
                "peak_topk")

    def num_launches(self):
        return 2  # per-cell score + peak / top-k selection


MAX_LOSS_GT = 128  # GT rows per image the loss kernels hold (kMaxGT in csrc/loss.cu)


def loss_ground_truth(ground_truth):
    """Ground truth [B,G,5] (y,x,h,w,id) padded with -1 -> float32 ndarray the loss kernels take.  An image's box
    count is the index of its first minimum in column 0 (the reference's argmin).  When G exceeds the kernels' 128
    rows, the array is cut to the rows the counts reach (max count + 1 rows keep every count: no earlier row holds the
    minimum), computed here in numpy; an image whose count needs more than 128 rows (128 boxes or more ahead of its
    first padding row) is a ValueError."""
    gt = np.ascontiguousarray(ground_truth, dtype=np.float32)
    if gt.ndim != 3 or gt.shape[2] != 5 or gt.shape[1] < 1:
        raise ValueError("ground truth: expected shape [B, G, 5] with G >= 1, got %s" % (gt.shape,))
    if gt.shape[1] <= MAX_LOSS_GT:
        return gt
    cnt = np.argmin(gt[:, :, 0], axis=1)
    need = int(cnt.max()) + 1
    if need > MAX_LOSS_GT:
        b = int(np.argmax(cnt))
        raise ValueError("ground truth: image %d has %d boxes ahead of its first padding row; the loss kernels hold %d "
                         "GT rows per image, so at most %d boxes when the rows are padded beyond %d"
                         % (b, int(cnt[b]), MAX_LOSS_GT, MAX_LOSS_GT - 1, MAX_LOSS_GT))
    return np.ascontiguousarray(gt[:, :need])


def check_class_labels(labels, batch, num_classes):
    """Sparse class labels [B] (or the reference's [B, 1] placeholder shape) -> int64 ndarray [B].  A label outside
    [0, num_classes) is a ValueError, as TF's sparse_softmax_cross_entropy CPU kernel rejects it."""
    lab = np.asarray(labels)
    if lab.ndim == 2 and lab.shape[1] == 1:
        lab = lab[:, 0]
    if lab.shape != (batch,):
        raise ValueError("labels: expected shape [%d], got %s" % (batch, np.asarray(labels).shape))
    if lab.dtype.kind not in "iu" and not (lab.dtype.kind == "f" and np.all(lab == np.floor(lab))):
        raise ValueError("labels must be integer class ids")
    lab = lab.astype(np.int64)
    bad = (lab < 0) | (lab >= num_classes)
    if bad.any():
        raise ValueError("label %d of image %d is outside [0, %d)" % (lab[bad][0], int(np.nonzero(bad)[0][0]),
                                                                     num_classes))
    return lab


class ClassifyTail:
    """Classification tail of RetinaNet's pretraining mode (ref RetinaNet.py:123-127) on the last feature tensor
    `feat`: fp32 logits [B, C] = mean over H x W, `pred` int64 [B] = their first maximum, and on request the
    per-image sparse softmax cross-entropy -- one odt_pool_classify launch.  Same interface as Tail."""

    def __init__(self, feat):
        self.feat = feat

    def prepare(self, net):
        self.logits = torch.zeros((net.batch, self.feat.C), dtype=torch.float32, device=net.device)
        self.pred = torch.zeros((net.batch,), dtype=torch.int64, device=net.device)

    def launch(self, net, stream, labels=None, loss=None):
        f = self.feat
        L.check(net.lib.odt_pool_classify(f.ptr(), net.dt, f.B, f.H, f.W, f.C, f.ld, f.halo, self.logits.data_ptr(),
                                          self.pred.data_ptr(), labels.data_ptr() if labels is not None else None,
                                          loss.data_ptr() if loss is not None else None, stream), "pool_classify")

    def loss(self, net, labels):
        """Per-image sparse softmax cross-entropy [B] (float32 ndarray) of the features the last forward left in
        `feat`; also refreshes `logits` / `pred`.  Labels are checked on the host before the launch."""
        lab = torch.from_numpy(check_class_labels(labels, net.batch, self.feat.C)).to(net.device)
        out = torch.zeros((net.batch,), dtype=torch.float32, device=net.device)
        self.launch(net, torch.cuda.current_stream().cuda_stream, lab, out)
        return out.cpu().numpy()

    def num_launches(self):
        return 1

    def results(self):
        """pred int64 [B] (ref RetinaNet.py:127,501-503)."""
        return self.pred.cpu().numpy()


class Detections:
    """Sequence view over packed detection records [M, D*6+2] (host memory): item b is the reference's
    per-image result `[scores f32[K], bbox f32[K,4] (y1,x1,y2,x2), class_id i32[K]]` (SSD300.py:190).
    Built with three vectorised passes over the whole record block; indexing slices views."""

    def __init__(self, rec):
        rec = np.asarray(rec)
        M, D = rec.shape[0], (rec.shape[1] - 2) // 6
        rows = rec[:, :D * 6].reshape(M, D, 6)
        self.count = rec[:, D * 6].astype(np.int64)
        self.scores = np.ascontiguousarray(rows[:, :, 0])
        self.boxes = np.ascontiguousarray(rows[:, :, 1:5])
        self.class_id = rows[:, :, 5].astype(np.int32)

    def __len__(self):
        return self.count.shape[0]

    def __getitem__(self, b):
        if isinstance(b, slice):
            return [self[i] for i in range(*b.indices(len(self)))]
        if b < 0:
            b += len(self)
        if not 0 <= b < len(self):
            raise IndexError(b)
        k = self.count[b]
        return [self.scores[b, :k], self.boxes[b, :k], self.class_id[b, :k]]

    def __iter__(self):
        return (self[i] for i in range(len(self)))


def unpack_records(rec, cap=None):
    """Packed records (numpy [M, D*6+2]) -> Detections; raises if any image's overflow flag is set
    (a candidate list was truncated at its capacity: the result would silently lack boxes)."""
    rec = np.asarray(rec)
    if rec.shape[0] and float(rec[:, -1].max()) != 0.0:
        bad = np.nonzero(rec[:, -1])[0]
        raise L.OdtError("NMS candidate list overflowed its capacity%s in image(s) %s"
                         % ("" if cap is None else " (cap=%d)" % cap, bad[:8].tolist()))
    return Detections(rec)


class RowsHarness:
    """Runs a Tail on caller-provided candidate rows [B,N,tail.row] (no backbone):
    the tail kernels in isolation, for parity tests and the decode/NMS microbench."""

    def __init__(self, tail, levels, rows, device="cuda"):
        self.lib = L.load()
        self.device = torch.device(device)
        self.levels = list(levels)
        self.head_buf = torch.as_tensor(np.ascontiguousarray(rows, dtype=np.float32)).to(self.device)
        self.batch, self.N = self.head_buf.shape[0], self.head_buf.shape[1]
        assert self.N == sum(h * w * a for h, w, a in self.levels) and self.head_buf.shape[2] == tail.row
        self.tail = tail
        tail.prepare(self)

    def run(self):
        self.tail.launch(self, torch.cuda.current_stream().cuda_stream)
        return self.tail.results()

    def keep_indices(self):
        cnt = self.tail.det_count.cpu().numpy()
        anc = self.tail.det_anchor.cpu().numpy()
        return [anc[b, :cnt[b]].copy() for b in range(self.batch)]

    def loss(self, kind, ground_truth, return_info=False, **kw):
        """Training-loss forward kernels on the same rows (Tail.loss)."""
        return self.tail.loss(self, kind, ground_truth, return_info, **kw)

    def loss_grad(self, kind, ground_truth, return_info=False, grad_out=None, **kw):
        """Training-loss gradient kernels on the same rows (Tail.loss_grad): (loss [B], gradient [B,N,row])."""
        return self.tail.loss_grad(self, kind, ground_truth, return_info, grad_out, **kw)


# ------------------------------------------------------------------ weights --
def init_weights(variables, seed=1, bn_mode="tf_init", stem_scale=1.0 / 64.0):
    """Seeded random initialisation in TF layout (HWIO kernels), creation order.
    Conv kernels He-normal N(0, 2/fan_in); biases 0 (or -log(99) for 'pi');
    BN/GN parameters at their TF initial values ('tf_init') or a 'trained'-like
    random set so that folding is actually exercised (SURVEY 8d).
    The kernel that consumes the image (Cin == 3) is additionally scaled by
    `stem_scale`: mean-subtracted pixels have std ~74, and with He init that
    magnitude would propagate to the logits (saturated softmax, exp overflow);
    1/64 keeps random-init activations O(1), as trained weights do."""
    rng = np.random.default_rng(seed)
    out = {}
    trained = bn_mode != "tf_init"
    for name, (shape, kind) in variables.items():
        if kind == "he":
            fan_in = shape[0] * shape[1] * shape[2]
            out[name] = (rng.standard_normal(shape) * math.sqrt(2.0 / fan_in)).astype(np.float32)
            if shape[2] == 3:
                out[name] *= np.float32(stem_scale)
            # pre-activation bottlenecks sum two conv branches (no identity path,
            # RetinaNet.py:641-643): halve the variance of each so random-init
            # activations do not double per block (2^16 over 16 blocks)
            if "/conv_branch/conv2d_2/" in name or "/identity_branch/conv2d/" in name:
                out[name] *= np.float32(math.sqrt(0.5))
            # basic units (RetinaNet.py:621-632) end their conv branch in conv2d_1 and add the unit's input at stride
            # 1: damp that conv likewise, or the variance would double per unit
            if name.endswith("/conv_branch/conv2d_1/kernel") and \
                    name.replace("/conv2d_1/", "/conv2d_2/") not in variables:
                out[name] *= np.float32(math.sqrt(0.5))
            # Darknet residual x + f(x) (YOLOv3.py:488-491): damp f's last conv likewise
            mres = re.match(r"backone/block\d+/conv2d_(\d+)/kernel", name)
            if mres and int(mres.group(1)) >= 2 and int(mres.group(1)) % 2 == 0:
                out[name] *= np.float32(0.25)
        elif kind == "zeros":
            out[name] = np.zeros(shape, np.float32)
        elif kind == "pi":
            out[name] = np.full(shape, -math.log((1 - 0.01) / 0.01), np.float32)
        elif kind.startswith("l2norm"):  # "l2norm": 20 (SSD); "l2norm_<v>": v
            out[name] = np.full(shape, 20.0 if kind == "l2norm" else float(kind[7:]), np.float32)
        elif kind in ("bn_gamma", "gn_gamma"):
            out[name] = (rng.uniform(0.8, 1.2, shape).astype(np.float32) if trained
                         else np.ones(shape, np.float32))
        elif kind in ("bn_beta", "gn_beta", "bn_mean"):
            out[name] = ((rng.standard_normal(shape) * 0.1).astype(np.float32) if trained
                         else np.zeros(shape, np.float32))
        elif kind == "bn_var":
            out[name] = (rng.uniform(0.8, 1.25, shape).astype(np.float32) if trained
                         else np.ones(shape, np.float32))
        else:
            raise ValueError(kind)
    return out
