"""Float64 references and per-element forward-error bounds for the two ends of the convolution stack: the Cin = 3 stems
and the fp32 head convolutions that scatter into the candidate rows (tests/test_gpu_conv_ends.py).  No GPU needed: every
function runs on whatever device its tensors live on.

Reference: the convolution in float64 of exactly the operands the kernel multiplies (the fp16 or fp32 weights; for the
stems the input fp16(fp32(image) - mean) on the tensor-core stems, and fp32(image) - mean, unrounded, on the CUDA-core
stems, which load the fp32 image in either output dtype), TF SAME padding from engine.same_pad, then
act(acc * scale + shift) with the fp32 scale / shift and the kernel's fp32 leaky slope 0.1f.

Bound, per element:  |got - ref| <= n_acc * u32 * |scale| * sum|x * w|  +  2 * u32 * |ref|  [ + fp16 output rounding ]
  * sum|x * w| is a second float64 convolution of |x| and |w|; relu, leaky and the identity are 1-Lipschitz, so the
    accumulation error passes the activation scaled by |scale| at most;
  * 2 * u32 * |ref|: the epilogue's fmaf rounds once, leaky's 0.1f * v rounds once more;
  * fp16 outputs: the fp32 value is rounded once more, by at most u16 * |value| + 2^-25 (half the subnormal spacing);
  * n_acc, the accumulation depth of the path (n_acc_* below):
      - CUDA-core kernels (conv_stem_kernel, conv_direct_kernel): one fmaf chain over K = R*S*Cin products, each step
        rounding once: |err| <= gamma_K * sum|x*w| <= (K + 1) * u32 * sum|x*w| (the +1 covers gamma's denominator
        K*u/(1 - K*u) at these K);
      - wgmma kernels (conv_stem_tc_kernel, conv_tc_kernel): fp16 x fp16 products are exact in fp32, but the tensor
        core adds a block of b products and the accumulator with the significands aligned to the largest exponent and
        truncated, then truncates the sum (no round-to-nearest: up to 2 u32 per lost bit position instead of u32).  A
        block then errs by at most 2 * u32 * (b + 2) * (|accumulator| + its products) <= 2 * u32 * (b + 2) * sum|x*w|
        over its prefix, and Kp / b blocks give 2 * (b + 2) / b * Kp <= 3 * Kp for b >= 4, where Kp is the K extent the
        kernel issues (k16 steps of its im2col row, zero padding included: zeros add exactly).

The body convolutions (tests/test_gpu_conv.py's _conv_case, tests/test_gpu_conv_body.py) add, per path and per output:
  * n_acc of the body kernels:
      - conv_tc_kernel and conv_tc_swap_kernel: 3 * Kp with Kp = R*S*in_ld (the swap kernel issues the same k16 steps
        in the same order, pixels on the other wgmma side);
      - conv_tapn_kernel: three tap partials of Kp/3 each on the tensor core, 3 * Kp/3 * u32 * sum_s|x*w| each, then
        p0 + p1 + p2 in two fp32 additions, at most 2 * u32 * (1 + Kp * u32) * sum|x*w| more: in all
        (Kp + 2 + 2 * Kp * u32) * u32 * sum|x*w| <= 3 * Kp * u32 * sum|x*w| since Kp >= 16;
      - conv_pw_kernel, conv_thin_kernel, conv_direct_kernel: fmaf chains (any order of fp32 additions is within
        gamma_K too), K + 1 with K = R*S*Cin.
  * Residual: v = act(acc*s + h) + r with r the fp16 (or fp32) residual: the element bound of a = act(...) above,
    then one more fp32 rounding of the sum, u32 * (|v| + that bound).
  * Fused 2x2/2 max-pool: the reference pools the float64 values, the bound is the window maximum of the element
    bounds.  max is 1-Lipschitz in the infinity norm and fp16 rounding is monotone, so pooling rounded values and
    rounding pooled values give the same result, within the largest element error of the window.
  * out1 / out2 = act2(fmaf(v, s2, h2)) when out0 is stored: against act2(out0_got * s2 + h2) from the kernel's own
    out0, at most one ulp of the output type (the kernel's fmaf is exact up to its one rounding, then fp16 rounds once;
    leaky's 0.1f * t adds u32).
  * out1 / out2 when out0 is not stored: v's bound, fp16 rounding included for fp16 layers (the kernels round v
    before the consumer step either way), times |s2|, plus the fmaf / leaky roundings 2 * u32 * |t| and the output
    rounding u16 * |t| + 2^-25.
"""
import numpy as np
import torch
import torch.nn.functional as F

U32 = 2.0 ** -24
U16 = 2.0 ** -11
F16_HALF_SUB = 2.0 ** -25
MEAN = np.array([123.68, 116.779, 103.979], np.float32)  # the stems' RGB mean (SSD300.py:52-66 of the reference)
LEAKY = float(np.float32(0.1))
ACTS = {None: 0, "relu": 1, "leaky": 2}


def same_pad(size, k, stride, dil=1):
    from odt_b200.engine import same_pad as sp
    return sp(size, k, stride, dil)


# ---- accumulation depth per path ------------------------------------------------------------------------------------
def n_acc_cuda_core(R, S, Cin):
    return R * S * Cin + 1


def n_acc_wgmma(kp):
    return 3 * kp


def n_acc_stem_tc(k, rgbx):
    """conv_stem_tc_kernel: the fp32-gather variants issue ceil(k*k*3 / 16) k16 steps; the packed RGBX variant k rows of
    8 pixels x 4 channels (the eighth tap and the X channel have zero weights)."""
    return n_acc_wgmma(k * 8 * 4 if rgbx else -(-k * k * 3 // 16) * 16)


def n_acc_conv_tc(R, S, in_ld):
    """conv_tc_kernel: R*S taps of in_ld / 64 channel chunks of 64."""
    return n_acc_wgmma(R * S * in_ld)


def n_acc_tapn(R, S, in_ld):
    """conv_tapn_kernel: three tap partials of R*in_ld each plus two fp32 additions, within 3 * Kp (see the module
    docstring)."""
    kp = R * S * in_ld
    assert kp + 2 <= n_acc_wgmma(kp)
    return n_acc_wgmma(kp)


def n_acc_body(kernel, R, S, Cin, in_ld):
    """n_acc of the body-convolution kernel named `kernel` (a launched kernel's name)."""
    if "conv_tapn_kernel" in kernel:
        return n_acc_tapn(R, S, in_ld)
    if "conv_tc_kernel" in kernel or "conv_tc_swap_kernel" in kernel:
        return n_acc_conv_tc(R, S, in_ld)
    assert any(k in kernel for k in ("conv_pw_kernel", "conv_thin_kernel", "conv_direct_kernel")), kernel
    return n_acc_cuda_core(R, S, Cin)


# ---- operands and reference ------------------------------------------------------------------------------------------
def stem_operand(img, f16):
    """fp32 image [B,H,W,3] -> the operand the stems multiply: fp32(img) - mean (one correctly rounded subtraction, as
    __fsub_rn), rounded to fp16 for the tensor-core stems (odt_pack_input_rgbx and the fp32 gather both do this)."""
    x = img.float() - torch.from_numpy(MEAN).to(img.device)
    return x.half() if f16 else x


def conv64(x, w, stride, dil=1):
    """TF SAME convolution of NHWC x [B,H,W,Cin] with KRSC w [Cout,R,S,Cin], in float64 -> NHWC."""
    _, H, W, _ = x.shape
    _, R, S, _ = w.shape
    _, pt, pb = same_pad(H, R, stride, dil)
    _, pl, pr = same_pad(W, S, stride, dil)
    t = F.pad(x.double().permute(0, 3, 1, 2), (pl, pr, pt, pb))
    y = F.conv2d(t, w.double().permute(0, 3, 1, 2), stride=stride, dilation=dil)
    return y.permute(0, 2, 3, 1)


def act64(v, act):
    if act == "relu":
        return v.clamp_min(0)
    if act == "leaky":
        return torch.maximum(v, LEAKY * v)
    return v


def reference(x, w, stride, scale, shift, act, dil=1):
    """(ref, mag): act(conv(x, w) * scale + shift) and |scale| * conv(|x|, |w|), float64 NHWC.  scale None = 1."""
    Cout = w.shape[0]
    sc = torch.ones(Cout, dtype=torch.float64, device=x.device) if scale is None else scale.double()[:Cout]
    sh = shift.double()[:Cout]
    ref = act64(conv64(x, w, stride, dil) * sc + sh, act)
    mag = conv64(x.abs(), w.abs(), stride, dil) * sc.abs()
    return ref, mag


def bound(ref, mag, n_acc, out16, res=None):
    """Element bound of act(acc * scale + shift) (+ res, the residual as the kernel reads it) against ref."""
    acc = n_acc * U32 * mag
    if res is None:
        b = acc + 2 * U32 * ref.abs()
        e = acc
    else:
        b = acc + 2 * U32 * (ref - res.double()).abs()
        b = b + U32 * (ref.abs() + b)
        e = b
    if out16:
        b = b + U16 * (ref.abs() + e) + F16_HALF_SUB
    return b


def pool2(t):
    """2x2 / stride-2 max-pool of NHWC t (even H and W: the fused pool's SAME pads are zero)."""
    B, H, W, Cc = t.shape
    return t.reshape(B, H // 2, 2, W // 2, 2, Cc).amax(dim=(2, 4))


def consumer(v, s2, h2, act2):
    """act2(v * s2 + h2) in float64: a consumer pre-activation (out1 / out2) of the value v."""
    return act64(v.double() * s2.double() + h2.double(), act2)


def bound_own(t, out16):
    """out1 / out2 against consumer() of the kernel's own stored out0: one ulp of the output type, plus leaky's
    extra rounding."""
    u = U16 if out16 else U32
    return 2 * u * t.abs() + 2 * U32 * t.abs() + (2.0 ** -24 if out16 else 2.0 ** -149)


def bound_through(t, b0, s2, out16):
    """out1 / out2 when out0 is not stored: v's bound b0 (its fp16 rounding included) through |s2|, the fmaf and leaky
    roundings, and the output rounding."""
    b = b0 * s2.double().abs() + 2 * U32 * t.abs()
    if out16:
        b = b + U16 * (t.abs() + b) + F16_HALF_SUB
    return b


def ratio(got, ref, b):
    """Worst |got - ref| / b (NaN in got counts as infinitely wrong, an exact element as 0 even where b is 0), and the
    first element at that fraction."""
    err = (got.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / b)
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    i = int(torch.argmax(r.reshape(-1)))
    return float(r.reshape(-1)[i]), tuple(int(a) for a in np.unravel_index(i, tuple(r.shape)))


def worst(got, ref, mag, n_acc, out16):
    """Worst |got - ref| as a fraction of the bound (NaN in got counts as infinitely wrong), and the first element at
    that fraction."""
    err = (got.double() - ref).abs()
    r = err / bound(ref, mag, n_acc, out16)
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    i = int(torch.argmax(r.reshape(-1)))
    return float(r.reshape(-1)[i]), tuple(int(a) for a in np.unravel_index(i, tuple(r.shape)))


def checked(got_fn, x, w, stride, scale, shift, act, n_acc, out16, chunk=None, dil=1):
    """worst() over the batch in chunks of `chunk` images (the float64 convolutions of a full-size batch would need
    several times the activation's memory at once).  got_fn(b0, b1) -> the kernel's output of images b0..b1-1."""
    B = x.shape[0]
    chunk = chunk or B
    out = (0.0, None)
    for b0 in range(0, B, chunk):
        b1 = min(B, b0 + chunk)
        ref, mag = reference(x[b0:b1], w, stride, scale, shift, act, dil)
        r, at = worst(got_fn(b0, b1), ref, mag, n_acc, out16)
        if r > out[0] or out[1] is None:
            out = (r, (b0 + at[0],) + tuple(int(a) for a in at[1:]))
        del ref, mag
    return out


# ---- head scatter ----------------------------------------------------------------------------------------------------
def regroup(n, group, gstride):
    """Column of output channel n within the head's slice of a candidate row (epilogue.cuh regroup)."""
    return (n // group) * gstride + n % group if group > 0 else n


def head_index(OH, OW, Cout, head, row):
    """Element offsets inside one image's [N, row] candidate rows of the head's outputs: [OH*OW, Cout] int64.
    head = (lvl_off, col, group, gstride, A) as the engine gives it (pixel stride A * row)."""
    lvl_off, col, group, gstride, A = head
    n = torch.arange(Cout, dtype=torch.int64)
    cols = regroup(n, group, gstride)
    pix = torch.arange(OH * OW, dtype=torch.int64)
    return lvl_off * row + col + pix[:, None] * (A * row) + cols[None, :]


def head_gather(rows, OH, OW, Cout, head, b0=0, b1=None):
    """The head's outputs [b1-b0, OH, OW, Cout] read back out of candidate rows [B, N, row]."""
    B, N, row = rows.shape
    b1 = B if b1 is None else b1
    idx = head_index(OH, OW, Cout, head, row).to(rows.device).reshape(-1)
    return rows[b0:b1].reshape(b1 - b0, N * row)[:, idx].reshape(b1 - b0, OH, OW, Cout)


def head_scatter(vals, N, row, head, fill=float("nan")):
    """Candidate rows [B, N, row] holding vals [B, OH, OW, Cout] at the head's columns and `fill` elsewhere."""
    B, OH, OW, Cout = vals.shape
    rows = torch.full((B, N * row), fill, dtype=vals.dtype, device=vals.device)
    idx = head_index(OH, OW, Cout, head, row).to(vals.device).reshape(-1)
    rows[:, idx] = vals.reshape(B, -1)
    return rows.reshape(B, N, row)


def head_owners(N, row, heads, device="cpu"):
    """How many heads write each element of one image's candidate rows: heads = [(OH, OW, Cout, head), ...]."""
    cnt = torch.zeros(N * row, dtype=torch.int32, device=device)
    for OH, OW, Cout, head in heads:
        idx = head_index(OH, OW, Cout, head, row).to(device).reshape(-1)
        assert int(idx.min()) >= 0 and int(idx.max()) < N * row, "head outside the candidate rows"
        cnt.index_add_(0, idx, torch.ones_like(idx, dtype=torch.int32))
    return cnt.reshape(N, row)
