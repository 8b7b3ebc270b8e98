"""ORACLE (test infrastructure -- never imported by the product path).

CPU restatement of the reference's altcorr ops in plain PyTorch (fp64 by default):
    corr_raw / corr_forward   dpvo/altcorr/correlation_kernel.cu:82-136 (8x8 integer taps, zero
                              outside the map) + :221-232 (bilinear blend to 7x7, swap to (x, y))
    corr_grid_sample          the algebraically identical F.grid_sample form named by BASELINE.json
                              config 1 (bilinear, zeros padding, align_corners=True); used as the
                              CPU baseline and as an independent cross-check of corr_forward
    patchify_forward          correlation_kernel.cu:16-47 + the Python blend of correlation.py:51-68
Backward passes are obtained by autograd through these (exact transposes of linear maps), which
restates correlation_kernel.cu:139-190, 252-269 and :49-80.

Pinning: the reference holds no golden vectors for altcorr (SURVEY 4).  The oracle is pinned by
(i) the two independent formulations agreeing to fp64 round-off (tests/test_oracle_corr.py) and
(ii) on the GPU box, the reference's own kernels compiled from /root/reference into oracle/_ref
(oracle/build_ref.py) agreeing with it on seeded inputs (tests/test_parity_ref_gpu.py), with the
committed fixtures in tests/golden/ generated from those kernels.

Per-element error bars of the kernels (corr_bar, corr_backward_bar, patchify_backward_bar, corr_interval).  The blend
weights are non-negative, so S = corr_forward(|f1|, |f2|) = sum_c w_c sum_k |f1_k f2_k| is exactly the magnitude the
fp32 accumulation and the blend act on.  The model, with u = 2^-24:
  * fp16 x fp16 products are exact in fp32 (and fp32 x fp32 products are fused into the accumulation, FMA);
  * the accumulation of one raw tap rounds once per step: per k16 step of the tensor-core accumulator (the model
    DESIGN section 4 states for the SoftAgg; it has NOT been measured), per channel in the generic kernel.  ACC_MMA
    (two chains of four k16 steps and their join), ACC_WGMMA (eight k16 steps in one chain), acc_generic(C);
  * the blend adds BLEND = 7 roundings: 1 - fx, 1 - fy and their product for each weight, then the four-term fp32
    multiply-add.  The fractions fx = x - floor(x) need no term: corr_forward forms them in fp32 as the kernels do
    (exact for x >= 0, the kernels' own rounding for x < 0);
  * so before the output rounding |kernel - ref| <= b = gamma(n) S with n = accumulator + BLEND roundings and
    gamma(n) = n u / (1 - n u) (Higham's bound for n roundings);
  * then one rounding to the output dtype, judged by brackets: an fp16 (bf16) output must lie in
    [RN(ref - b), RN(ref + b)], rounded from float64 in one step (round_to); an fp32 output in [ref - b, ref + b].
Backward: the same bound on the gradients of the absolute-value form, with n counting every rounding on the way
to a gradient element, the fp32 atomics (one per contributing edge) included.
"""
import numpy as np
import torch
import torch.nn.functional as F


def corr_raw(fmap1, fmap2, coords, ii, jj, radius):
    """[B, M, D(y tap), D(x tap), P, P] raw taps, D = 2R+2  (correlation_kernel.cu:82-136)."""
    B, M, _, P, _ = coords.shape
    C = fmap1.shape[2]
    H2, W2 = fmap2.shape[3], fmap2.shape[4]
    D = 2 * radius + 2
    dt = fmap1.dtype
    f1 = fmap1[:, ii]                                   # [B, M, C, P, P]
    f2 = fmap2.transpose(1, 2).reshape(B, C, -1)        # [B, C, S2 * H2 * W2]: gathered per tap, not per edge frame
    x0 = torch.floor(coords[:, :, 0]).long()            # [B, M, P, P]
    y0 = torch.floor(coords[:, :, 1]).long()
    taps = torch.arange(D, device=coords.device) - radius
    yy = y0[:, :, None, None] + taps[None, None, :, None, None, None]      # [B,M,D,1,P,P]
    xx = x0[:, :, None, None] + taps[None, None, None, :, None, None]      # [B,M,1,D,P,P]
    yy = yy.expand(B, M, D, D, P, P)
    xx = xx.expand(B, M, D, D, P, P)
    inb = (yy >= 0) & (yy < H2) & (xx >= 0) & (xx < W2)
    lin = jj.to(coords.device)[None, :, None, None, None, None] * (H2 * W2) + yy.clamp(0, H2 - 1) * W2 + xx.clamp(0, W2 - 1)
    g = torch.gather(f2, 2, lin.reshape(B, 1, -1).expand(B, C, -1)).reshape(B, C, M, D, D, P, P).transpose(1, 2)
    out = (g * f1[:, :, :, None, None]).sum(2)
    return torch.where(inb, out, torch.zeros((), dtype=dt, device=out.device))


def corr_forward(fmap1, fmap2, coords, ii, jj, radius, chunk=256):
    """cuda_corr.forward: [B, M, 2R+1 (x off), 2R+1 (y off), P, P]  (:193-233)."""
    M = coords.shape[1]
    if M > chunk:   # bound the [chunk, C, D, D, P, P] gather
        return torch.cat([corr_forward(fmap1, fmap2, coords[:, s:s + chunk], ii[s:s + chunk], jj[s:s + chunk], radius, chunk)
                          for s in range(0, M, chunk)], 1)
    D = 2 * radius + 2
    raw = corr_raw(fmap1, fmap2, coords, ii, jj, radius)
    # fractions are formed in the dtype of coords (fp32 in DPVO) and only then cast (:221-224)
    x, y = coords[:, :, 0, None, None], coords[:, :, 1, None, None]
    dx = (x - torch.floor(x)).to(fmap1.dtype)
    dy = (y - torch.floor(y)).to(fmap1.dtype)
    out = (1 - dx) * (1 - dy) * raw[:, :, 0:D - 1, 0:D - 1]
    out = out + dx * (1 - dy) * raw[:, :, 0:D - 1, 1:D]
    out = out + (1 - dx) * dy * raw[:, :, 1:D, 0:D - 1]
    out = out + dx * dy * raw[:, :, 1:D, 1:D]
    return out.permute(0, 1, 3, 2, 4, 5)


def corr_grid_sample(fmap1, fmap2, coords, ii, jj, radius):
    """Same result through F.grid_sample: correlation is linear in fmap2 and out-of-image taps are
    zero, so sampling fmap2 bilinearly at coords + integer offsets and dotting with fmap1 equals the
    blend of raw integer taps (SURVEY 8(c))."""
    B, M, _, P, _ = coords.shape
    C = fmap1.shape[2]
    H2, W2 = fmap2.shape[3], fmap2.shape[4]
    O = 2 * radius + 1
    offs = torch.arange(O, device=coords.device, dtype=coords.dtype) - radius
    out = torch.zeros(B, M, O, O, P, P, dtype=fmap1.dtype, device=fmap1.device)
    for b in range(B):
        for j in torch.unique(jj).tolist():                           # one grid_sample per target frame
            sel = torch.nonzero(jj == j).squeeze(1)
            n = sel.numel()
            f1 = fmap1[b, ii[sel]]                                    # [n, C, P, P]
            x = coords[b, sel, 0].to(fmap1.dtype)                     # [n, P, P]
            y = coords[b, sel, 1].to(fmap1.dtype)
            gx = (x[:, None, None] + offs.to(fmap1.dtype)[None, :, None, None, None]).expand(n, O, O, P, P)
            gy = (y[:, None, None] + offs.to(fmap1.dtype)[None, None, :, None, None]).expand(n, O, O, P, P)
            grid = torch.stack([2 * gx / (W2 - 1) - 1, 2 * gy / (H2 - 1) - 1], -1).reshape(1, n * O * O * P, P, 2)
            samp = F.grid_sample(fmap2[b, j][None], grid, mode="bilinear", padding_mode="zeros", align_corners=True)
            samp = samp.reshape(C, n, O, O, P, P).permute(1, 0, 2, 3, 4, 5)
            out[b, sel] = (samp * f1[:, :, None, None]).sum(1)
    return out


def patchify_raw(net, coords, radius):
    """cuda_corr.patchify_forward: [B, M, C, D, D] window at floor(coords), zero outside (:16-47)."""
    B, C, H, W = net.shape
    M = coords.shape[1]
    D = 2 * radius + 2
    taps = torch.arange(D, device=coords.device) - radius
    x0 = torch.floor(coords[..., 0]).long()
    y0 = torch.floor(coords[..., 1]).long()
    yy = (y0[:, :, None, None] + taps[None, None, :, None]).expand(B, M, D, D)
    xx = (x0[:, :, None, None] + taps[None, None, None, :]).expand(B, M, D, D)
    inb = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
    lin = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).reshape(B, 1, M * D * D).expand(B, C, -1)
    g = torch.gather(net.reshape(B, C, H * W), 2, lin).reshape(B, C, M, D, D).permute(0, 2, 1, 3, 4)
    return torch.where(inb[:, :, None], g, torch.zeros((), dtype=net.dtype, device=net.device))


def patchify(net, coords, radius, mode="bilinear"):
    """altcorr.patchify (correlation.py:51-68)."""
    patches = patchify_raw(net, coords, radius)
    if mode == "bilinear":
        offset = coords - coords.floor()
        dx, dy = offset[:, :, None, None, None].unbind(dim=-1)
        d = 2 * radius + 1
        x00 = (1 - dy) * (1 - dx) * patches[..., :d, :d]
        x01 = (1 - dy) * dx * patches[..., :d, 1:]
        x10 = dy * (1 - dx) * patches[..., 1:, :d]
        x11 = dy * dx * patches[..., 1:, 1:]
        return x00 + x01 + x10 + x11
    return patches


# ------------------------------------------------------------------------------------------------ error bars
U32 = 2.0 ** -24
ACC_MMA = 5          # corr_fwd_mma / corr_fwd_l1_tiles: two chains of four k16 steps (C = 128) and their join
ACC_WGMMA = 8        # corr_fwd_tc: eight k16 steps on one accumulator
BLEND = 7            # 1 - fx, 1 - fy, the weight product; the four-term multiply-add


def acc_generic(C):
    """corr_fwd_generic: one fused multiply-add per channel, over the channels padded to a multiple of 4"""
    return (C + 3) // 4 * 4


def gamma(n):
    return n * U32 / (1 - n * U32)


def level_coords(coords, div):
    """the coordinates of a pyramid level as the kernels form them: x / div in fp32 (IEEE division; a CUDA tensor
    divided by a Python scalar is multiplied by its reciprocal instead)"""
    if div == 1:
        return coords
    c = coords.detach().float().cpu().numpy() / np.float32(div)
    return torch.from_numpy(c).to(coords.device)


def corr_bar(fmap1, fmap2, coords, ii, jj, radius, n_acc):
    """(ref, b): the float64 correlation and the bar before the output rounding, per output element"""
    f1, f2 = fmap1.double(), fmap2.double()
    ref = corr_forward(f1, f2, coords, ii, jj, radius)
    S = corr_forward(f1.abs(), f2.abs(), coords, ii, jj, radius)
    return ref, gamma(n_acc + BLEND) * S


_FORMATS = {torch.float16: (11, -24), torch.bfloat16: (8, -133)}     # significand bits, exponent of the least ulp
_MAX = {torch.float16: 65504.0, torch.bfloat16: float(torch.finfo(torch.bfloat16).max)}


def round_to(x, dtype):
    """float64 -> the nearest fp16 / bf16 value (ties to even, overflow to inf), in ONE rounding, as float64.  torch's
    CPU cast from float64 may go through float32 first, which rounds twice.  Computed on the CPU, where it is pinned to
    numpy's conversion (tests/test_corr_ref_cpu.py), whatever the device of x"""
    dev, p, qmin = x.device, *_FORMATS[dtype]
    x = x.double().cpu()
    _, e = torch.frexp(x)                                 # x = m 2^e, 1/2 <= |m| < 1
    ulp = torch.pow(2.0, torch.clamp(e - p, min=qmin).double())
    r = torch.round(x / ulp) * ulp                        # division by a power of two: exact; round: ties to even
    return torch.where(r.abs() > _MAX[dtype], torch.copysign(torch.full_like(r, float("inf")), r), r).to(dev)


def corr_interval(ref, b, dtype):
    """[lo, hi] that an output of `dtype` must lie in"""
    lo, hi = ref - b, ref + b
    if dtype in _FORMATS:
        lo, hi = round_to(lo, dtype), round_to(hi, dtype)
    return lo, hi


def bar_use(out, ref, b):
    """the smallest bar b' with out in corr_interval(ref, b', out.dtype), over b (<= 1: inside the bar).  0 for an fp16
    output that is ref correctly rounded; ties to even are ignored"""
    o = out.double().to(ref.device)
    if out.dtype in _FORMATS:
        # the rounding cell of each output value: half-way to its neighbours (int16 patterns +-1 for fp16 and bf16)
        bits = out.contiguous().view(torch.int16).to(torch.int32)
        zero = o == 0
        safe = torch.where(zero, torch.ones_like(bits), bits)
        up = (safe + 1).to(torch.int16).view(out.dtype).double().to(ref.device)
        down = (safe - 1).to(torch.int16).view(out.dtype).double().to(ref.device)
        a, c = (o + down) / 2, (o + up) / 2
        lo_c, hi_c = torch.minimum(a, c), torch.maximum(a, c)
        tiny = 2.0 ** (_FORMATS[out.dtype][1] - 1)
        lo_c = torch.where(zero, torch.full_like(o, -tiny), lo_c)
        hi_c = torch.where(zero, torch.full_like(o, tiny), hi_c)
        inf = torch.isinf(o)
        hi_c = torch.where(inf & (o > 0), o, hi_c)
        lo_c = torch.where(inf & (o < 0), o, lo_c)
        need = torch.clamp(torch.maximum(lo_c - ref, ref - hi_c), min=0)
    else:
        need = (o - ref).abs()
    return torch.where(need == 0, torch.zeros_like(need), need / b)


def within(out, ref, b):
    """bool tensor: out inside its bar, element by element"""
    lo, hi = corr_interval(ref, b, out.dtype)
    o = out.double().to(ref.device)
    return (o >= lo) & (o <= hi)


def corr_backward_bar(fmap1, fmap2, coords, ii, jj, grad, radius):
    """(g1, g2, b1, b2) for corr_bwd_generic with fp32 features: per element, the float64 gradients and the bars.
    Roundings on the way to a patch-feature element: BLEND for the tap gradient, D^2 taps, one add per pass and one
    atomic per edge of its patch slot; to a frame-feature element: BLEND, P^2 patch pixels per tap and, in the nine-pass
    fallback, P^2 atomics per edge of its frame slot"""
    B, M, _, P, _ = coords.shape
    D = 2 * radius + 2
    g = grad.double()
    a = fmap1.double().requires_grad_(True)
    c = fmap2.double().requires_grad_(True)
    (corr_forward(a, c, coords, ii, jj, radius) * g).sum().backward()
    aa = fmap1.double().abs().requires_grad_(True)
    cc = fmap2.double().abs().requires_grad_(True)
    (corr_forward(aa, cc, coords, ii, jj, radius) * g.abs()).sum().backward()
    n1 = BLEND + D * D + 1 + torch.bincount(ii.cpu(), minlength=fmap1.shape[1]).double()
    n2 = BLEND + P * P * (1 + torch.bincount(jj.cpu(), minlength=fmap2.shape[1]).double())
    n1, n2 = n1.to(a.device)[None, :, None, None, None], n2.to(a.device)[None, :, None, None, None]
    return a.grad, c.grad, gamma(n1) * aa.grad, gamma(n2) * cc.grad


def patchify_backward_bar(net, coords, grad, radius):
    """(g, b) for patchify_backward in fp32: every contribution to a feature element is one fp32 atomic"""
    x = net.double().requires_grad_(True)
    patchify_raw(x, coords, radius).backward(grad.double())
    xa = net.double().requires_grad_(True)
    patchify_raw(xa, coords, radius).backward(grad.double().abs())
    xn = net.double().requires_grad_(True)
    patchify_raw(xn, coords, radius).backward(torch.ones_like(grad, dtype=torch.float64))
    return x.grad, gamma(xn.grad) * xa.grad
