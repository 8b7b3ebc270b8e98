"""ORACLE (test infrastructure -- never imported by the product path).

The three fused layer chains of the update operator (csrc/chain.cu; net.py:74-92, blocks.py:15-29 of the reference)
restated in float64 at the kernels' own rounding points, with a per-element error bar of the kernels:

    A  dpvo_update_corr_norm     net = norm(net + inp[index] + corr.5(relu(corr.3(corr.2(relu(corr.0(corr)))))))
    C  dpvo_update_neighbor_mlp  net = net + c.2(relu(c.0(mask * x16[index])))              (c1 and c2)
    G  dpvo_update_gru_heads     net = gru(net + hkk[group_kk] + hij[group_of]),  delta = d(net) + centre,  weight = w(net)

Everything is read from an `Update` module's own submodules (corr[0, 2, 3, 5], norm, c1, c2, gru[0..3], d[1], w[1]),
while the kernels are fed `Update.pack()`'s A_* / C*_* / G_* blocks: a mistake in the packing shows as a mismatch.

Rounding points of the kernels, where the restatement rounds to fp16 (every other value is fp32 in the kernels and
exact here):
  - the weights of every dense layer; biases, LayerNorm gamma / beta and the head weights are fp32;
  - every GEMM operand: the inputs corr, x16 (C's gather source), the fp16 rows inp, hkk, hij; relu(corr.0), relu of
    corr.2's LayerNorm output, relu(c.0), gru.0's and gru.2's LayerNorm outputs, relu(res.0);
  - the gate: its pre-activation x Wg + bg is rounded to fp16, and so is the gate sigmoid(.) itself;
  - not rounded: corr.2's output before its LayerNorm, r2 = res.2's output, the residual x the gate multiplies into,
    the state; the heads run in fp32 on relu(net);
  - delta = the d head + coords[e, :, P // 2, P // 2] (the centre pixel of [E, 2, P, P] coords), or the head alone
    without coords.
Where the kernels depart from the reference's autocast (dpvo.py:332): there corr.2's output, r2 and the heads' outputs
are fp16 GEMM results; the kernels keep them in fp32.  tests/test_update_gpu.py remains the check against autocast.

`rounding=False` drops every rounding point (weights as they are, no fp16 anywhere): the restatement is then the
Update module's own arithmetic, which tests/test_chain_ref_cpu.py pins to oracle/update.py in float64.
"""
import copy

import torch

from .softagg import ACC, ulp16

DIM = 384
EPS = 1e-3
U = 2.0 ** -24                                   # fp32 unit roundoff (round to nearest)
# oracle/softagg.py's accumulator model (one fp32 rounding per k16 MMA step and one for the bias) at K = 896, the
# zero-padded correlation rows of corr.0: 56 k16 steps instead of 24
ACC_K0 = ACC * (896 // 16 + 1) / (384 // 16 + 1)
# the fp32 sum of a LayerNorm row: a value passes through at most 28 additions (its pair, 24 per thread in at most 6 + 2,
# 2 quad shuffles, the column-half exchange; 28 also bounds the former sequential 24) and the multiplication by the rounded 1/384
LN_SUM = 30 * U
# relative error of the row variance.  The kernels take S2 / 384 - mean^2 from one pass where 17 mean^2 <= S2 / 384:
# S2 is 28 additions deep (2 roundings per square), so its error is below 30 u S2 and mean^2's below 61 u mean^2, and
# the variance is at least 16/17 of S2 / 384: (30 + 61 / 17) 17 / 16 u < 36 u.  Elsewhere they take a second pass,
# M2 = sum (x - m)^2 about the first pass's fp32 mean m: 31 u (the difference, the square, 28 additions), plus
# n (m - mean)^2, whose relative size (LN_SUM mean|x| / std)^2 the bar carries as it stands
LN_VAR0 = 36 * U
# rsqrtf: 2 ulp (CUDA C Programming Guide, "Mathematical Functions", single precision)
RSQRT = 2.0 ** -22
# __expf: 2 + floor(|1.173 x|) ulp; __fdividef: 2 ulp for 2^-126 <= |y| <= 2^126 (same tables, "Intrinsic Functions")
FDIV = 2.0 ** -22
# tanh.approx.f16x2: absolute error 2^-11 (PTX ISA, tanh); the gate 0.5 + 0.5 t halves it
TANH = 2.0 ** -11


class Params:
    """float64 copies of an Update module's chain parameters: weights rounded to fp16, vectors to fp32 (`rounding`),
    or exactly as they are"""

    def __init__(self, upd, rounding=True, device=None):
        def W(lin):
            w = lin.weight.detach()
            return (w.half() if rounding else w).to(device).double()

        def v(t):
            t = t.detach()
            return (t.float() if rounding else t).to(device).double()
        self.rounding = rounding
        self.corr = [(W(upd.corr[i]), v(upd.corr[i].bias)) for i in (0, 2, 5)]
        if rounding and self.corr[0][0].shape[1] < 896:
            self.corr[0] = (torch.nn.functional.pad(self.corr[0][0], (0, 896 - self.corr[0][0].shape[1])), self.corr[0][1])
        self.ln_corr = (v(upd.corr[3].weight), v(upd.corr[3].bias))
        self.ln_norm = (v(upd.norm.weight), v(upd.norm.bias))
        self.c = {nm: [(W(m[i]), v(m[i].bias)) for i in (0, 2)] for nm, m in (("c1", upd.c1), ("c2", upd.c2))}
        self.ln_gru = [(v(upd.gru[i].weight), v(upd.gru[i].bias)) for i in (0, 2)]
        self.gr = [[(W(lin), v(lin.bias)) for lin in (blk.gate[0], blk.res[0], blk.res[2])] for blk in (upd.gru[1], upd.gru[3])]
        self.heads = (torch.cat([v(upd.d[1].weight), v(upd.w[1].weight)]), torch.cat([v(upd.d[1].bias), v(upd.w[1].bias)]))


class Arith:
    """The arithmetic a chain runs in.  Default: float64 at the kernels' rounding points (`rounding`), carrying the error
    bar (`bars`).  `emulate`: the kernels' own arithmetic in float32 on the CPU -- fp32 GEMM of the fp16 operands, the
    LayerNorm in the kernels' order (`ln_emulated`; with `one_pass`, the former S2/n - mean^2 on every row), the gate
    through a tanh rounded to fp16.  `eps` replaces the LayerNorm epsilon, and `flip` (a torch.Generator; float64 with
    bars) moves the value by a random -1, 0 or +1 ulp at every rounding point where the kernel's value could round the
    other way: both exist to test the bar."""

    def __init__(self, rounding=True, bars=True, emulate=False, one_pass=False, eps=EPS, flip=None):
        self.rnd, self.bars, self.emu, self.one_pass, self.eps, self.flip = rounding, bars and not emulate, emulate, one_pass, eps, flip
        self.dt = torch.float32 if emulate else torch.float64

    def t(self, x):
        return x.to(self.dt)

    def dense(self, x, e, W, b, acc=ACC):
        """x W^T + b, and its bar: the fp32 accumulator (acc sum_k |x_k W_k| + |b|, oracle/softagg.py's model) plus the
        input's bar through the layer, |W| e"""
        W, b = self.t(W), self.t(b)
        y = x @ W.t() + b
        if not self.bars:
            return y, None
        eb = acc * (x.abs() @ W.abs().t() + b.abs())
        return y, eb if e is None else eb + e @ W.abs().t()

    def r16(self, v, e):
        """an fp16 rounding point.  The kernel's fp32 value lies within the bar e of v, so it rounds to the same fp16
        value as v unless a rounding boundary (the midpoint between two neighbouring fp16 values) lies within e of v.
        Only there can the two differ, by at most e + the value's own ulp; everywhere else the rounding absorbs the
        error and the bar is 0.  An exact value (e None) rounds as v does.  `flip` moves the value by a random -1, 0 or
        +1 ulp at the points where the kernel's could round the other way."""
        if not self.rnd:
            return v, e
        v16 = v.half().to(self.dt)
        assert torch.isfinite(v16).all(), "a value at an fp16 rounding point is outside the fp16 range"
        if not self.bars or e is None:
            return v16, None
        a, a16 = v.abs(), v16.abs().double()
        up, down = ulp16(a16), ulp16(a16 * (1 - 2.0 ** -13))     # fp16 spacing above and below |v16|
        near = torch.minimum((a - (a16 + up / 2)).abs(), (a - (a16 - down / 2)).abs()) <= e
        if self.flip is not None:
            s = torch.randint(-1, 2, v16.shape, generator=self.flip).to(v16.device, self.dt)
            v16 = torch.where(near, v16 + s * ulp16(v16.double()).to(self.dt), v16)
        return v16, torch.where(near, e + ulp16(a + e), torch.zeros_like(e))

    def add32(self, y, e, x):
        """y + x in fp32: one rounding of the sum"""
        s = y + self.t(x)
        if not self.bars:
            return s, None
        return s, (0 if e is None else e) + U * s.abs()

    def ln(self, x, e, g, b):
        """nn.LayerNorm(eps).  Bar, first order in the input's bar e:
              |g| rstd (|e| + mean|e| + |xh| mean(|xh| |e|))
           plus the fp32 arithmetic of the kernels' mean and variance (one pass, or two where the mean dominates):
              |g| rstd LN_SUM mean|x|                     the mean
              (RSQRT + 2u + (LN_VAR0 + (LN_SUM mean|x| rstd)^2) / 2) |g xh|   rstd: rsqrtf, the eps add and 1/384,
                                                          half the variance's relative error
              4u |g xh| + u |y|                           x - mean, * rstd, * g, + b
           The terms left out are of second order in e rstd and in the relative errors above; they are negligible where
           the bar is used, e << sqrt(var + eps) (the first-order terms are then already a small fraction of |g|)."""
        if self.emu:
            return ln_emulated(x, g, b, self.one_pass, self.eps), None
        m = x.mean(-1, keepdim=True)
        c = x - m
        r = 1.0 / torch.sqrt((c * c).mean(-1, keepdim=True) + self.eps)
        xh = c * r
        y = xh * g + b
        if not self.bars:
            return y, None
        ax = x.abs().mean(-1, keepdim=True)
        gx = (xh * g).abs()
        B = g.abs() * r * LN_SUM * ax + (RSQRT + 2 * U + 0.5 * (LN_VAR0 + (LN_SUM * ax * r) ** 2) + 4 * U) * gx + U * y.abs()
        if e is not None:
            B = B + g.abs() * r * (e + e.mean(-1, keepdim=True) + xh.abs() * (xh.abs() * e).mean(-1, keepdim=True))
        return y, B

    def relu(self, v, e):
        return v.clamp(min=0), e                                     # 1-Lipschitz

    def gate(self, a, e):
        """sigmoid of the fp16 pre-activation, as fp16: the pre-activation's bar and rounding through sigmoid's 1/4
        Lipschitz bound, tanh.approx's error halved, the gate's own fp16 rounding"""
        if self.emu:                                                 # 0.5 + 0.5 tanh(fp16(a / 2)), tanh as fp16
            t = torch.tanh((0.5 * a).half().float()).half().float()
            return (0.5 * t + 0.5).half().float(), None
        a, e = self.r16(a, e)
        g = torch.sigmoid(a)
        if not self.rnd:
            return g, None
        return self.r16(g, None if not self.bars else 0.25 * (0 if e is None else e) + TANH / 2)


def chain_a(P, corr16, net32, inp16, inp_index=None, ar=None):
    """chain A: (net [E, 384], bar).  corr16 [E, 882 or 896], net32 [E, 384], inp16 [n, 384] (row inp_index[e], or e)"""
    ar = ar or Arith(P.rounding)
    (W0, b0), (W2, b2), (W5, b5) = P.corr
    x = ar.t(corr16.reshape(-1, corr16.shape[-1]))
    x = x[:, :W0.shape[1]] if x.shape[1] >= W0.shape[1] else torch.nn.functional.pad(x, (0, W0.shape[1] - x.shape[1]))
    h, e = ar.r16(*ar.relu(*ar.dense(x, None, W0, b0, ACC_K0)))
    h, e = ar.dense(h, e, W2, b2)
    h, e = ar.r16(*ar.relu(*ar.ln(h, e, *P.ln_corr)))
    y, e = ar.dense(h, e, W5, b5)
    y, e = ar.add32(y, e, net32.reshape(-1, DIM))
    inp = inp16.reshape(-1, DIM)
    y, e = ar.add32(y, e, inp if inp_index is None else inp[inp_index.long()])
    return ar.ln(y, e, *P.ln_norm)


def chain_c(P, which, x16, index, net32, ar=None):
    """chain C (`which` = "c1" or "c2"): (net [E, 384], bar).  Row e gathers x16[index[e]], or zeros where index < 0"""
    ar = ar or Arith(P.rounding)
    (Wa, ba), (Wb, bb) = P.c[which]
    idx = index.long()
    x = ar.t(x16.reshape(-1, DIM))[idx.clamp(min=0)] * ar.t(idx >= 0)[:, None]
    h, e = ar.r16(*ar.relu(*ar.dense(x, None, Wa, ba)))
    y, e = ar.dense(h, e, Wb, bb)
    return ar.add32(y, e, net32.reshape(-1, DIM))


def chain_g(P, net32, hij16=None, group_of=None, hkk16=None, group_kk=None, coords=None, ar=None):
    """chain G: (net, bar), (delta [E, 2], bar), (weight [E, 2], bar)"""
    ar = ar or Arith(P.rounding)
    x, e = ar.t(net32.reshape(-1, DIM)), None
    for tab, gid in ((hkk16, group_kk), (hij16, group_of)):          # the kernel's order: state, hkk, hij
        if tab is not None:
            x, e = ar.add32(x, e, tab.reshape(-1, DIM)[gid.long()])
    x, e = ar.ln(x, e, *P.ln_gru[0])
    for blk in range(2):
        (Wg, bg), (Wa, ba), (Wb, bb) = P.gr[blk]
        x16, e16 = ar.r16(x, e)
        g, eg = ar.gate(*ar.dense(x16, e16, Wg, bg))
        r, er = ar.r16(*ar.relu(*ar.dense(x16, e16, Wa, ba)))
        r, er = ar.dense(r, er, Wb, bb)
        v = x + g * r
        if ar.bars:                                                  # x + g r in fp32: two roundings, or one if fused
            e = e + g.abs() * er + r.abs() * eg + eg * er + 2 * U * (x.abs() + (g * r).abs())
        x = v
        if blk == 0:
            x, e = ar.ln(x, e, *P.ln_gru[1])
    W4, b4 = ar.t(P.heads[0]), ar.t(P.heads[1])
    rx = x.clamp(min=0)
    hd = rx @ W4.t() + b4
    ctr = torch.zeros_like(hd[:, :2]) if coords is None else ar.t(centre(coords))
    delta, weight = hd[:, :2] + ctr, torch.sigmoid(hd[:, 2:])
    if not ar.bars:
        return (x, None), (delta, None), (weight, None)
    # the heads' fp32 dot products: a product passes through at most 24 additions per thread, 2 shuffles, the
    # column-half exchange, the bias (and for delta the centre): 29 roundings of partial sums <= sum |x W| + |b| + |ctr|
    mag = rx @ W4.abs().t() + b4.abs()
    ez = e @ W4.abs().t() + 29 * U * mag
    ed = ez[:, :2] + 29 * U * ctr.abs()
    # weight = __fdividef(1, 1 + __expf(-z)): through sigmoid's 1/4 Lipschitz bound; w (1 - w) times __expf's relative
    # error; the rounding of 1 + e and __fdividef's 2 ulp, relative to w
    z, w = hd[:, 2:], weight
    ew = 0.25 * ez[:, 2:] + w * (1 - w) * (2 + torch.floor(1.173 * z.abs())) * 2.0 ** -23 + w * (U + FDIV)
    return (x, e), (delta, ed), (weight, ew)


def ln_emulated(x, g, b, one_pass=False, eps=EPS):
    """the kernels' LayerNorm in float32 on [rows, 384] x, in their reduction order: per column half h and quad lane l
    the 48 columns h 192 + 8 j + 2 l + {0, 1} summed in order, the 4 lanes of a quad by two shuffles (^1, ^2), the two
    halves last.  One pass gives S and S2; the 16 rows of a warp pair (rows 16 k .. 16 k + 15 of the launch) take the
    second pass, M2 about the first pass's mean, when one of them has 17 mean^2 > S2 / 384.  `one_pass` is the former
    form: S2 / 384 - mean^2 everywhere"""
    x, dev = x.float(), x.device
    rows = x.shape[0]
    cols = torch.tensor([[h * 192 + 8 * j + 2 * l + k for j in range(24) for k in (0, 1)] for h in (0, 1) for l in range(4)], device=dev)
    part = x[:, cols].reshape(rows, 2, 4, 48)                       # [rows, half, quad lane, 48]
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)

    def reduce(terms):                                               # terms [rows, 2, 4, 24]: per-thread order, quad, halves
        t = x.new_zeros(rows, 2, 4)
        for j in range(terms.shape[-1]):
            t = t + terms[..., j]
        for o in (1, 2):
            t = t + t[:, :, [l ^ o for l in range(4)]]
        return t[:, 0, 0] + t[:, 1, 0]

    t0, t1 = part[..., 0::2], part[..., 1::2]
    mean = reduce(t0 + t1) * f32(1.0 / DIM)
    ms = reduce(t0 * t0 + t1 * t1) * f32(1.0 / DIM)
    var = ms - mean * mean
    if not one_pass:
        again = 17 * (mean * mean) > ms
        again = torch.nn.functional.pad(again, (0, -rows % 16)).reshape(-1, 16).any(1).repeat_interleave(16)[:rows]
        d0, d1 = t0 - mean[:, None, None, None], t1 - mean[:, None, None, None]
        var = torch.where(again, reduce(d0 * d0 + d1 * d1) * f32(1.0 / DIM), var)
    rstd = torch.rsqrt(var.clamp(min=0) + f32(eps))[:, None]
    return (x - mean[:, None]) * rstd * g.float() + b.float()


# The per-element bar is a worst case over the signs of the rounding errors, carried through each layer as |W| bar; across
# several 384-wide layers and the LayerNorms that rescale them it can grow far past what rounding does in practice.  The
# tests therefore also hold every output to the max-norm tolerance of rel * max(max |ref|, 1) (delta: of the head alone),
# which the float32 emulation meets with at least 10x to spare in every regime of the tests
MAX_NORM = {"A": 2e-3, "C": 2e-3, "G": 3e-3}


def capped(bar, ref, rel):
    """the bar, but nowhere above the max-norm tolerance rel * max(max |ref|, 1)"""
    return bar.clamp(max=rel * max(ref.abs().max().item(), 1.0))


def outputs_capped(chain, outs, coords=None):
    """[(ref, bar)] of a chain (A, C: the state; G: state, delta, weight) with each bar capped by MAX_NORM[chain]"""
    rel = MAX_NORM[chain]
    res = []
    for k, (v, b) in enumerate(outs):
        head = v - centre(coords).to(v) if chain == "G" and k == 1 and coords is not None else v
        res.append((v, capped(b, head, rel)))
    return res


def centre(coords):
    """coords [E, 2, P, P] -> the centre pixel [E, 2] (index (P // 2) P + P // 2 of the flattened patch)"""
    pp = coords.shape[-1]
    return coords.reshape(-1, 2, pp * pp)[:, :, (pp // 2) * pp + pp // 2]


# ------------------------------------------------------------------ test cases: modules, inputs and value regimes
def module(seed, cls, dev):
    """an Update with every parameter random: nn.Linear's own initialisation, LayerNorm gamma of either sign and 0.4 to
    1.6 in size (away from 1), beta ~ 0.5 N(0, 1)"""
    torch.manual_seed(seed)
    upd = cls()
    with torch.no_grad():
        for ln in (upd.corr[3], upd.norm, upd.gru[0], upd.gru[2]):
            g = torch.rand(DIM) * 1.2 + 0.4
            ln.weight.copy_(torch.where(torch.rand(DIM) < 0.2, -g, g))
            ln.bias.copy_(torch.randn(DIM) * 0.5)
    return upd.to(dev).eval()


def _max_abs(x):
    return max(float(x.abs().max()), 1e-30)


def case_a(upd, E, dev, regime="nominal", variant="index", seed=0):
    """(module, corr [E, 896] fp16 (a view with row stride > 896 for variant "stride"), net32, inp16, inp_index)"""
    g = torch.Generator(device=dev).manual_seed(1000 * seed + E)
    upd = copy.deepcopy(upd)
    corr = torch.zeros(E, 896, device=dev, dtype=torch.half)
    corr[:, :882] = torch.randn(E, 882, generator=g, device=dev).half()
    net = torch.randn(E, DIM, generator=g, device=dev)
    n_ctx = max(1, E // 20)
    inp = torch.randn(n_ctx if variant == "index" else E, DIM, generator=g, device=dev).half()
    idx = torch.randint(0, n_ctx, (E,), generator=g, device=dev) if variant == "index" else None
    with torch.no_grad():
        if regime.startswith("offset"):                              # offset<m>/<s>: state rows m + s N(0, 1)
            m, s = (float(t) for t in regime[6:].split("/"))
            net = m * torch.sign(torch.randn(E, 1, generator=g, device=dev)) + s * net
            # the correlation branch and the context well below the spread s, so that the state's offset decides
            upd.corr[5].weight.mul_(1e-3 * s)
            upd.corr[5].bias.mul_(1e-3 * s)
            inp = (inp.float() * 1e-3 * s).half()
        elif regime.startswith("innerbias"):                         # corr.2's output offset ahead of its LayerNorm
            upd.corr[2].bias.add_(float(regime[9:]))
            net = net * 1e-2
        elif regime == "constant":                                   # both LayerNorms on rows of one value: rstd = 1/sqrt(eps)
            upd.corr[2].weight.zero_()
            upd.corr[2].bias.fill_(0.75)
            upd.corr[5].weight.zero_()
            upd.corr[5].bias.zero_()
            inp.zero_()
            net = (torch.randint(-64, 64, (E, 1), generator=g, device=dev).float() / 8).expand(E, DIM).contiguous()
        elif regime == "large":                                      # corr.0's output and corr.3's up to ~2.5e4
            P = Params(upd, device=dev)
            a = Arith(bars=False)
            h0 = corr.double() @ P.corr[0][0].t() + P.corr[0][1]
            corr = (corr.float() * (2.5e4 / _max_abs(h0))).half()
            h = a.dense(a.r16(*a.relu(*a.dense(corr.double(), None, *P.corr[0])))[0], None, *P.corr[1])[0]
            s = 2.5e4 / _max_abs(a.ln(h, None, *P.ln_corr)[0])
            upd.corr[3].weight.mul_(s)
            upd.corr[3].bias.mul_(s)
        elif regime == "deadrelu":                                   # every third row: corr.0 all negative
            upd.corr[0].bias.copy_(-upd.corr[0].bias.abs() - 0.05)
            corr[::3] = 0
        else:
            assert regime == "nominal", regime
    if variant == "stride":                                          # row stride 1024, finite garbage past column 882
        wide = torch.randn(E, 1024, generator=g, device=dev).half()
        wide[:, :896] = corr
        corr = wide[:, :896]
    return upd, corr, net, inp, idx


def case_c(upd, E, dev, regime="nominal", variant="mixed", which="c1", seed=0):
    g = torch.Generator(device=dev).manual_seed(1000 * seed + E + 1)
    upd = copy.deepcopy(upd)
    x16 = torch.randn(E, DIM, generator=g, device=dev).half()
    net = torch.randn(E, DIM, generator=g, device=dev)
    idx = {"mixed": lambda: torch.randint(-1, E, (E,), generator=g, device=dev),
           "all_masked": lambda: torch.full((E,), -1, device=dev),
           "none_masked": lambda: torch.randint(0, E, (E,), generator=g, device=dev),
           "self": lambda: torch.arange(E, device=dev),
           "row0": lambda: torch.zeros(E, dtype=torch.long, device=dev),
           "rowlast": lambda: torch.full((E,), E - 1, device=dev)}[variant]()
    if variant == "mixed":
        idx[::7] = -1
    mlp = getattr(upd, which)
    with torch.no_grad():
        if regime.startswith("offset"):
            m, s = (float(t) for t in regime[6:].split("/"))
            net = m * torch.sign(torch.randn(E, 1, generator=g, device=dev)) + s * net
        elif regime == "large":                                      # the hidden layer's output up to ~2.5e4
            Wa = Params(upd, device=dev).c[which][0][0]
            s = 2.5e4 / _max_abs(x16.double() @ Wa.t())
            x16 = (x16.float() * min(s, 2.0e4 / _max_abs(x16.float()))).half()
        elif regime == "deadrelu":                                   # every third source row zero, c.0's bias negative
            mlp[0].bias.copy_(-mlp[0].bias.abs() - 0.05)
            x16[::3] = 0
        else:
            assert regime == "nominal", regime
    return upd, which, x16, idx, net


def case_g(upd, E, dev, regime="nominal", groups="both", P=3, gid="random", coords=True, seed=0):
    g = torch.Generator(device=dev).manual_seed(1000 * seed + E + 2)
    upd = copy.deepcopy(upd)
    net = torch.randn(E, DIM, generator=g, device=dev)
    G1, G2 = max(1, E // 90), max(1, E // 22)
    hij = (torch.randn(G1, DIM, generator=g, device=dev) * 0.5).half()
    hkk = (torch.randn(G2, DIM, generator=g, device=dev) * 0.5).half()
    pick = {"random": lambda n: torch.randint(0, n, (E,), generator=g, device=dev, dtype=torch.int32),
            "zero": lambda n: torch.zeros(E, device=dev, dtype=torch.int32),
            "max": lambda n: torch.full((E,), n - 1, device=dev, dtype=torch.int32)}[gid]
    gof, gkk = pick(G1), pick(G2)
    cd = torch.randn(E, 2, P, P, generator=g, device=dev) * 50 if coords else None
    with torch.no_grad():
        if regime.startswith("offset"):
            m, s = (float(t) for t in regime[6:].split("/"))
            net = m * torch.sign(torch.randn(E, 1, generator=g, device=dev)) + s * net
            hij, hkk = (hij.float() * 1e-3 * s).half(), (hkk.float() * 1e-3 * s).half()
            # both gates closed (pre-activation <= -20: the gate is 0): net is gru.2's LayerNorm of gru.0's, and the
            # gated branches' rounding does not cover the LayerNorms' arithmetic
            for blk in (upd.gru[1], upd.gru[3]):
                blk.gate[0].bias.fill_(-40.0)
        elif regime.startswith("innerbias"):                         # gru.2's input offset by m: gru.0's beta + m
            upd.gru[0].bias.add_(float(regime[9:]))
            for blk in (upd.gru[1], upd.gru[3]):                     # the residual branches small against the offset,
                blk.res[0].weight.mul_(1e-3)                         # so that the gates' tanh.approx error (2^-12 of
            upd.gru[3].gate[0].bias.fill_(-40.0)                     # r2) stays below the spread; net = gru.2's output
        elif regime == "constant":                                   # gru.0 on rows of one value
            groups = "none"
            net = (torch.randint(-64, 64, (E, 1), generator=g, device=dev).float() / 8).expand(E, DIM).contiguous()
        elif regime == "large":                                      # gru.0's and gru.2's outputs up to ~2.5e4
            for i, blk in ((0, upd.gru[1]), (2, upd.gru[3])):
                ln = upd.gru[i]
                s = 2.5e4 / (19.6 * float(ln.weight.abs().max()) + float(ln.bias.abs().max()))
                ln.weight.mul_(s)
                ln.bias.mul_(s)
                blk.gate[0].weight.div_(s)
                blk.res[0].weight.div_(s)
        elif regime == "deadrelu":                                   # res.0's ReLU dead in both blocks
            for blk in (upd.gru[1], upd.gru[3]):
                blk.res[0].bias.fill_(-50.0)
        elif regime == "satgate":                                    # |gate pre-activation| >= 20, both signs
            for blk in (upd.gru[1], upd.gru[3]):
                blk.gate[0].bias.copy_(torch.where(torch.arange(DIM, device=dev) % 2 == 0, 40.0, -40.0))
        elif regime == "satlogit":                                   # weight logits near +-100
            upd.w[1].bias.copy_(torch.tensor([100.0, -100.0], device=dev))
            upd.w[1].weight.mul_(1e-2)
        else:
            assert regime == "nominal", regime
    hij_, gof_ = (hij, gof) if groups in ("both", "hij") else (None, None)
    hkk_, gkk_ = (hkk, gkk) if groups in ("both", "hkk") else (None, None)
    return upd, net, hij_, gof_, hkk_, gkk_, cd
