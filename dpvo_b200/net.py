"""The recurrent update operator (dpvo/net.py:27-92, dpvo/blocks.py:15-48) on sm_90a kernels.

`Update` keeps the reference's sub-module names, so a DPVO checkpoint's "update.*" state_dict keys
load unchanged (update.c1.0.weight, update.agg_kk.f.weight, update.gru.1.gate.0.weight, ...).

Inference forward = 17 dense layers + fused row kernels:
    corr MLP 882->384->384->LN->384 | LN(net+inp+.) | c1,c2 on masked temporal neighbours |
    SoftAgg over patches (kk) and over frame pairs (ii,jj) | 2x (LN, gated residual) | heads
Data flow is fp32 for the carried state `net`, fp16 for every GEMM operand (what the reference's
autocast does, dpvo.py:332), with the fp16 copies produced inside the fused row kernels.  The edge
groupings come from ONE device radix-sort launch each (no host sync, no torch.unique, no D2H sort).

Every dense layer runs on hand-written wgmma kernels (csrc/chain.cu: the three fused layer chains; csrc/softagg.cu:
each SoftAgg's f|g layer fused with its segment softmax; csrc/gemm.cu: dpvo_linear_f16 for the two SoftAgg h layers);
there is no library GEMM and no other backend.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import extensions

DIM = 384
CORR_PAD = 896      # 2*49*9 = 882 correlation features rounded up to a multiple of 64


class GradClip(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return x

    @staticmethod
    def backward(ctx, g):
        g = torch.where(torch.isnan(g), torch.zeros_like(g), g)
        return g.clamp(min=-0.01, max=0.01)


class GradientClip(nn.Module):
    def forward(self, x):
        return GradClip.apply(x)


class GatedResidual(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.gate = nn.Sequential(nn.Linear(dim, dim), nn.Sigmoid())
        self.res = nn.Sequential(nn.Linear(dim, dim), nn.ReLU(inplace=True), nn.Linear(dim, dim))

    def forward(self, x):
        return x + self.gate(x) * self.res(x)


class SoftAgg(nn.Module):
    """blocks.py:31-48.  Inference: parameters only, f|g and the reduction run in dpvo_softagg_fused.  Training:
    `forward(x, group_of, n_groups)` is the differentiable fp32 form -- a per-group softmax of g(x) weighting f(x),
    summed per group, mapped by h and handed back to every member; group ids come from the device grouping kernel
    (no torch.unique), the per-group max / sums are index reductions."""

    def __init__(self, dim=512, expand=True):
        super().__init__()
        self.dim, self.expand = dim, expand
        self.f = nn.Linear(dim, dim)
        self.g = nn.Linear(dim, dim)
        self.h = nn.Linear(dim, dim)

    def forward(self, x, group_of, n_groups):
        logits = self.g(x)
        idx = group_of.view(1, -1, 1).expand_as(logits)
        top = torch.full((x.shape[0], n_groups, x.shape[2]), float("-inf"), dtype=x.dtype, device=x.device)
        top = top.scatter_reduce(1, idx, logits.detach(), reduce="amax", include_self=True)
        e = torch.exp(logits - top[:, group_of])               # the shift cancels in the ratio: no gradient through it
        den = torch.zeros_like(top).index_add_(1, group_of, e)
        y = torch.zeros_like(top).index_add_(1, group_of, self.f(x) * (e / den[:, group_of]))
        y = self.h(y)
        return y[:, group_of] if self.expand else y


class EdgeGroups:
    """Device-resident CSR of an edge grouping (dpvo_group_edges); G bounds are host hints."""

    def __init__(self, key_a, key_b=None, sec=None, max_groups=None, _fields=None):
        if _fields is None:
            _fields = extensions()[3].group_edges(key_a, key_b, sec)
        self.order, self.group_of, self.group_start, self.key_a, self.key_b, self.n = _fields
        # `max_groups` sizes the per-group buffers.  Callers that know a bound (UpdateRunner: patch slots, frame
        # pairs) pass it and nothing ever leaves the device; without one the count is read back (one sync -- the
        # reference's torch.unique in blocks.py:41 synchronises too).
        self.max_groups = int(self.n.item()) if max_groups is None else int(max_groups)

    @classmethod
    def pair(cls, spec0, spec1, max_groups0=None, max_groups1=None):
        """both groupings of an update -- spec = (key_a, key_b, sec) -- in one cooperative launch; missing bounds
        are read back together (a single device->host copy for both)"""
        f = extensions()[3].group_edges_pair(*spec0, *spec1)
        if max_groups0 is None or max_groups1 is None:
            n0, n1 = torch.stack([f[5].reshape(()), f[11].reshape(())]).tolist()
            max_groups0 = n0 if max_groups0 is None else max_groups0
            max_groups1 = n1 if max_groups1 is None else max_groups1
        return cls(None, max_groups=max_groups0, _fields=f[:6]), cls(None, max_groups=max_groups1, _fields=f[6:])


class Update(nn.Module):
    def __init__(self, p=3):
        super().__init__()
        self.c1 = nn.Sequential(nn.Linear(DIM, DIM), nn.ReLU(inplace=True), nn.Linear(DIM, DIM))
        self.c2 = nn.Sequential(nn.Linear(DIM, DIM), nn.ReLU(inplace=True), nn.Linear(DIM, DIM))
        self.norm = nn.LayerNorm(DIM, eps=1e-3)
        self.agg_kk = SoftAgg(DIM)
        self.agg_ij = SoftAgg(DIM)
        self.gru = nn.Sequential(nn.LayerNorm(DIM, eps=1e-3), GatedResidual(DIM),
                                 nn.LayerNorm(DIM, eps=1e-3), GatedResidual(DIM))
        self.corr = nn.Sequential(nn.Linear(2 * 49 * p * p, DIM), nn.ReLU(inplace=True), nn.Linear(DIM, DIM),
                                  nn.LayerNorm(DIM, eps=1e-3), nn.ReLU(inplace=True), nn.Linear(DIM, DIM))
        self.d = nn.Sequential(nn.ReLU(inplace=False), nn.Linear(DIM, 2), GradientClip())
        self.w = nn.Sequential(nn.ReLU(inplace=False), nn.Linear(DIM, 2), GradientClip(), nn.Sigmoid())
        self.inplace_state = False     # True: forward() overwrites an fp32 `net` argument with the new state
        self._packed = None
        self._packed_key = None

    # The packed fp16 copies follow the parameters: any in-place change (load_state_dict, an optimiser step) bumps
    # the parameters' version counters, .to()/.cuda() replaces their storage -- both change this key.
    def _param_key(self):
        return tuple((p.data_ptr(), p._version, p.device) for p in self.parameters())

    def packed(self):
        key = self._param_key()
        if self._packed is None or self._packed_key != key:
            self.pack()
            self._packed_key = key
        return self._packed

    # ------------------------------------------------------------------ packed inference weights
    def pack(self):
        """fp16 copies of the dense weights (+ fp32 biases) for the inference path (rebuilt by `packed()` whenever
        the parameters changed)."""
        def lin(m):
            return (m.weight.detach().half().contiguous(), m.bias.detach().float().contiguous())
        P = {}
        P["corr0"], P["corr2"], P["corr5"] = lin(self.corr[0]), lin(self.corr[2]), lin(self.corr[5])
        # the first dense layer consumes correlation rows padded from 882 to 896 columns (one 64-wide
        # k-block of the wgmma kernel); the extra weight columns are zero
        w0, b0 = P["corr0"]
        P["corr0"] = (F.pad(w0, (0, CORR_PAD - w0.shape[1])).contiguous(), b0)
        P["c1a"], P["c1b"], P["c2a"], P["c2b"] = lin(self.c1[0]), lin(self.c1[2]), lin(self.c2[0]), lin(self.c2[2])
        for nm, agg in (("kk", self.agg_kk), ("ij", self.agg_ij)):
            # f and g stacked for one linear_f16 with N = 768: the two-kernel form (linear_f16 + softagg_reduce) that the
            # fused op is tested and timed against
            P["fg_" + nm] = (torch.cat([agg.f.weight, agg.g.weight], 0).detach().half().contiguous(),
                             torch.cat([agg.f.bias, agg.g.bias], 0).detach().float().contiguous())
            # dpvo_softagg_fused: the f and g rows interleaved by 96-channel slice, [f 0..95; g 0..95; f 96..191; ...]
            def il(f, g):
                return torch.stack([f.reshape(DIM // 96, 96, -1), g.reshape(DIM // 96, 96, -1)], 1).reshape(2 * DIM, -1).detach()
            P["fgi_" + nm] = (il(agg.f.weight, agg.g.weight).half().contiguous(), il(agg.f.bias, agg.g.bias).reshape(-1).float().contiguous())
            P["h_" + nm] = lin(agg.h)
        for i, blk in ((1, self.gru[1]), (3, self.gru[3])):
            P["gr%d_g" % i], P["gr%d_a" % i], P["gr%d_b" % i] = lin(blk.gate[0]), lin(blk.res[0]), lin(blk.res[2])
            # gate and first residual layer share their input: one GEMM with N = 768 (sigmoid | relu halves)
            (wg, bg), (wa, ba) = P["gr%d_g" % i], P["gr%d_a" % i]
            P["gr%d_ga" % i] = (torch.cat([wg, wa], 0).contiguous(), torch.cat([bg, ba], 0).contiguous())
        # fused layer chains (csrc/chain.cu): stacked fp16 weights and one fp32 parameter block per chain
        def f32cat(*ts):
            return torch.cat([t.detach().float().reshape(-1) for t in ts]).contiguous()
        P["A_W0"] = P["corr0"][0]
        P["A_W25"] = torch.cat([P["corr2"][0], P["corr5"][0]], 0).contiguous()
        P["A_p"] = f32cat(self.corr[0].bias, self.corr[2].bias, self.corr[3].weight, self.corr[3].bias, self.corr[5].bias,
                          self.norm.weight, self.norm.bias)
        for nm, mlp in (("C1", self.c1), ("C2", self.c2)):
            P[nm + "_W"] = torch.cat([mlp[0].weight, mlp[2].weight], 0).detach().half().contiguous()
            P[nm + "_p"] = f32cat(mlp[0].bias, mlp[2].bias)
        g1, g3 = self.gru[1], self.gru[3]
        P["G_W6"] = torch.cat([g1.gate[0].weight, g1.res[0].weight, g1.res[2].weight,
                               g3.gate[0].weight, g3.res[0].weight, g3.res[2].weight], 0).detach().half().contiguous()
        P["G_p"] = f32cat(self.gru[0].weight, self.gru[0].bias, g1.gate[0].bias, g1.res[0].bias, g1.res[2].bias,
                          self.gru[2].weight, self.gru[2].bias, g3.gate[0].bias, g3.res[0].bias, g3.res[2].bias,
                          self.d[1].weight, self.w[1].weight, self.d[1].bias, self.w[1].bias)
        P["heads_w"] = torch.cat([self.d[1].weight, self.w[1].weight], 0).detach().float().contiguous()
        P["heads_b"] = torch.cat([self.d[1].bias, self.w[1].bias], 0).detach().float().contiguous()
        self._packed = P
        return P

    # ------------------------------------------------------------------------------- training forward
    def forward_train(self, net, inp, corr, flow, ii, jj, kk):
        """Differentiable fp32 form of net.py:74-92 (training runs without autocast, net.py:187): torch dense layers
        and LayerNorm with autograd, the temporal neighbours from our cuda_ba.neighbors kernel, both aggregations
        on groupings built by one launch of the device radix sort.  Same parameters, same arithmetic order as the
        reference module, so losses and gradients are comparable at fp32 round-off (tests/test_train_gpu.py)."""
        net = self.norm(net + inp + self.corr(corr))
        ix, jx = extensions()[1].neighbors(kk, jj)
        for idx, mlp in ((ix, self.c1), (jx, self.c2)):
            live = (idx >= 0).to(net.dtype).view(1, -1, 1)
            net = net + mlp(live * net[:, idx])
        gk, gp = EdgeGroups.pair((kk, None, jj), (ii, jj, None))
        net = net + self.agg_kk(net, gk.group_of.long(), gk.max_groups)
        net = net + self.agg_ij(net, gp.group_of.long(), gp.max_groups)
        net = self.gru(net)
        return net, (self.d(net), self.w(net), None)

    # ------------------------------------------------------------------------------- forward
    def forward(self, net, inp, corr, flow, ii, jj, kk, groups_kk=None, groups_ij=None, inp_index=None, coords=None):
        """training mode with autograd enabled -> the differentiable fp32 path; otherwise the fused inference kernels"""
        if self.training and torch.is_grad_enabled():
            return self.forward_train(net, inp, corr, flow, ii, jj, kk)
        with torch.no_grad():
            return self.forward_infer(net, inp, corr, flow, ii, jj, kk, groups_kk, groups_ij, inp_index, coords)

    def forward_infer(self, net, inp, corr, flow, ii, jj, kk, groups_kk=None, groups_ij=None, inp_index=None, coords=None):
        """net [1,E,384] (fp16 or fp32), inp [1,E,384], corr [1,E,882 or 896], ii/jj/kk int64 [E].
        Returns (net fp32, (delta [1,E,2], weight [1,E,2], None)) like net.py:92.
        Optional fusions for the inference loop: `inp_index` -- `inp` is the whole context table and row
        e uses inp[inp_index[e]] (dpvo.py:334); `coords` [1,E,2,P,P] -- `delta` is returned as the BA
        target coords[..., P//2, P//2] + delta (dpvo.py:341)."""
        self._inp_index, self._coords = inp_index, coords
        corr = corr if corr.dtype == torch.half else corr.half()
        if corr.shape[-1] != CORR_PAD:
            corr = F.pad(corr, (0, CORR_PAD - corr.shape[-1]))
        inp = inp if inp.dtype in (torch.half, torch.float32) else inp.half()
        if groups_kk is None and groups_ij is None:
            groups_kk, groups_ij = EdgeGroups.pair((kk, None, jj), (ii, jj, None))
        elif groups_kk is None:
            groups_kk = EdgeGroups(kk, None, jj)
        elif groups_ij is None:
            groups_ij = EdgeGroups(ii, jj, None)
        return self._forward_chains(net, inp, corr, groups_kk, groups_ij)

    def _forward_chains(self, net, inp, corr, groups_kk, groups_ij):
        """The row-local stretches of net.py:74-92 as one wgmma chain kernel each (csrc/chain.cu): corr MLP + context
        add + LayerNorm; c1 and c2 on the masked temporal neighbours; group add + GRU + heads.  Between them only the two
        SoftAgg aggregations (which mix rows of a group) run as separate kernels."""
        ex = extensions()[3]
        P = self.packed()
        inplace = net.dtype == torch.float32 and net.is_contiguous() and self.inplace_state
        net32 = net if inplace else net.float().contiguous().clone()
        inp16 = inp if inp.dtype == torch.half else inp.half()
        inp16 = inp16.reshape(-1, DIM).contiguous()
        gev = getattr(self, "gemm_events", None)          # bench.py: CUDA events around every tensor-core launch

        def timed(f, *args):
            if gev is None:
                return f(*args)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = f(*args)
            e1.record()
            gev.append((e0, e1))
            return y

        def L(x, name):
            return timed(ex.linear_f16, x, P[name][0], P[name][1], 0)
        n16 = timed(ex.update_corr_norm, corr, P["A_W0"], P["A_W25"], P["A_p"], net32, inp16, self._inp_index)
        ix, jx = ex.neighbors_from_groups(groups_kk.order, groups_kk.group_of)
        n16b = timed(ex.update_neighbor_mlp, n16, ix, P["C1_W"], P["C1_p"], net32)
        n16 = timed(ex.update_neighbor_mlp, n16b, jx, P["C2_W"], P["C2_p"], net32, n16)
        def agg(x, grp, name):                            # the f|g layer and its segment softmax in one op
            return timed(ex.softagg_fused, x, grp.order, grp.group_of, grp.group_start, grp.n, grp.max_groups, *P[name])
        y = agg(n16, groups_kk, "fgi_kk")
        # net + agg_kk(net) is only needed as the fp16 operand of the next aggregation; the fp32 state itself takes both
        # aggregation results in the prologue of the GRU chain (net.py:87-88), one pass over the state instead of two
        h_kk = L(y, "h_kk").reshape(-1, DIM)
        n16 = ex.residual_sum16(net32, h_kk, groups_kk.group_of)
        y = agg(n16, groups_ij, "fgi_ij")
        h_ij = L(y, "h_ij")
        delta, weight = timed(ex.update_gru_heads, net32, h_ij.reshape(-1, DIM), groups_ij.group_of, P["G_W6"], P["G_p"], self._coords, None,
                              h_kk, groups_kk.group_of)
        return net32, (delta, weight, None)
