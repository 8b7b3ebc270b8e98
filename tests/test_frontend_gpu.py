"""The frame encoders on the sm_90a kernels (csrc/encoder.cu): each layer shape through encoder_conv against float64
convolutions, a whole frame against Patchifier, the exact relations between the slots, the RNG draws, determinism,
slot isolation, CUDA-graph capture and argument rejection."""
import pytest
import torch
import torch.nn.functional as F

from dpvo_b200 import extensions, frontend, synthetic
from dpvo_b200.runner import UpdateRunner

pytestmark = pytest.mark.gpu

SIZES = [(480, 640), (480, 752), (250, 330)]
# (shape id, k, stride, cin, cout)
SHAPES = {"stem": (0, 7, 2, 3, 32), "c3_32": (1, 3, 1, 32, 32), "c3s2_32_64": (2, 3, 2, 32, 64), "c1s2_32_64": (3, 1, 2, 32, 64),
          "c3_64": (4, 3, 1, 64, 64), "out_128": (5, 1, 1, 64, 128), "out_384": (6, 1, 1, 64, 384)}


@pytest.fixture(scope="module")
def ex():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return extensions()[3]


def structured_image(H, W, seed=0, hwc=False):
    """gradients plus noise, uint8 [3, H, W] (a permuted HWC buffer when hwc)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ys = torch.linspace(0, 1, H, device="cuda")[:, None]
    xs = torch.linspace(0, 1, W, device="cuda")[None, :]
    base = torch.stack([160 * xs + 60 * ys, 200 * ys * (1 - xs) + 30, 120 + 100 * torch.sin(12 * xs + 7 * ys)])
    img = (base + 25 * torch.randn(3, H, W, device="cuda", generator=g)).clamp(0, 255).to(torch.uint8)
    if hwc:
        img = img.permute(1, 2, 0).contiguous().permute(2, 0, 1)
    return img


def fp16_ulp(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def level_size(name, H, W):
    h1, w1 = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    if name == "stem":
        return H, W
    if name in ("c3_32", "c3s2_32_64", "c1s2_32_64"):
        return h1, w1
    return frontend.encoder_output_size(H, W)


def _transform(x, stats, relu):
    f = x.float()
    if stats is not None:
        f = (f - stats[0]) * stats[1]
    return f.clamp_min(0) if relu else f


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("prologue", ["plain", "norm_relu", "join"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_encoder_conv_layer(ex, name, prologue, size):
    sid, k, s, cin, cout = SHAPES[name]
    if name == "stem" and prologue != "plain":
        pytest.skip("the stem's prologue is the image normalisation")
    H, W = level_size(name, *size)
    torch.manual_seed(sid * 10 + len(prologue))
    conv = torch.nn.Conv2d(cin, cout, k, stride=s, padding=k // 2).cuda()
    w = frontend.pack_conv(conv.weight)
    bias = conv.bias.detach().float().contiguous()
    scale = 0.25 if name.startswith("out") else 1.0
    kw = {}
    if name == "stem":
        x = structured_image(H, W, seed=sid, hwc=True)
        xin = (2 * (x / 255.0) - 0.5).half()[None]                       # dpvo.py:389, then autocast's fp16 operand
    else:
        x = (torch.randn(H, W, cin, device="cuda") * 1.5 + 0.3).half()
        xs = torch.stack([torch.randn(cin, device="cuda") * 0.3, torch.rand(cin, device="cuda") + 0.5]).contiguous()
        if prologue == "plain":
            t = _transform(x, None, False)
        elif prologue == "norm_relu":
            kw = dict(x_stats=xs, x_relu=True)
            t = _transform(x, xs[:, None, None, :], True)
        else:
            skip = (torch.randn(H, W, cin, device="cuda")).half()
            ss = torch.stack([torch.randn(cin, device="cuda") * 0.2, torch.rand(cin, device="cuda") + 0.5]).contiguous()
            skip_relu = sid % 2 == 1
            kw = dict(x_stats=xs, x_relu=True, skip=skip, skip_stats=ss, skip_relu=skip_relu, want_joined=(k == 3))
            t = (_transform(skip, ss[:, None, None, :], skip_relu) + _transform(x, xs[:, None, None, :], True)).clamp_min(0)
        xin = t.half().permute(2, 0, 1)[None]
    y, st, joined, pool = ex.encoder_conv(sid, x, w, bias, want_stats=cout <= 64, want_pool=(name == "out_128"), scale=scale, **kw)
    torch.cuda.synchronize()
    ref = (F.conv2d(xin.double(), conv.weight.detach().half().double(), conv.bias.detach().double(), stride=s, padding=k // 2) * scale)[0]
    ref = ref.permute(1, 2, 0)
    assert y.shape == ref.shape
    err = (y.double() - ref).abs()
    tol = torch.maximum(fp16_ulp(ref), torch.full_like(ref, 2.0 ** -14))
    assert bool((err <= tol).all()), "%s/%s %s: max err %g (%d over the bar)" % (name, prologue, size, err.max().item(), int((err > tol).sum()))
    if joined is not None:
        assert torch.equal(joined, t.half()), "joined block output"
    if st is not None:
        yd = y.double().reshape(-1, cout)
        mean, var = yd.mean(0), yd.var(0, unbiased=False)
        rstd = 1 / torch.sqrt(var + 1e-5)
        assert bool(((st[0].double() - mean).abs() <= 1e-5 * (mean.abs() + var.sqrt())).all()), "instance-norm mean"
        assert bool(((st[1].double() - rstd).abs() <= 1e-5 * rstd).all()), "instance-norm rstd"
    if pool is not None:
        assert torch.equal(pool.permute(2, 0, 1), F.avg_pool2d(y.permute(2, 0, 1), 4, 4)), "4x4 average"


# ------------------------------------------------------------------------------------------------ whole frames
def _patchifier(seed=0):
    torch.manual_seed(seed)
    return frontend.Patchifier().cuda().eval()


def _slots(H, W, M):
    h, w = frontend.encoder_output_size(H, W)
    dev = "cuda"
    return dict(fmap1=torch.empty(h, w, 128, device=dev, dtype=torch.half), fmap2=torch.empty(h // 4, w // 4, 128, device=dev, dtype=torch.half),
                gmap=torch.empty(M, 3, 3, 128, device=dev, dtype=torch.half), imap=torch.empty(M, 384, device=dev, dtype=torch.half),
                patches=torch.empty(M, 3, 3, 3, device=dev))


def _encode(fe, img, M, strategy="RANDOM", coords=None):
    s = _slots(img.shape[1], img.shape[2], M)
    c = fe.encode_into(img, M, strategy, s["fmap1"], s["fmap2"], s["gmap"], s["imap"], s["patches"], coords=coords)
    return s, c


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_frame_against_patchifier(ex, size):
    H, W = size
    M = 96
    p = _patchifier(1)
    fe = frontend.FrameEncoder(p)
    img = structured_image(H, W, seed=5)
    images = (2 * (img[None, None] / 255.0) - 0.5)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False                             # a true fp32 reference
    with torch.no_grad():
        torch.manual_seed(11)
        fmap, gmap, imap, _, _ = p(images, patches_per_image=M)
        torch.manual_seed(11)
        with torch.autocast("cuda", dtype=torch.float16):
            fmap_a, gmap_a, imap_a, _, _ = p(images, patches_per_image=M)
    torch.backends.cudnn.allow_tf32 = tf32
    torch.manual_seed(11)
    s, _ = _encode(fe, img, M)
    torch.cuda.synchronize()
    pairs = {"fmap1": (s["fmap1"].permute(2, 0, 1), fmap[0, 0], fmap_a[0, 0]),
             "imap": (s["imap"], imap.view(M, 384), imap_a.view(M, 384)),
             "gmap": (s["gmap"].permute(0, 3, 1, 2), gmap.view(M, 128, 3, 3), gmap_a.view(M, 128, 3, 3))}
    for nm, (ours, ref, ac) in pairs.items():
        e_ours = (ours.double() - ref.double()).abs().max().item()
        e_ac = (ac.double() - ref.double()).abs().max().item()
        rms = ref.double().pow(2).mean().sqrt()
        bar = 2 * e_ac + fp16_ulp(rms).item()
        print("\n[%dx%d %s] max err vs fp32: ours %.3g, autocast %.3g" % (H, W, nm, e_ours, e_ac))
        assert e_ours <= bar, "%s: %g > 2 x %g + ulp(rms)" % (nm, e_ours, e_ac)


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_exact_slot_relations_and_determinism(ex, size):
    H, W = size
    M = 48
    fe = frontend.FrameEncoder(_patchifier(2))
    img = structured_image(H, W, seed=9, hwc=size[1] == 752)
    torch.manual_seed(3)
    s, c = _encode(fe, img, M)
    s2, c2 = _encode(fe, img, M, coords=c)
    torch.cuda.synchronize()
    for k in s:
        assert torch.equal(s[k], s2[k]), "two launches differ in %s" % k
    f1 = s["fmap1"].permute(2, 0, 1)
    assert torch.equal(s["fmap2"].permute(2, 0, 1), F.avg_pool2d(f1, 4, 4))
    x, y = c[:, 0].long(), c[:, 1].long()
    for m in range(M):
        assert torch.equal(s["gmap"][m], s["fmap1"][y[m] - 1:y[m] + 2, x[m] - 1:x[m] + 2])
    offs = torch.tensor([-1.0, 0.0, 1.0], device="cuda")
    assert torch.equal(s["patches"][:, 0], (c[:, 0, None, None] + offs[None, None, :]).expand(M, 3, 3))
    assert torch.equal(s["patches"][:, 1], (c[:, 1, None, None] + offs[None, :, None]).expand(M, 3, 3))
    assert bool((s["patches"][:, 2] == 1).all())


def _runner(config, strategy="RANDOM", seed=4):
    st = synthetic.make_state(config, 12, device="cuda", seed=7, mem=16)
    fe = frontend.FrameEncoder(_patchifier(seed), strategy=strategy)
    return UpdateRunner(st, encoder=fe), st


@pytest.mark.parametrize("strategy", ["RANDOM", "GRADIENT_BIAS"])
def test_centroids_depth_and_rng_follow_the_reference_order(ex, strategy):
    run, st = _runner("default", strategy)
    M = st.cfg["M"]
    img = structured_image(480, 640, seed=2)
    images = (2 * (img[None, None] / 255.0) - 0.5)
    torch.manual_seed(21)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        _, _, _, patches, _ = run.encoder.patchifier(images, patches_per_image=M, centroid_sel_strat=strategy)
    depth = torch.rand_like(patches[:, :, 2, 0, 0, None, None])          # dpvo.py:427
    rng_ref = torch.cuda.get_rng_state()
    torch.manual_seed(21)
    c = run.ingest_image(img)
    rng = torch.cuda.get_rng_state()
    q = st.patches[(st.n - 1) * M:st.n * M]
    assert torch.equal(c[:, 0], patches[0, :, 0, 1, 1]) and torch.equal(c[:, 1], patches[0, :, 1, 1, 1])
    assert torch.equal(q[:, 2], depth[0].expand(M, 3, 3))
    assert torch.equal(rng, rng_ref)


def test_ingest_image_touches_only_its_slots(ex):
    run, st = _runner("fast")
    M = st.cfg["M"]
    for t in (st.fmap1, st.fmap2, st.gmap, st.imap):
        t.fill_(7.0)
    st.patches.fill_(-3.0)
    img = structured_image(480, 752, seed=1)
    before = {k: getattr(st, k).clone() for k in ("fmap1", "fmap2", "gmap", "imap", "patches")}
    run.ingest_image(img, depth=torch.tensor(0.5, device="cuda"))
    torch.cuda.synchronize()
    slot, pslot = (st.n - 1) % run.mem, (st.n - 1) % run.pmem
    for k in ("fmap1", "fmap2"):
        a, b = getattr(st, k)[0], before[k][0]
        assert not torch.equal(a[slot], b[slot])
        keep = [i for i in range(a.shape[0]) if i != slot]
        assert torch.equal(a[keep], b[keep]), k
    for k in ("gmap", "imap"):
        a, b = getattr(st, k)[0], before[k][0]
        assert not torch.equal(a[pslot * M:(pslot + 1) * M], b[pslot * M:(pslot + 1) * M])
        assert torch.equal(a[:pslot * M], b[:pslot * M]) and torch.equal(a[(pslot + 1) * M:], b[(pslot + 1) * M:]), k
    lo, hi = (st.n - 1) * M, st.n * M
    assert torch.equal(st.patches[:lo], before["patches"][:lo]) and torch.equal(st.patches[hi:], before["patches"][hi:])
    assert bool((st.patches[lo:hi, 2] == 0.5).all())


def test_graph_of_ingest_image_and_step_equals_eager(ex):
    run, st = _runner("fast")
    M = st.cfg["M"]
    img = structured_image(480, 752, seed=4)
    torch.manual_seed(5)
    coords = run.encoder.centroids(img, M, "RANDOM")
    depth = torch.rand(M, 1, 1, device="cuda")
    names = ("poses", "patches", "fmap1", "fmap2", "gmap", "imap")
    snap = {k: getattr(st, k).clone() for k in names}
    net0 = run.net.clone()

    def restore():
        for k in names:
            getattr(st, k).copy_(snap[k])
        run.net.copy_(net0)

    def frame():
        run.ingest_image(img, depth=depth, coords=coords)
        return run.step()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        frame()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    restore()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out_g = frame()
    restore()
    g.replay()
    torch.cuda.synchronize()
    res_g = [t.clone() for t in out_g] + [getattr(st, k).clone() for k in names]
    restore()
    out_e = frame()
    torch.cuda.synchronize()
    res_e = list(out_e) + [getattr(st, k) for k in names]
    for a, b in zip(res_g, res_e):
        assert torch.equal(a, b)


def test_rejected_arguments(ex):
    run, st = _runner("fast")
    img = structured_image(480, 752)
    with pytest.raises(RuntimeError, match="CUDA"):
        run.ingest_image(img.cpu())
    with pytest.raises(RuntimeError, match="uint8"):
        run.ingest_image(img.float())
    with pytest.raises(RuntimeError, match="rings hold"):
        run.ingest_image(structured_image(480, 640))
    s = _slots(480, 752, 8)
    with pytest.raises(RuntimeError, match="encodes to"):
        w16, b32 = run.encoder.packed()
        ex.encode_frame(structured_image(480, 640), w16, b32, torch.zeros(8, 2, device="cuda"), s["fmap1"], s["fmap2"], s["gmap"],
                        s["imap"], s["patches"], torch.empty(1 << 20, dtype=torch.uint8, device="cuda"))
