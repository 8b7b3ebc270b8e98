"""Several camera images in one pass of the frame encoders (dpvo_encode_frames, FrameEncoder.encode_frames_into,
UpdateRunner.ingest_images): every image's slots bit-identical to encoding it alone, only the named streams' slots
written, the CUDA generator drawn as the per-stream calls draw it, determinism, launches independent of the number of
images, CUDA-graph capture and argument rejection."""
import pytest
import torch

from dpvo_b200 import extensions, frontend, synthetic
from dpvo_b200.runner import UpdateRunner

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = ("fmap1", "fmap2", "gmap", "imap", "patches")


@pytest.fixture(scope="module")
def ex():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return extensions()[3]


def structured_image(H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ys = torch.linspace(0, 1, H, device=DEV)[:, None]
    xs = torch.linspace(0, 1, W, device=DEV)[None, :]
    base = torch.stack([160 * xs + 60 * ys, 200 * ys * (1 - xs) + 30, 120 + 100 * torch.sin(12 * xs + 7 * ys)])
    return (base + 25 * torch.randn(3, H, W, device=DEV, generator=g)).clamp(0, 255).to(torch.uint8)


def images_for(B, H, W, hwc=False):
    """B different images: a structured one, a constant one and a high-contrast noise one first (instance-norm
    statistics leaking between images would show there), then structured images of other seeds"""
    g = torch.Generator(device=DEV).manual_seed(B)
    imgs = [structured_image(H, W, 100), torch.full((3, H, W), 77, dtype=torch.uint8, device=DEV),
            (torch.randint(0, 2, (3, H, W), generator=g, device=DEV) * 255).to(torch.uint8)]
    imgs += [structured_image(H, W, 100 + b) for b in range(3, B)]
    x = torch.stack(imgs[:B])
    return x.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2) if hwc else x


def _encoder(strategy="RANDOM", seed=4):
    torch.manual_seed(seed)
    return frontend.FrameEncoder(frontend.Patchifier().cuda().eval(), strategy=strategy)


def _rings(H, W, M, R, Rg, Rp, fill=7.0):
    h, w = frontend.encoder_output_size(H, W)
    return dict(fmap1=torch.full((R, h, w, 128), fill, device=DEV, dtype=torch.half),
                fmap2=torch.full((R, h // 4, w // 4, 128), fill, device=DEV, dtype=torch.half),
                gmap=torch.full((Rg, 3, 3, 128), fill, device=DEV, dtype=torch.half),
                imap=torch.full((Rg, 384), fill, device=DEV, dtype=torch.half),
                patches=torch.full((Rp, 3, 3, 3), -3.0, device=DEV))


def _encode_alone(fe, img, M, coords):
    H, W = img.shape[1], img.shape[2]
    s = _rings(H, W, M, 1, M, M)
    fe.encode_into(img, M, "RANDOM", s["fmap1"][0], s["fmap2"][0], s["gmap"], s["imap"], s["patches"], coords=coords)
    return s


def _check_batch_against_alone(fe, images, M):
    B, H, W = images.shape[0], images.shape[2], images.shape[3]
    # destinations out of order and with gaps, in rings larger than the batch
    frame_rows = [B - b for b in range(B)]
    feat_rows = [(2 * b + 1) * M for b in range(B)]
    patch_rows = [(2 * (B - 1 - b)) * M + 3 for b in range(B)]
    r = _rings(H, W, M, B + 2, (2 * B + 1) * M, 2 * B * M + 3)
    before = {k: v.clone() for k, v in r.items()}
    torch.manual_seed(3)
    coords = fe.encode_frames_into(images, M, "RANDOM", r["fmap1"], r["fmap2"], r["gmap"], r["imap"], r["patches"],
                                   frame_rows, feat_rows, patch_rows)
    assert coords.shape == (B, M, 2)
    written = {k: torch.zeros(v.shape[0], dtype=torch.bool, device=DEV) for k, v in r.items()}
    for b in range(B):
        s = _encode_alone(fe, images[b], M, coords[b])
        rows = {"fmap1": (frame_rows[b], 1), "fmap2": (frame_rows[b], 1), "gmap": (feat_rows[b], M),
                "imap": (feat_rows[b], M), "patches": (patch_rows[b], M)}
        for k, (lo, n) in rows.items():
            assert torch.equal(r[k][lo:lo + n], s[k]), "image %d of %d: %s differs from encoding it alone" % (b, B, k)
            written[k][lo:lo + n] = True
    for k in r:
        assert torch.equal(r[k][~written[k]], before[k][~written[k]]), "%s: a row no image owns was written" % k


@pytest.mark.parametrize("size", [(480, 640), (480, 752), (250, 330)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("B", [1, 2, 3, 8])
def test_each_image_bit_identical_to_encoding_it_alone(ex, B, size):
    _check_batch_against_alone(_encoder(), images_for(B, *size, hwc=size[1] == 752), 48)


def test_sixty_four_images(ex):
    _check_batch_against_alone(_encoder(), images_for(64, 64, 96), 8)


# ------------------------------------------------------------------------------------------------ the runner
def _batch_runner(strategy="RANDOM", B=3, frames=(12, 9, 14)):
    batch = synthetic.make_batch("fast", B, [11 + b for b in range(B)], n_frames=list(frames), device=DEV,
                                 frames_per_stream=64, mem=16)
    return UpdateRunner(batch, encoder=_encoder(strategy)), batch


def _fill_sentinels(batch):
    for t in (batch.fmap1, batch.fmap2, batch.gmap, batch.imap):
        t.fill_(7.0)
    batch.patches.fill_(-3.0)


def _camera_images(n, seed=0):
    return torch.stack([structured_image(480, 752, seed + i) for i in range(n)])


def test_ingest_images_writes_only_the_named_streams_slots(ex):
    run, batch = _batch_runner()
    M, mem, pmem, F = batch.M, batch.mem, batch.pmem, batch.F
    _fill_sentinels(batch)
    names = NAMES + ("poses", "intrinsics")
    before = {k: getattr(batch, k).clone() for k in names}
    imgs = _camera_images(2, seed=30)
    streams = [2, 0]
    depth = torch.rand(2, M, device=DEV) + 0.5
    torch.manual_seed(8)
    coords = run.ingest_images(imgs, depth=depth, streams=streams)
    torch.cuda.synchronize()
    written = {k: torch.zeros(getattr(batch, k).shape[1 if k in ("fmap1", "fmap2", "gmap", "imap") else 0], dtype=torch.bool,
                              device=DEV) for k in NAMES}
    for i, b in enumerate(streams):
        s = batch.stream(b)
        slot, pslot, prow = b * mem + (s.n - 1) % mem, (b * pmem + (s.n - 1) % pmem) * M, (b * F + s.n - 1) * M
        written["fmap1"][slot] = written["fmap2"][slot] = True
        written["gmap"][pslot:pslot + M] = written["imap"][pslot:pslot + M] = True
        written["patches"][prow:prow + M] = True
        assert torch.equal(batch.patches[prow:prow + M, 2], depth[i, :, None, None].expand(M, 3, 3))
    for k in names:
        a, o = getattr(batch, k), before[k]
        if k not in written:
            assert torch.equal(a, o), k
            continue
        sel = written[k]
        a, o = (a[0], o[0]) if k != "patches" else (a, o)
        assert not torch.equal(a[sel], o[sel]), k
        assert torch.equal(a[~sel], o[~sel]), "%s: a row outside streams %s was written" % (k, streams)
    # the same bytes as ingest_image(stream=b) of each image
    after = {k: getattr(batch, k).clone() for k in NAMES}
    _fill_sentinels(batch)
    for i, b in enumerate(streams):
        run.ingest_image(imgs[i], depth=depth[i, :, None, None], coords=coords[i], stream=b)
    torch.cuda.synchronize()
    for k in NAMES:
        assert torch.equal(getattr(batch, k), after[k]), k


@pytest.mark.parametrize("strategy", ["RANDOM", "GRADIENT_BIAS"])
def test_rng_draws_follow_the_per_stream_calls(ex, strategy):
    run, batch = _batch_runner(strategy)
    imgs = _camera_images(3, seed=40)
    streams = [1, 2, 0]
    snap = {k: getattr(batch, k).clone() for k in NAMES}
    torch.manual_seed(21)
    c = run.ingest_images(imgs, streams=streams)
    rng = torch.cuda.get_rng_state()
    torch.cuda.synchronize()
    batched = {k: getattr(batch, k).clone() for k in NAMES}
    for k in NAMES:
        getattr(batch, k).copy_(snap[k])
    torch.manual_seed(21)
    c_ref = torch.stack([run.ingest_image(imgs[i], stream=b) for i, b in enumerate(streams)])
    rng_ref = torch.cuda.get_rng_state()
    torch.cuda.synchronize()
    assert torch.equal(c, c_ref), "centroids"
    assert torch.equal(rng, rng_ref), "CUDA generator state afterwards"
    for k in NAMES:                                    # patches carry the depths
        assert torch.equal(batched[k], getattr(batch, k)), k


def test_two_batched_launches_give_identical_bits(ex):
    run, batch = _batch_runner()
    imgs = _camera_images(3, seed=50)
    _fill_sentinels(batch)
    torch.manual_seed(2)
    c = run.ingest_images(imgs, depth=torch.tensor(0.75, device=DEV))
    torch.cuda.synchronize()
    first = {k: getattr(batch, k).clone() for k in NAMES}
    _fill_sentinels(batch)
    run.ingest_images(imgs, depth=torch.tensor(0.75, device=DEV), coords=c)
    torch.cuda.synchronize()
    for k in NAMES:
        assert torch.equal(first[k], getattr(batch, k)), k


def test_launches_do_not_grow_with_the_number_of_images(ex):
    run, batch = _batch_runner(B=8, frames=[12, 9, 14, 10, 11, 13, 12, 9])
    M = batch.M
    imgs = _camera_images(8, seed=60)
    coords = torch.stack([run.encoder.centroids(imgs[i], M, "RANDOM") for i in range(8)])
    depth = torch.ones(8, M, device=DEV)

    def launches(fn):
        n0 = ex.launch_count()
        fn()
        torch.cuda.synchronize()
        return ex.launch_count() - n0

    one = launches(lambda: run.ingest_images(imgs[:1], coords=coords[:1], depth=depth[:1], streams=[3]))
    eight = launches(lambda: run.ingest_images(imgs, coords=coords, depth=depth))
    single = launches(lambda: run.ingest_image(imgs[0], coords=coords[0], depth=depth[0, :, None, None], stream=3))
    assert one == eight == single == 12, (one, eight, single)


def test_graph_of_ingest_images_and_step_equals_eager(ex):
    run, batch = _batch_runner()
    M = batch.M
    imgs = _camera_images(3, seed=70)
    torch.manual_seed(5)
    coords = torch.stack([run.encoder.centroids(imgs[i], M, "RANDOM") for i in range(3)])
    depth = torch.rand(3, M, device=DEV)
    names = ("poses", "patches", "fmap1", "fmap2", "gmap", "imap")
    snap = {k: getattr(batch, k).clone() for k in names}
    net0 = run.net.clone()

    def restore():
        for k in names:
            getattr(batch, k).copy_(snap[k])
        run.net.copy_(net0)

    def frame():
        run.ingest_images(imgs, depth=depth, coords=coords)
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
    res_g = [t.clone() for t in out_g] + [getattr(batch, k).clone() for k in names]
    restore()
    out_e = frame()
    torch.cuda.synchronize()
    res_e = list(out_e) + [getattr(batch, k) for k in names]
    for a, b in zip(res_g, res_e):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ rejection
def test_runner_rejects_bad_calls(ex):
    run, batch = _batch_runner()
    imgs = _camera_images(2)
    with pytest.raises(RuntimeError, match="use ingest_image"):
        st = synthetic.make_state("fast", 12, device=DEV, seed=7, mem=16)
        UpdateRunner(st, encoder=run.encoder, update=run.update).ingest_images(imgs)
    with pytest.raises(RuntimeError, match="twice"):
        run.ingest_images(imgs, streams=[1, 1])
    with pytest.raises(RuntimeError, match="outside the batch"):
        run.ingest_images(imgs, streams=[0, 3])
    with pytest.raises(RuntimeError, match="2 images for 3 streams"):
        run.ingest_images(imgs)
    with pytest.raises(RuntimeError, match="rings hold"):
        run.ingest_images(torch.zeros(2, 3, 480, 640, dtype=torch.uint8, device=DEV), streams=[0, 1])
    with pytest.raises(RuntimeError, match="uint8"):
        run.ingest_images(imgs.float(), streams=[0, 1])
    with pytest.raises(RuntimeError, match="CUDA"):
        run.ingest_images(imgs.cpu(), streams=[0, 1])


def test_shim_rejects_bad_calls(ex):
    fe = _encoder()
    w16, b32 = fe.packed()
    H, W, M = 64, 96, 8
    r = _rings(H, W, M, 70, 70 * M, 70 * M)
    ws = fe.workspace(H, W, torch.device(DEV), 64)

    def call(B, frame_rows=None, feat_rows=None, patch_rows=None, images=None, rings=r):
        images = torch.zeros(B, 3, H, W, dtype=torch.uint8, device=DEV) if images is None else images
        frame_rows = list(range(B)) if frame_rows is None else frame_rows
        feat_rows = [b * M for b in range(B)] if feat_rows is None else feat_rows
        patch_rows = [b * M for b in range(B)] if patch_rows is None else patch_rows
        ex.encode_frames(images, w16, b32, torch.zeros(B, M, 2, device=DEV), rings["fmap1"], rings["fmap2"], rings["gmap"],
                         rings["imap"], rings["patches"], frame_rows, feat_rows, patch_rows, None, ws)

    with pytest.raises(RuntimeError, match="B=65 images, 1 to 64"):
        call(65)
    with pytest.raises(RuntimeError, match="images 0 and 1 write the same destination fmap1"):
        call(2, frame_rows=[5, 5])
    with pytest.raises(RuntimeError, match="same destination gmap / imap"):
        call(2, feat_rows=[0, M // 2])
    with pytest.raises(RuntimeError, match="same destination patch"):
        call(2, patch_rows=[M, 1])
    with pytest.raises(RuntimeError, match="outside the 70-row"):
        call(2, frame_rows=[0, 70])
    with pytest.raises(RuntimeError, match="encodes to"):
        call(2, images=torch.zeros(2, 3, 480, 640, dtype=torch.uint8, device=DEV))
    with pytest.raises(RuntimeError, match="uint8"):
        call(2, images=torch.zeros(2, 3, H, W, device=DEV))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        call(2, images=torch.zeros(2, 3, H, W, dtype=torch.uint8))
    torch.cuda.synchronize()
    assert torch.equal(r["fmap1"], torch.full_like(r["fmap1"], 7.0)), "a rejected call wrote"
