"""Front end of the path: feature / context encoders and patch extraction -- the role of dpvo/net.py:95-157
(`Patchifier`) and dpvo/extractor.py:200-264 (`BasicEncoder4`), written so that the reference's checkpoint keys
("patchify.fnet.layer1.0.conv1.weight", ...) load unchanged.  `Patchifier` is the training module (library
convolutions through autograd) and the reference the inference path is tested against; `FrameEncoder` is the
inference path: one uint8 image into the ring-buffer slots on the sm_90a encoder kernels (csrc/encoder.cu).

The encoder is a 7x7/2 stem, two residual stages (the second strided: 1/4 resolution in total) and a 1x1 output
convolution.  fnet uses instance normalisation, inet none.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import altcorr, extensions
from .net import DIM as CTX_DIM

ENC_DIM = 32


def _norm(kind, ch):
    return nn.InstanceNorm2d(ch) if kind == "instance" else nn.Sequential()


class _Res(nn.Module):
    """two 3x3 convolutions with a (possibly strided, 1x1-projected) skip; attribute names follow the checkpoint"""

    def __init__(self, cin, cout, norm, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1, stride=stride)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.norm1, self.norm2 = _norm(norm, cout), _norm(norm, cout)
        self.downsample = None
        if stride != 1:
            self.norm3 = _norm(norm, cout)
            self.downsample = nn.Sequential(nn.Conv2d(cin, cout, 1, stride=stride), self.norm3)

    def forward(self, x):
        y = F.relu(self.norm1(self.conv1(x)))
        y = F.relu(self.norm2(self.conv2(y)))
        return F.relu((x if self.downsample is None else self.downsample(x)) + y)


class Encoder4(nn.Module):
    """[b,n,3,H,W] -> [b,n,out,H/4,W/4]"""

    def __init__(self, output_dim=128, norm_fn="instance"):
        super().__init__()
        self.conv1 = nn.Conv2d(3, ENC_DIM, 7, stride=2, padding=3)
        self.norm1 = _norm(norm_fn, ENC_DIM)
        self.layer1 = nn.Sequential(_Res(ENC_DIM, ENC_DIM, norm_fn, 1), _Res(ENC_DIM, ENC_DIM, norm_fn, 1))
        self.layer2 = nn.Sequential(_Res(ENC_DIM, 2 * ENC_DIM, norm_fn, 2), _Res(2 * ENC_DIM, 2 * ENC_DIM, norm_fn, 1))
        self.conv2 = nn.Conv2d(2 * ENC_DIM, output_dim, 1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def forward(self, x):
        b, n = x.shape[:2]
        x = x.flatten(0, 1)
        x = F.relu(self.norm1(self.conv1(x)))
        x = self.conv2(self.layer2(self.layer1(x)))
        return x.view(b, n, *x.shape[1:])


def select_centroids(strategy, n, h, w, M, device, images=None):
    """Patch centroids of `n` frames whose features are h x w (net.py:122-139): int64 x, y [n, M].
    RNG: torch.randint for x, then for y, on `device`'s generator -- the reference's draws, in its order.
    GRADIENT_BIAS needs the normalised images [1, n, 3, H, W] and keeps the M of 3M draws with the largest gradient."""
    if strategy == "GRADIENT_BIAS":
        gray = ((images + 0.5) * (255.0 / 2)).sum(dim=2)
        dx = gray[..., :-1, 1:] - gray[..., :-1, :-1]
        dy = gray[..., 1:, :-1] - gray[..., :-1, :-1]
        g = F.avg_pool2d(torch.sqrt(dx ** 2 + dy ** 2), 4, 4)
        x = torch.randint(1, w - 1, size=[n, 3 * M], device=device)
        y = torch.randint(1, h - 1, size=[n, 3 * M], device=device)
        score = altcorr.patchify(g[0, :, None], torch.stack([x, y], -1).float(), 0).view(n, 3 * M)
        keep = torch.argsort(score, dim=1)[:, -M:]
        return torch.gather(x, 1, keep), torch.gather(y, 1, keep)
    if strategy == "RANDOM":
        x = torch.randint(1, w - 1, size=[n, M], device=device)
        y = torch.randint(1, h - 1, size=[n, M], device=device)
        return x, y
    raise NotImplementedError("Patch centroid selection not implemented: %s" % strategy)


def pixel_grid_with_depth(disps):
    """[b,n,h,w] inverse depths -> [b,n,3,h,w] (x, y, d) per pixel"""
    b, n, h, w = disps.shape
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float, device=disps.device),
                            torch.arange(w, dtype=torch.float, device=disps.device), indexing="ij")
    return torch.stack([xs.expand(b, n, h, w), ys.expand(b, n, h, w), disps], dim=2)


class Patchifier(nn.Module):
    def __init__(self, patch_size=3):
        super().__init__()
        self.patch_size = patch_size
        self.fnet = Encoder4(128, "instance")
        self.inet = Encoder4(CTX_DIM, "none")

    def forward(self, images, patches_per_image=80, disps=None, centroid_sel_strat="RANDOM", return_color=False):
        """features, patch features, context, patches [b, n*M, 3, P, P] and their frame index (net.py:110-157).
        RNG: torch.randint x then y on the CUDA generator, in the reference's order."""
        fmap = self.fnet(images) / 4.0
        imap = self.inet(images) / 4.0
        b, n, _, h, w = fmap.shape
        P = self.patch_size
        dev = fmap.device
        x, y = select_centroids(centroid_sel_strat, n, h, w, patches_per_image, dev, images)
        coords = torch.stack([x, y], dim=-1).float()
        imap = altcorr.patchify(imap[0], coords, 0).view(b, -1, CTX_DIM, 1, 1)
        gmap = altcorr.patchify(fmap[0], coords, P // 2).view(b, -1, 128, P, P)
        if disps is None:
            disps = torch.ones(b, n, h, w, device=dev)
        patches = altcorr.patchify(pixel_grid_with_depth(disps)[0], coords, P // 2).view(b, -1, 3, P, P)
        index = torch.arange(n, device=dev).repeat_interleave(patches_per_image)
        if return_color:
            clr = altcorr.patchify(images[0], 4 * (coords + 0.5), 0).view(b, -1, 3)
            return fmap, gmap, imap, patches, index, clr
        return fmap, gmap, imap, patches, index


# ---------------------------------------------------------------------------------------- inference front end
# the convolutions of an Encoder4 in the order of the packed weight blob (include/dpvo_b200.h, "Frame encoders")
def encoder_layers(enc):
    l1, l2 = enc.layer1, enc.layer2
    return [enc.conv1, l1[0].conv1, l1[0].conv2, l1[1].conv1, l1[1].conv2, l2[0].conv1, l2[0].downsample[0],
            l2[0].conv2, l2[1].conv1, l2[1].conv2, enc.conv2]


BIAS_STRIDE = 384          # b32 is [2 encoders][11 layers][384]
STEM_K = 160               # 3 x 7 x 7 = 147 stem taps, zero-padded to 20 chunks of 8


def pack_conv(weight):
    """[cout, cin, k, k] -> fp16 [taps][cin / 8][cout][8] (the stem: one tap of K = 147 padded to 160)"""
    cout, cin, k, _ = weight.shape
    w = weight.detach().half()
    if cin == 3:
        w = F.pad(w.reshape(cout, cin * k * k), (0, STEM_K - cin * k * k)).reshape(1, cout, STEM_K // 8, 8)
    else:
        w = w.permute(2, 3, 0, 1).reshape(k * k, cout, cin // 8, 8)
    return w.permute(0, 2, 1, 3).contiguous().reshape(-1)


def unpack_conv(flat, cout, cin, k):
    """inverse of pack_conv"""
    if cin == 3:
        w = flat.view(1, STEM_K // 8, cout, 8).permute(0, 2, 1, 3).reshape(cout, STEM_K)[:, :cin * k * k]
        return w.reshape(cout, cin, k, k)
    w = flat.view(k * k, cin // 8, cout, 8).permute(0, 2, 1, 3).reshape(k, k, cout, cin)
    return w.permute(2, 3, 0, 1)


def encoder_output_size(H, W):
    """feature size of an H x W image: the 7x7/2 stem, then the 3x3/2 of layer2"""
    h1, w1 = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    return (h1 - 1) // 2 + 1, (w1 - 1) // 2 + 1


class FrameEncoder:
    """Inference front end of a Patchifier: a uint8 image [3, H, W] (CHW or HWC strides) in, the new frame's ring slots
    out, on the sm_90a encoder kernels (csrc/encoder.cu) -- the work of dpvo.py:389-438 minus poses and the viewer.
    The weights are the Patchifier's own (e.g. VONet.patchify, so a checkpoint's patchify.fnet.* / patchify.inet.* are
    used unchanged), repacked whenever they change.  The workspace persists, so encode_into can be captured in a CUDA
    graph (pass `coords` then: the centroid draws are host-side RNG calls)."""

    def __init__(self, patchifier, strategy="RANDOM"):
        self.patchifier = patchifier
        self.strategy = strategy
        self._packed = None
        self._packed_key = None
        self._ws = None

    def _param_key(self):
        return tuple((p.data_ptr(), p._version, p.device) for p in self.patchifier.parameters())

    def pack(self):
        ws, bs = [], torch.zeros(2, 11, BIAS_STRIDE)
        for e, enc in enumerate((self.patchifier.fnet, self.patchifier.inet)):
            for l, conv in enumerate(encoder_layers(enc)):
                ws.append(pack_conv(conv.weight))
                bs[e, l, :conv.out_channels] = conv.bias.detach().float().cpu()
        dev = self.patchifier.fnet.conv1.weight.device
        self._packed = (torch.cat(ws).to(dev).contiguous(), bs.to(dev).contiguous())

    def packed(self):
        """(w16, b32) in the layout of include/dpvo_b200.h"""
        key = self._param_key()
        if self._packed is None or self._packed_key != key:
            self.pack()
            self._packed_key = key
        return self._packed

    def unpack(self):
        """{(encoder, layer): (weight fp16, bias fp32)} read back from the packed blob"""
        w16, b32 = self.packed()
        out, o = {}, 0
        for e, enc in enumerate((self.patchifier.fnet, self.patchifier.inet)):
            for l, conv in enumerate(encoder_layers(enc)):
                cout, cin, k, _ = conv.weight.shape
                n = (1 if cin == 3 else k * k) * (STEM_K if cin == 3 else cin) * cout
                out[(e, l)] = (unpack_conv(w16[o:o + n], cout, cin, k), b32[e, l, :cout])
                o += n
        return out

    def workspace(self, H, W, device, B=1):
        """scratch of B H x W images; it grows and is kept, so a CUDA graph captured with a larger B or image than a
        later call's stays valid (a graph captured before a call that grows it must be captured again)"""
        nb = extensions()[3].encode_frames_workspace_bytes(B, H, W)
        if self._ws is None or self._ws.numel() < nb or self._ws.device != device:
            self._ws = torch.empty(nb, dtype=torch.uint8, device=device)
        return self._ws

    def centroids(self, image, M, strategy):
        """[M, 2] float (x, y) drawn as Patchifier.forward draws them for this image"""
        h, w = encoder_output_size(image.shape[1], image.shape[2])
        images = (2 * (image[None, None] / 255.0) - 0.5) if strategy == "GRADIENT_BIAS" else None
        x, y = select_centroids(strategy, 1, h, w, M, image.device, images)
        return torch.stack([x, y], dim=-1).float()[0]

    @torch.no_grad()
    def encode_into(self, image, M, strategy, fmap1_slot, fmap2_slot, gmap_slot, imap_slot, patches_slot, coords=None,
                    colors_slot=None):
        """Encode `image` into the slots: fmap1 [h, w, 128], fmap2 [h/4, w/4, 128], gmap [M, 3, 3, 128] (all fp16,
        channels-last), imap fp16 [M, 384], patches fp32 [M, 3, 3, 3] with depth 1, and, when `colors_slot` (contiguous
        uint8 [M, 3]) is given, the viewer colours of dpvo.py:392-404 there.  Returns the centroids [M, 2]."""
        if not (isinstance(image, torch.Tensor) and image.is_cuda):
            raise RuntimeError("FrameEncoder: the image must be a CUDA tensor (there is no CPU path)")
        if image.dtype != torch.uint8 or image.dim() != 3 or image.shape[0] != 3:
            raise RuntimeError("FrameEncoder: the image must be uint8 [3, H, W], got %s %s" % (image.dtype, tuple(image.shape)))
        if coords is None:
            coords = self.centroids(image, M, strategy)
        elif coords.shape != (M, 2):
            raise RuntimeError("FrameEncoder: coords must be [M, 2] = [%d, 2], got %s" % (M, tuple(coords.shape)))
        w16, b32 = self.packed()
        extensions()[3].encode_frame(image, w16, b32, coords.float().contiguous(), fmap1_slot, fmap2_slot, gmap_slot,
                                     imap_slot, patches_slot, self.workspace(image.shape[1], image.shape[2], image.device),
                                     colors=colors_slot)
        return coords

    @torch.no_grad()
    def encode_frames_into(self, images, M, strategy, fmap1_ring, fmap2_ring, gmap_ring, imap_ring, patches_ring,
                           frame_rows, feat_rows, patch_rows, coords=None, depth=None, colors_ring=None):
        """encode_into for B images in one pass of the encoders.  images: uint8 [B, 3, H, W] (CHW or HWC strides).
        Image b goes to row frame_rows[b] of the rings fmap1 [R, h, w, 128] and fmap2 [R, h/4, w/4, 128], rows
        feat_rows[b] + [0, M) of gmap [Rg, 3, 3, 128] and imap [Rg, 384], and rows patch_rows[b] + [0, M) of patches
        [Rp, 3, 3, 3] with depth[b] (fp32 [B, M]; None: depth 1).  Each image's slots are bit-identical to encode_into
        of that image alone with the same centroids.  Centroids are drawn once per image, in image order, unless
        `coords` [B, M, 2] is given (then nothing is drawn and the call can be captured).  colors_ring (contiguous uint8
        with Rp rows of 3 bytes, e.g. [Rp / M, M, 3]) receives image b's viewer colours in rows patch_rows[b] + [0, M),
        the rows of its patches.  Returns the coords."""
        if not (isinstance(images, torch.Tensor) and images.is_cuda):
            raise RuntimeError("FrameEncoder: the images must be a CUDA tensor (there is no CPU path)")
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[1] != 3:
            raise RuntimeError("FrameEncoder: the images must be uint8 [B, 3, H, W], got %s %s" % (images.dtype, tuple(images.shape)))
        B, H, W = images.shape[0], images.shape[2], images.shape[3]
        if B < 1:
            raise RuntimeError("FrameEncoder: no images (B = 0)")
        if coords is None:
            coords = torch.stack([self.centroids(images[b], M, strategy) for b in range(B)])
        elif coords.shape != (B, M, 2):
            raise RuntimeError("FrameEncoder: coords must be [B, M, 2] = [%d, %d, 2], got %s" % (B, M, tuple(coords.shape)))
        w16, b32 = self.packed()
        extensions()[3].encode_frames(images, w16, b32, coords.float().contiguous(), fmap1_ring, fmap2_ring, gmap_ring, imap_ring,
                                      patches_ring, [int(r) for r in frame_rows], [int(r) for r in feat_rows],
                                      [int(r) for r in patch_rows], depth, self.workspace(H, W, images.device, B),
                                      colors=colors_ring)
        return coords
