"""torch.autograd bindings of the C-ABI kernels (include/bts_b200.h).

PyTorch is plumbing here: device memory, the current stream, autograd bookkeeping.  Every op launches
hand-written sm_90a kernels from libbts_b200.so through ctypes with raw device pointers; there is no eager
or CPU fallback -- non-CUDA inputs raise.
"""
import ctypes

import numpy as np
import torch

from . import _lib, data

_vp = ctypes.c_void_p


def _ptr(t):
    return None if t is None else _vp(t.data_ptr())


def _stream():
    return _vp(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("bts_b200 ops run on CUDA (sm_90a) tensors only; got a %s tensor -- "
                               "there is no CPU fallback" % t.device.type)


def _f32c(t):
    if t.dtype != torch.float32:
        raise TypeError("bts_b200 ops compute in fp32; got %s" % t.dtype)
    return t.contiguous()


# ----------------------------------------------------------------------------------------------- LPG
class _Lpg(torch.autograd.Function):
    """local_planar_guidance.forward (reference pytorch/bts.py:132-146) as one kernel each way."""

    @staticmethod
    def forward(ctx, plane, r, layout, tf_compat):
        _need_cuda(plane)
        plane = _f32c(plane)
        if layout == 0:
            B, four, h, w = plane.shape
        else:
            B, h, w, four = plane.shape
        if four != 4:
            raise ValueError("plane_eq must have 4 coefficients per patch, got %d" % four)
        depth = torch.empty((B, h * r, w * r), device=plane.device, dtype=torch.float32)
        with torch.cuda.device(plane.device):
            _lib.check(_lib.lib().bts_lpg_fwd(_ptr(plane), _ptr(depth), B, h, w, r, layout, _stream()), "bts_lpg_fwd")
        _lib.count()
        ctx.save_for_backward(plane)
        ctx.meta = (B, h, w, r, layout, tf_compat)
        return depth

    @staticmethod
    def backward(ctx, dy):
        (plane,) = ctx.saved_tensors
        B, h, w, r, layout, tf_compat = ctx.meta
        dy = _f32c(dy)
        dplane = torch.empty_like(plane)
        with torch.cuda.device(plane.device):
            _lib.check(_lib.lib().bts_lpg_bwd(_ptr(dy), _ptr(plane), _ptr(dplane), B, h, w, r, layout,
                                              int(tf_compat), _stream()), "bts_lpg_bwd")
        _lib.count()
        return dplane, None, None, None


def lpg(plane_eq, upratio, layout="nchw", tf_compat=False):
    """depth (B,H,W) from plane_eq (B,4,h,w) [layout='nchw'] or (B,h,w,4) [layout='nhwc', the TF op's]."""
    return _Lpg.apply(plane_eq, int(upratio), 0 if layout == "nchw" else 1, bool(tf_compat))


# ------------------------------------------------------------------------------- fused head tail + LPG
class _PlaneHeadLpg(torch.autograd.Function):
    """reduction_1x1's trig tail + F.normalize + cat + LPG + /max_depth + nearest down-sample
    (reference pytorch/bts.py:112-120 and 223-229 / 237-243 / 251-256): ~35 ATen kernels -> 1 each way."""

    @staticmethod
    def forward(ctx, c3, r, max_depth, ds_stride):
        _need_cuda(c3)
        c3 = _f32c(c3)
        B, three, h, w = c3.shape
        if three != 3:
            raise ValueError("plane_params output must have 3 channels, got %d" % three)
        H, W = h * r, w * r
        scaled = torch.empty((B, 1, H, W), device=c3.device, dtype=torch.float32)
        ds = None
        if ds_stride:
            ds = torch.empty((B, 1, H // ds_stride, W // ds_stride), device=c3.device, dtype=torch.float32)
        with torch.cuda.device(c3.device):
            _lib.check(_lib.lib().bts_plane_head_fwd(_ptr(c3), None, _ptr(scaled), _ptr(ds), float(max_depth),
                                                     int(ds_stride or 1), B, h, w, r, _stream()), "bts_plane_head_fwd")
        _lib.count()
        ctx.save_for_backward(c3)
        ctx.meta = (B, h, w, r, float(max_depth), int(ds_stride or 0))
        if ds is None:
            return scaled
        return scaled, ds

    @staticmethod
    def backward(ctx, d_scaled, d_ds=None):
        (c3,) = ctx.saved_tensors
        B, h, w, r, max_depth, S = ctx.meta
        if d_scaled is None and d_ds is None:
            return None, None, None, None
        d_scaled = None if d_scaled is None else _f32c(d_scaled)
        d_ds = None if (d_ds is None or not S) else _f32c(d_ds)
        dc3 = torch.empty_like(c3)
        with torch.cuda.device(c3.device):
            _lib.check(_lib.lib().bts_plane_head_bwd(_ptr(d_scaled), _ptr(d_ds), _ptr(c3), _ptr(dc3), max_depth,
                                                     S or 1, B, h, w, r, _stream()), "bts_plane_head_bwd")
        _lib.count()
        return dc3, None, None, None


def plane_head_lpg(c3, upratio, max_depth, ds_stride=0):
    """(scaled[, ds]) = fused head tail + LPG.  scaled (B,1,H,W) = depth/max_depth; ds = scaled[::S, ::S]."""
    return _PlaneHeadLpg.apply(c3, int(upratio), float(max_depth), int(ds_stride))


# --------------------------------------------------------------------------------------------- silog
class _Silog(torch.autograd.Function):
    """silog_loss.forward (reference pytorch/bts.py:46-48) + its backward: 2 streaming passes total."""

    @staticmethod
    def forward(ctx, est, gt, mask, lam):
        _need_cuda(est, gt, mask)
        est, gt = _f32c(est), _f32c(gt)
        if mask.dtype != torch.bool and mask.dtype != torch.uint8:
            raise TypeError("mask must be bool/uint8")
        mask = mask.contiguous()
        if est.shape != gt.shape or est.shape != mask.shape:
            raise ValueError("depth_est / depth_gt / mask shapes differ")
        n = est.numel()
        ws = torch.empty(4, device=est.device, dtype=torch.float64)
        loss = torch.empty((), device=est.device, dtype=torch.float32)
        with torch.cuda.device(est.device):
            _lib.check(_lib.lib().bts_silog_fwd(_ptr(est), _ptr(gt), _ptr(mask), n, float(lam), _ptr(ws), _ptr(loss),
                                                _stream()), "bts_silog_fwd")
        _lib.count(2)
        ctx.save_for_backward(est, gt, mask, ws)
        ctx.lam = float(lam)
        return loss

    @staticmethod
    def backward(ctx, gout):
        est, gt, mask, ws = ctx.saved_tensors
        gout = gout.to(torch.float32).contiguous()
        dest = torch.empty_like(est)
        with torch.cuda.device(est.device):
            _lib.check(_lib.lib().bts_silog_bwd(_ptr(est), _ptr(gt), _ptr(mask), est.numel(), ctx.lam, _ptr(ws),
                                                _ptr(gout), _ptr(dest), _stream()), "bts_silog_bwd")
        _lib.count()
        return dest, None, None, None


def silog(depth_est, depth_gt, mask, variance_focus):
    return _Silog.apply(depth_est, depth_gt, mask, float(variance_focus))


# ------------------------------------------------------------------------------------------------ data formats (SURVEY 8f)
def input_prep(img_u8, params, out_hw, depth_u16=None, depth_div=1000.0, angles=None):
    """reference loader transform on the GPU (pytorch/bts_dataloader.py:128-140,202-235,244-249): img_u8 (B,Hs,Ws,3) uint8
    CUDA, params (B,9) fp32 = y0,x0,flip,augment,gamma,brightness,colour rgb -> (image (B,3,H,W) channels_last fp32,
    depth (B,1,H,W) fp32 in metres or None).
    angles: None, or B rotation angles in degrees (PIL's convention, counter-clockwise): each frame is first rotated about
    its centre as Image.rotate(angle) does it (:122-125; bilinear image, nearest depth, 0 outside), bit for bit, and the
    crop window is cut from the rotated frame.  The frames are the ones after the fixed crops (bts_b200.data.fixed_crop)."""
    _need_cuda(img_u8, params)
    if img_u8.dtype != torch.uint8 or img_u8.dim() != 4 or img_u8.shape[3] != 3 or not img_u8.is_contiguous():
        raise ValueError("img_u8 must be a contiguous (B,Hs,Ws,3) uint8 tensor")
    B, Hs, Ws, _ = img_u8.shape
    H, W = out_hw
    params = params.contiguous().float()
    if tuple(params.shape) != (B, 9):
        raise ValueError("params must be (B,9)")
    img = torch.empty((B, 3, H, W), device=img_u8.device, dtype=torch.float32).contiguous(memory_format=torch.channels_last)
    dep = None
    if depth_u16 is not None:
        if depth_u16.dtype not in (torch.uint16, torch.int16) or tuple(depth_u16.shape) != (B, Hs, Ws):
            raise ValueError("depth_u16 must be (B,Hs,Ws) uint16")
        depth_u16 = depth_u16.contiguous()
        dep = torch.empty((B, 1, H, W), device=img_u8.device, dtype=torch.float32)
    if angles is None:
        _lib.check(_lib.lib().bts_input_prep(_ptr(img_u8), Hs, Ws, _ptr(depth_u16), float(depth_div), _ptr(params), B, H, W,
                                             _ptr(img), 3, _ptr(dep), _stream()), "bts_input_prep")
    else:
        angles = [float(a) for a in (angles.tolist() if torch.is_tensor(angles) else angles)]
        if len(angles) != B:
            raise ValueError("angles must hold one angle per sample (%d), got %d" % (B, len(angles)))
        affine = torch.tensor([data.rotate_affine(a, Ws, Hs) for a in angles], dtype=torch.float64).to(img_u8.device)
        _lib.check(_lib.lib().bts_input_prep_rotated(_ptr(img_u8), Hs, Ws, _ptr(depth_u16), float(depth_div), _ptr(params),
                                                     _ptr(affine), B, H, W, _ptr(img), 3, _ptr(dep), _stream()),
                   "bts_input_prep_rotated")
    _lib.count()
    return img, dep


def eval_errors(pred, gt, min_depth, max_depth, crop=None):
    """the nine eval metrics of one image + valid-pixel count, on the GPU (pytorch/bts_main.py:144-165,275-296).
    pred, gt: (H,W) fp32 CUDA; crop = (y0,y1,x0,x1) or None.  Returns a 10-float CUDA tensor (no host sync)."""
    _need_cuda(pred, gt)
    pred, gt = pred.contiguous().float(), gt.contiguous().float()
    H, W = pred.shape[-2], pred.shape[-1]
    if pred.numel() != H * W or gt.numel() != H * W:
        raise ValueError("eval_errors takes one image at a time")
    y0, y1, x0, x1 = crop if crop is not None else (0, H, 0, W)
    ws = torch.empty(10, device=pred.device, dtype=torch.float64)
    out = torch.empty(10, device=pred.device, dtype=torch.float32)
    _lib.check(_lib.lib().bts_eval_errors(_ptr(pred), _ptr(gt), H, W, float(min_depth), float(max_depth), int(y0), int(y1),
                                          int(x0), int(x1), _ptr(ws), _ptr(out), _stream()), "bts_eval_errors")
    _lib.count(2)
    return out


def depth_to_u16(depth, scale):
    """uint16(depth * scale): the 16-bit PNG wire format of bts_test.py:179-185 (scale 256 KITTI / 1000 NYU)"""
    _need_cuda(depth)
    depth = depth.contiguous().float()
    out = torch.empty(depth.shape, device=depth.device, dtype=torch.uint16)
    _lib.check(_lib.lib().bts_depth_to_u16(_ptr(depth), float(scale), depth.numel(), _ptr(out), _stream()), "bts_depth_to_u16")
    _lib.count()
    return out


_PNG_REASONS = {1: "truncated stream", 2: "bad zlib header", 3: "bad DEFLATE block", 4: "bad Huffman code table",
                5: "distance too far back", 6: "wrong decompressed size", 7: "Adler-32 mismatch", 8: "bad filter type"}


def decode_png(blobs, origins=None, out_hw=None):
    """Decodes a batch of PNG files on the current CUDA device and stream, cropped: what
    np.stack([np.asarray(Image.open(f))[y0:y0 + Hc, x0:x0 + Wc] ...]) gives, as (B, Hc, Wc, 3) uint8 for 8-bit RGB or
    (B, Hc, Wc) uint16 in native byte order for 16-bit grayscale (the inputs of input_prep).

    blobs: the files' bytes, all of one format.  origins: None or one (y0, x0) per file; out_hw: None or (Hc, Wc).
    Without out_hw every frame must have the same size and the window is the frame less its origin; with the training
    recipe the windows are data.fixed_crop_box(dataset, do_kb_crop, h, w).

    The container is checked on the host (data.parse_png) before anything reaches the device.  The streams go to the device
    in one pinned host-to-device copy, with one copy of the per-image metadata; bts_png_inflate and bts_png_unfilter run on
    the current stream.  The call then synchronises once, to read each image's status back: a stream that fails to decode
    raises ValueError naming the first failing image's index and reason, and leaves nothing behind."""
    blobs = list(blobs)
    if not blobs:
        raise ValueError("decode_png needs at least one PNG")
    parsed = [data.parse_png(b) for b in blobs]
    fmt, bpp = parsed[0][0], parsed[0][1]
    for i, p in enumerate(parsed):
        if p[0] != fmt:
            raise ValueError("decode_png takes one format per call: image 0 is %s, image %d is %s" % (fmt, i, p[0]))
    n = len(parsed)
    if origins is None:
        origins = [(0, 0)] * n
    origins = [(int(y), int(x)) for y, x in origins]
    if len(origins) != n:
        raise ValueError("origins must hold one (y0, x0) per image (%d), got %d" % (n, len(origins)))
    if out_hw is None:
        sizes = {p[2:4] for p in parsed}
        if len(sizes) != 1:
            raise ValueError("without out_hw every frame must have the same size, got %s" % sorted(sizes))
        h, w = sizes.pop()
        if len(set(origins)) != 1:
            raise ValueError("without out_hw every image must have the same origin")
        out_hw = (h - origins[0][0], w - origins[0][1])
    Hc, Wc = int(out_hw[0]), int(out_hw[1])
    meta = np.zeros((n, 8), dtype=np.int64)
    src_off = raw_off = 0
    for i, ((_, _, h, w, stream), (y0, x0)) in enumerate(zip(parsed, origins)):
        if Hc < 1 or Wc < 1 or y0 < 0 or x0 < 0 or y0 + Hc > h or x0 + Wc > w:
            raise ValueError("image %d: the crop (%d, %d, %d, %d) is outside its %dx%d frame" % (i, y0, x0, Hc, Wc, h, w))
        meta[i] = (src_off, len(stream), raw_off, h, w, y0, x0, 0)
        src_off += len(stream)
        raw_off += h * (1 + w * bpp)
    dev = torch.device("cuda", torch.cuda.current_device())
    host = torch.empty(max(src_off, 1), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for i, p in enumerate(parsed):
        hv[meta[i, 0]:meta[i, 0] + meta[i, 1]] = np.frombuffer(p[4], dtype=np.uint8)
    src = host.to(dev, non_blocking=True)
    meta_d = torch.from_numpy(meta).to(dev)
    raw = torch.empty(raw_off, dtype=torch.uint8, device=dev)
    work = torch.empty(2 * n, dtype=torch.int32, device=dev)   # status [n], stored Adler-32 [n]
    out = torch.empty((n, Hc, Wc, 3) if bpp == 3 else (n, Hc, Wc), dtype=torch.uint8 if bpp == 3 else torch.uint16,
                      device=dev)
    L = _lib.lib()
    status, adler = work[:n], work[n:]
    _lib.check(L.bts_png_inflate(_ptr(src), _ptr(meta_d), n, bpp, _ptr(raw), _ptr(adler), _ptr(status), _stream()),
               "bts_png_inflate")
    _lib.check(L.bts_png_unfilter(_ptr(raw), _ptr(meta_d), _ptr(adler), n, bpp, Hc, Wc, _ptr(out), _ptr(status),
                                  _stream()), "bts_png_unfilter")
    _lib.count(2)
    st = status.cpu().numpy()   # the one synchronisation of the call
    bad = np.nonzero(st)[0]
    if len(bad):
        i = int(bad[0])
        raise ValueError("decode_png: image %d: %s (status %d)" % (i, _PNG_REASONS.get(int(st[i]), "unknown"), int(st[i])))
    return out
