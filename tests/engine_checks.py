"""Checks shared by the engine parity tests (test_wgrad_engines_gpu.py, test_conv_engine_gpu.py, test_conv_engine_cpu.py):
NaN-guarded output buffers, NHWC channel slices, the names and template arguments of the kernels a profiled region
launched, and the fp64 CPU reference of the forward / dgrad engine (csrc/conv_tc.cu), full or sampled per 128-pixel
m-tile, with the shapes of the persistent-walk cases sized on a GPU's SM count."""
import math
import re

import torch
import torch.nn.functional as F

GUARD = 64              # NaN floats on each side of a guarded view
BLOCK_M = 128           # output pixels per m-tile of conv_tc_kernel


# ----------------------------------------------------------------------------------------------- buffers and launches
def template_arg(a):
    a = re.sub(r"^\((int|bool)\)", "", a.strip())           # '(bool)1' / 'true' / '1', whichever demangler named it
    return {"true": 1, "false": 0}[a] if a in ("true", "false") else int(a)


def kernels(prof, names=r"wgrad2?_tc_kernel|conv_tc_kernel"):
    """(name, template arguments as ints) of every kernel matching `names` the profiled region launched"""
    out = []
    for e in prof.events():
        m = re.search(r"(%s)<([^<>]*)>" % names, e.name)
        if m:
            out.append((m.group(1), tuple(template_arg(a) for a in m.group(2).split(","))))
            continue
        m = re.search(r"(%s)I((?:L[ib]\d+E)+)E" % names, e.name)       # a name left mangled
        if m:
            out.append((m.group(1), tuple(int(a) for a in re.findall(r"L[ib](\d+)E", m.group(2)))))
    return out


def ran(ks, name, args=()):
    """the profiled call launched `name` once (and no other kernel of those recorded) with template arguments starting
    with `args`.  CUPTI now and then delivers no kernel record for a profiled region this short; there is then nothing
    to compare, and the numerical checks of the test stand alone."""
    if not ks:
        return True
    return [n for n, _ in ks] == [name] and ks[0][1][:len(args)] == tuple(int(a) for a in args)


def nan(n):
    return torch.full((n,), float("nan"), device="cuda")


def guarded(shape, strides, offset=0):
    """a NaN-filled view of `shape` with `strides`, starting `offset` floats past GUARD NaN floats, inside a larger
    NaN-filled buffer: (view, buffer, membership mask)"""
    extent = offset + 1 + sum((n - 1) * s for n, s in zip(shape, strides))
    buf = nan(extent + 2 * GUARD)
    inside = torch.zeros(buf.numel(), dtype=torch.bool, device="cuda")
    inside.as_strided(shape, strides, GUARD + offset).fill_(True)
    assert int(inside.sum()) == torch.Size(shape).numel()          # the layout does not alias
    return buf.as_strided(shape, strides, GUARD + offset), buf, inside


def check_written(v, buf, inside):
    assert bool(torch.isfinite(v).all()), "the view has %d non-finite elements" % int((~torch.isfinite(v)).sum())
    assert bool(torch.isnan(buf[~inside]).all()), "a write landed outside the view"


def guarded_nhwc(B, C, H, W, width=None, off=1):
    """(B, C, H, W) as the channel slice [off, off + C) of a NaN-filled NHWC slab `width` channels wide (default: one
    guard channel on each side), inside a NaN-filled buffer: (view, buffer, membership mask)"""
    width = C + off + 1 if width is None else width
    assert off >= 1 and width > off + C
    return guarded((B, C, H, W), (H * W * width, 1, W * width, width), off)


def nhwc_slice(t, width=None, off=0):
    """t on the GPU, NHWC in memory, as the channel slice [off, off + C) of a slab `width` channels wide (other channels
    hold unrelated values)"""
    B, C, H, W = t.shape
    width = C if width is None else width
    slab = torch.randn(B, width, H, W).cuda().contiguous(memory_format=torch.channels_last)
    v = slab[:, off:off + C]
    v.copy_(t)
    return v


# ---------------------------------------------------------------------------------- fp64 reference of conv_tc_kernel
class Op:
    """one call of the forward / dgrad engine as the kernel sees it: the source x (B, Cin, Hs, Ws), the pre-op
    pre(x) = [relu](x * scale + shift) per input channel, then the source mode (0: as is, 1: nearest x2 up-sample, 2:
    zero-stuffed x2 expansion, value at (2i, 2j) = pre(x)[i, j] and zeros elsewhere, read at an explicit output size),
    then conv2d at (stride, pad, dil) with the operator `w` and the activation (None, 'elu', 'sigmoid').  `weight` is the
    layer's parameter as conv.conv2d_tc takes it; a dgrad (transpose_flip) runs the operator w = weight transposed and
    tap-flipped, at pad = dil * (k - 1) - the layer's padding."""

    def __init__(self, weight, stride=1, pad=0, dil=1, scale=None, shift=None, relu=False, mode=0, out_hw=None, act=None,
                 groups=1, transpose_flip=False):
        self.weight, self.stride, self.pad, self.dil = weight, stride, pad, dil
        self.scale, self.shift, self.relu, self.mode, self.out_hw, self.act = scale, shift, relu, mode, out_hw, act
        self.groups, self.transpose_flip = groups, transpose_flip
        self.w = weight.transpose(0, 1).flip(2, 3) if transpose_flip else weight

    @property
    def pre(self):
        return (2 if self.scale is not None else 0) | (1 if self.relu else 0)

    def out_size(self, Hs, Ws):
        if self.mode == 2:
            return self.out_hw
        k, d = self.w.shape[2], self.dil
        Hv, Wv = (2 * Hs, 2 * Ws) if self.mode == 1 else (Hs, Ws)
        return (Hv + 2 * self.pad - d * (k - 1) - 1) // self.stride + 1, (Wv + 2 * self.pad - d * (k - 1) - 1) // self.stride + 1

    def pre_op(self, x):
        """pre(x) in fp64, channels on dim 1"""
        x = x.double()
        if self.scale is not None:
            shp = (1, -1) + (1,) * (x.dim() - 2)
            x = x * self.scale.double().cpu().view(shp) + self.shift.double().cpu().view(shp)
        return F.relu(x) if self.relu else x

    def activate(self, y):
        if self.act == "elu":
            return F.elu(y)
        if self.act == "sigmoid":
            return torch.sigmoid(y)
        return y

    def full(self, x):
        """fp64 reference of the whole output, on the CPU"""
        B, C, Hs, Ws = x.shape
        s = self.pre_op(x.cpu())
        if self.mode == 1:
            s = F.interpolate(s, scale_factor=2, mode="nearest")
        elif self.mode == 2:
            z = torch.zeros(B, C, 2 * Hs, 2 * Ws, dtype=torch.float64)
            z[:, :, ::2, ::2] = s                      # the stuffed zeros stay zero whatever the pre-op's shift
            s = z
        y = F.conv2d(s, self.w.double().cpu(), None, self.stride, self.pad, self.dil, self.groups)
        Ho, Wo = self.out_size(Hs, Ws)
        assert y.shape[2] >= Ho and y.shape[3] >= Wo
        return self.activate(y[:, :, :Ho, :Wo])

    def sample(self, x, m, chunk=4096):
        """fp64 reference of all output channels at the output pixels m = (b * Hout + y) * Wout + x (a 1-D integer
        tensor), from the input window of each pixel gathered on x's device: (len(m), Cout) on the CPU"""
        B, C, Hs, Ws = x.shape
        Ho, Wo = self.out_size(Hs, Ws)
        k = self.w.shape[2]
        Hv, Wv = (Hs, Ws) if self.mode == 0 else (2 * Hs, 2 * Ws)
        w = self.w.double().cpu()
        if self.groups > 1:                            # block-diagonal dense operator
            cpg, co = C // self.groups, w.shape[0] // self.groups
            wd = torch.zeros(w.shape[0], C, k, k, dtype=torch.float64)
            for g in range(self.groups):
                wd[g * co:(g + 1) * co, g * cpg:(g + 1) * cpg] = w[g * co:(g + 1) * co]
            w = wd
        w = w.reshape(w.shape[0], C, k * k)
        ky, kx = torch.meshgrid(torch.arange(k), torch.arange(k), indexing="ij")
        ky, kx = ky.reshape(-1) * self.dil, kx.reshape(-1) * self.dil
        xn = x.permute(0, 2, 3, 1)                      # (B, Hs, Ws, C) view of the NHWC memory
        outs = []
        for m0 in range(0, m.numel(), chunk):
            mm = m[m0:m0 + chunk].long()
            b, r = mm // (Ho * Wo), mm % (Ho * Wo)
            oy, ox = r // Wo, r % Wo
            vy = (oy * self.stride - self.pad)[:, None] + ky[None]            # (P, taps) virtual source coordinates
            vx = (ox * self.stride - self.pad)[:, None] + kx[None]
            ok = (vy >= 0) & (vy < Hv) & (vx >= 0) & (vx < Wv)
            if self.mode == 2:
                ok &= (vy % 2 == 0) & (vx % 2 == 0)
            sy, sx = (vy, vx) if self.mode == 0 else (vy.div(2, rounding_mode="floor"), vx.div(2, rounding_mode="floor"))
            sy, sx = sy.clamp(0, Hs - 1), sx.clamp(0, Ws - 1)
            bb = b[:, None].expand_as(sy)
            dev = x.device
            win = xn[bb.to(dev), sy.to(dev), sx.to(dev)].cpu()                 # (P, taps, C) fp32
            win = self.pre_op(win.permute(0, 2, 1)) * ok[:, None, :]           # padding after the pre-op
            outs.append(self.activate(torch.einsum("pct,oct->po", win, w)))
        return torch.cat(outs)


def sample_pixels(M, per_tile=2, seed=0):
    """per_tile distinct output pixels of every 128-pixel m-tile, the partial last tile included, in the engine's pixel
    order: the first and last pixel of the tile and seeded ones between"""
    g = torch.Generator().manual_seed(seed)
    tiles = -(-M // BLOCK_M)
    base = torch.arange(tiles) * BLOCK_M
    live = (M - base).clamp(max=BLOCK_M)
    picks = [base, base + live - 1]
    for _ in range(per_tile - 2):
        picks.append(base + (torch.rand(tiles, generator=g) * live).long())
    return torch.unique(torch.cat(picks))


def pixels_of(y, m):
    """(len(m), C) values of the (B, C, H, W) tensor y at output pixels m = (b * H + y) * W + x"""
    B, C, H, W = y.shape
    m = m.to(y.device).long()
    return y.permute(0, 2, 3, 1)[m // (H * W), (m % (H * W)) // W, m % W].cpu()


def rel_err(got, ref):
    return float((got.detach().cpu().double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------ persistent walks
def n_tile(Cout):
    """bts_conv_n_tile through the library (loads without a GPU)"""
    from bts_b200 import _lib
    return int(_lib.lib().bts_conv_n_tile(int(Cout)))


def kblocks(Kch, k):
    """k-blocks per tile: 16-byte channel quads, tap-major, 8 to a k-block"""
    return -(-(k * k * -(-Kch // 4)) // 8)


def walk_rows(G, n_tiles, B, W, even=False, target=2.5):
    """the first output height H (even if asked) from about target * G tiles (m_tiles * n_tiles) upwards at which
    M = B * H * W is not a multiple of 128 and the tile count is not a multiple of G, so the G CTAs walk unequal numbers
    of tiles"""
    H = max(2, round(target * G * BLOCK_M / (n_tiles * B * W)))
    while True:
        M = B * H * W
        if not (even and H % 2) and M % BLOCK_M and (-(-M // BLOCK_M) * n_tiles) % G:
            return H
        H += 1


# name -> layer of a persistent-walk case: B, Cin (the operator's K channels), output W, Cout (the output width), k,
# and what it exercises.  The output height comes from walk_rows for the GPU's SM count.
WALKS = {
    "kb1_stats": dict(B=2, Cin=24, W=53, Cout=48, k=1),          # KB = 1: each producer group fills whole tiles in turn
    "kb_odd": dict(B=2, Cin=36, W=53, Cout=32, k=3),             # KB = 11: the group filling k-block 0 alternates
    "kb_even": dict(B=2, Cin=64, W=53, Cout=48, k=3),            # KB = 18
    "nt_coprime": dict(B=1, Cin=20, W=29, Cout=560, k=3),        # 5 n-tiles of 112: the n-tile changes along a walk
    "nt_divides": dict(B=1, Cin=40, W=37, Cout=192, k=3),        # 2 n-tiles of 96: it stays constant along a walk
    "bnbwd": dict(B=2, Cin=48, W=37, Cout=192, k=3),             # dgrad 48 -> 192 with the BatchNorm-backward epilogue
    "zero_stuffed": dict(B=2, Cin=40, W=45, Cout=64, k=3),       # dgrad of a stride-2 3x3 64 -> 40
    "grouped": dict(B=1, Cin=256, W=29, Cout=256, k=3),          # ResNeXt 3x3, 32 groups of 8: 2 n-tiles of 128
    "act": dict(B=2, Cin=32, W=53, Cout=32, k=3),                # ELU / sigmoid epilogue
    "odd_slice": dict(B=2, Cin=40, W=53, Cout=48, k=3),          # output at an odd channel offset: scalar stores
    "ring3": dict(B=1, Cin=2300, W=97, Cout=128, k=1),           # 3-stage smem ring (see ring_stages)
}


def walk_shape(name, G):
    c = WALKS[name]
    grouped = name == "grouped"                       # one 128-channel K window per n-tile of 128 rows
    nt = 128 if grouped else n_tile(c["Cout"])
    n_tiles = -(-c["Cout"] // nt)
    H = walk_rows(G, n_tiles, c["B"], c["W"])
    M = c["B"] * H * c["W"]
    return dict(c, H=H, M=M, n_tile=nt, n_tiles=n_tiles, tiles=-(-M // BLOCK_M) * n_tiles,
                KB=kblocks(128 if grouped else c["Cin"], c["k"]))


def ring_stages(Cin, n_tile, stats, affine):
    """smem stages of conv_tc_kernel (conv_fwd_impl's plan): as many 16 KB A + 2 x n_tile x 128 B stages as fit in
    227 KB next to the pre-op's scale / shift, the barriers and the per-warp fp64 statistics, at most 6"""
    stage = 16384 + 2 * n_tile * 128
    pre = -(-Cin // 32) * 32 * 8 if affine else 0
    st = 8 * 2 * n_tile * 8 if stats else 0
    return min(6, (232448 - 1024 - 256 - pre - st) // stage)


def coprime(a, b):
    return math.gcd(a, b) == 1
