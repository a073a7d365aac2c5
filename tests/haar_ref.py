"""float32 and fp64 restatements of the one-level Haar kernels (include/wmd.h), in plain numpy / torch.

  idwt32  wmd_idwt_haar_f32's reconstruction: s ll, s lh (and s hl, s hh), then the sum or difference, then s again, then
          the sum or difference, every step rounded to float32 (the dependency's separable order, oracle/haar.py)
  dwt32   wmd_dwt_haar_f32 in the kernel's stated order: per input row s x0 +- s x1, then per column pair s lo0 +- s lo1
  dwt64   the same analysis in fp64, with S = 1/2 the sum of the four |x| of each output
  disp    torch.clamp(out * scale, 0, 1): a NaN stays NaN
numpy's float32 arithmetic rounds every operation and keeps subnormals, so these are the exact results of the kernels'
stated orders.  Independent of libwmd and ops.*.
"""
import numpy as np
import torch

S32 = np.float32(0.70710678118654752440)
S64 = 0.70710678118654752440
# dwt_haar's bound against fp64: |err| <= DWT_ULP 2^-24 S + DWT_FLOOR.  Four roundings on each path bound the relative part
# by 4 x 2^-24 S (twice that is the bar); a product that lands among the subnormals may also lose up to 2^-150 absolute,
# two in the row pass (carried by s = 1/sqrt2) and two in the column pass: 2^-150 (2 + 2 s) < 2 x 2^-149.
DWT_ULP = 8
DWT_FLOOR = 2 * 2.0 ** -149


def _np32(t):
    return t.detach().cpu().numpy().astype(np.float32, copy=False) if torch.is_tensor(t) else np.asarray(t, np.float32)


def synth32(ll, lh, hl, hh):
    """(y00, y01, y10, y11) of one Haar butterfly per element, float32, in the kernel's order."""
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        sll, slh, shl, shh = S32 * ll, S32 * lh, S32 * hl, S32 * hh
        lo0, lo1, hi0, hi1 = sll + slh, sll - slh, shl + shh, shl - shh
        a0, b0, a1, b1 = S32 * lo0, S32 * hi0, S32 * lo1, S32 * hi1
        return a0 + b0, a0 - b0, a1 + b1, a1 - b1


def idwt32(ll, hf):
    """ll (N, C, H, W), hf (N, C, 3, H, W) [LH, HL, HH] -> out (N, C, 2H, 2W) float32 torch tensor on the CPU."""
    ll, hf = _np32(ll), _np32(hf)
    y00, y01, y10, y11 = synth32(ll, hf[:, :, 0], hf[:, :, 1], hf[:, :, 2])
    n, c, h, w = ll.shape
    out = np.empty((n, c, 2 * h, 2 * w), np.float32)
    out[:, :, 0::2, 0::2], out[:, :, 0::2, 1::2], out[:, :, 1::2, 0::2], out[:, :, 1::2, 1::2] = y00, y01, y10, y11
    return torch.from_numpy(out)


def dwt32(x):
    """x (N, C, H, W), H and W even -> (ll (N, C, H/2, W/2), hf (N, C, 3, H/2, W/2)) float32 torch tensors on the CPU."""
    x = _np32(x)
    x00, x01, x10, x11 = x[:, :, 0::2, 0::2], x[:, :, 0::2, 1::2], x[:, :, 1::2, 0::2], x[:, :, 1::2, 1::2]
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        lo0, hi0 = S32 * x00 + S32 * x01, S32 * x00 - S32 * x01
        lo1, hi1 = S32 * x10 + S32 * x11, S32 * x10 - S32 * x11
        ll = S32 * lo0 + S32 * lo1
        hf = np.stack([S32 * lo0 - S32 * lo1, S32 * hi0 + S32 * hi1, S32 * hi0 - S32 * hi1], 2)
    return torch.from_numpy(np.ascontiguousarray(ll)), torch.from_numpy(np.ascontiguousarray(hf))


def dwt64(x):
    """(ll, hf, S) of the analysis in fp64; S (N, C, H/2, W/2) = 1/2 the sum of the four |x| each output mixes."""
    x = x.detach().double().cpu()
    x00, x01, x10, x11 = x[:, :, 0::2, 0::2], x[:, :, 0::2, 1::2], x[:, :, 1::2, 0::2], x[:, :, 1::2, 1::2]
    ll = 0.5 * (x00 + x01 + x10 + x11)
    hf = torch.stack([0.5 * (x00 + x01 - x10 - x11), 0.5 * (x00 - x01 + x10 - x11), 0.5 * (x00 - x01 - x10 + x11)], 2)
    return ll, hf, 0.5 * (x00.abs() + x01.abs() + x10.abs() + x11.abs())


def disp(out, scale, clamp01):
    """[torch.clamp](out * scale, 0, 1) in float32 on out's device: the scale rounded to float32 first, as the kernels take
    it."""
    v = out * torch.tensor(float(scale), dtype=torch.float32, device=out.device)
    return torch.clamp(v, 0.0, 1.0) if clamp01 else v


def same_bits(got, want):
    """NaN exactly where want is NaN, every other element bit-identical (so +-Inf and the sign of zero too)."""
    got, want = got.detach().cpu().float(), want.detach().cpu().float()
    if got.shape != want.shape:
        return False
    nan = torch.isnan(want)
    if not torch.equal(torch.isnan(got), nan):
        return False
    return torch.equal(got.view(torch.int32)[~nan], want.view(torch.int32)[~nan])


def same_values(got, want):
    """NaN exactly where want is NaN, every other element equal in value (-0.0 == 0.0: the clamped planes, whose zero sign
    torch's own CPU and CUDA clamps may disagree on)."""
    got, want = got.detach().cpu().float(), want.detach().cpu().float()
    if got.shape != want.shape:
        return False
    nan = torch.isnan(want)
    return torch.equal(torch.isnan(got), nan) and torch.equal(got[~nan], want[~nan])
