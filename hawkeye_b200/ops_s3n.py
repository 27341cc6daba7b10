"""Autograd bindings for S3N (reference model/methods/S3N.py): the sampler that turns the class response maps into the two
31x31 sampling maps, the grid of each map and the image warp.  Host plumbing only; all arithmetic is in libhawkeye_b200.so.

The reference finds the peaks and builds the maps in a Python loop over images and peaks, with a host read of every score
(S3N.py:193-270); here one launch covers the batch and nothing is read back, so a training step never synchronises."""
import torch
from torch.autograd import Function

from . import _lib
from .ops import _check_cuda, _f32c, _ws

GRID = 31                   # grid_size (S3N.py:124)
PAD = 30                    # padding_size (S3N.py:125)


class SampleMapsFn(Function):
    """crm NHWC [N, h, w, K] (no gradient), rnd [N, 961], p int32 [1], radius [1], radius_inv [1] -> maps [2N, 31, 31]: the
    zoom maps, then the complementary maps (hk_s3n_sample_maps).  Differentiable in radius and radius_inv."""

    @staticmethod
    def forward(ctx, crm, rnd, p, radius, radius_inv, base_ratio):
        _check_cuda(crm, rnd, p, radius, radius_inv)
        crm, rnd = _f32c(crm), _f32c(rnd)
        N, h, w, K = crm.shape
        dev = crm.device
        maps = torch.empty(2 * N, GRID, GRID, device=dev, dtype=torch.float32)
        peaks = torch.empty(N, GRID * GRID, device=dev, dtype=torch.int32)
        scores = torch.empty(N, GRID * GRID, device=dev, dtype=torch.float32)
        counts = torch.empty(N, device=dev, dtype=torch.int32)
        radius, radius_inv = _f32c(radius), _f32c(radius_inv)
        _lib.call('hk_s3n_sample_maps', crm, rnd, p.to(torch.int32), radius, radius_inv, float(base_ratio), maps, peaks,
                  scores, counts, N, h, w, K, _lib.stream_ptr())
        ctx.save_for_backward(peaks, scores, counts, radius, radius_inv)
        ctx.mark_non_differentiable(peaks, scores, counts)
        return maps, peaks, scores, counts

    @staticmethod
    def backward(ctx, dmaps, _dpeaks, _dscores, _dcounts):
        peaks, scores, counts, radius, radius_inv = ctx.saved_tensors
        dr, dri = torch.empty_like(radius), torch.empty_like(radius_inv)
        _lib.call('hk_s3n_sample_maps_bwd', _f32c(dmaps), peaks, scores, counts, radius, radius_inv, dr, dri,
                  counts.shape[0], _lib.stream_ptr())
        return None, None, None, dr, dri, None


def sample_maps(crm, rnd, p, radius, radius_inv, base_ratio):
    """-> (maps [2N, 31, 31], the peak record (peaks, scores, counts), see hk_s3n_sample_maps)."""
    maps, peaks, scores, counts = SampleMapsFn.apply(crm, rnd, p, radius, radius_inv, base_ratio)
    return maps, (peaks, scores, counts)


class GridFn(Function):
    """maps [B, 31, 31], filter [1, 1, 61, 61] -> coarse grid [B, 31, 31, 2] (create_grid before its F.interpolate,
    S3N.py:156-183, on the replication-padded map)."""

    @staticmethod
    def forward(ctx, maps, filt):
        _check_cuda(maps, filt)
        maps, filt = _f32c(maps), _f32c(filt)
        B = maps.shape[0]
        grid = torch.empty(B, GRID, GRID, 2, device=maps.device, dtype=torch.float32)
        sums = torch.empty(B, GRID, GRID, 3, device=maps.device, dtype=torch.float32)
        _lib.call('hk_s3n_grid_fwd', maps, filt, grid, sums, B, _lib.stream_ptr())
        ctx.save_for_backward(maps, filt, sums)
        return grid

    @staticmethod
    def backward(ctx, dgrid):
        maps, filt, sums = ctx.saved_tensors
        B = maps.shape[0]
        dmaps, dfilt = torch.empty_like(maps), torch.empty_like(filt)
        ws = _ws(_lib.query('hk_s3n_grid_bwd_workspace_bytes', B), maps.device)
        _lib.call('hk_s3n_grid_bwd', maps, filt, sums, _f32c(dgrid), dmaps, dfilt, B, ws, ws.numel(), _lib.stream_ptr())
        return dmaps, dfilt


class WarpFn(Function):
    """x NCHW [N, C, H, W] (no gradient), grid [B, 31, 31, 2] -> [B, C, H, W]: image b % N sampled at the grid upsampled to
    H x W (S3N.py:186 and F.grid_sample, :274/:279).  Differentiable in the grid."""

    @staticmethod
    def forward(ctx, x, grid):
        _check_cuda(x, grid)
        x, grid = _f32c(x), _f32c(grid)
        N, C, H, W = x.shape
        B = grid.shape[0]
        out = torch.empty(B, C, H, W, device=x.device, dtype=torch.float32)
        _lib.call('hk_s3n_warp_fwd', x, grid, out, N, B, C, H, W, H, W, _lib.stream_ptr())
        ctx.save_for_backward(x, grid)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, grid = ctx.saved_tensors
        N, C, H, W = x.shape
        B = grid.shape[0]
        dgrid = torch.empty_like(grid)
        ws = _ws(_lib.query('hk_s3n_warp_bwd_workspace_bytes', B, H, W), x.device)
        _lib.call('hk_s3n_warp_bwd', x, grid, _f32c(dout), dgrid, N, B, C, H, W, H, W, ws, ws.numel(), _lib.stream_ptr())
        return None, dgrid


def sample_images(x, crm, rnd, p, radius, radius_inv, filt, base_ratio):
    """generate_map (S3N.py:193-284): x [N, 3, H, W] -> (zoomed images [N, 3, H, W], complementary images [N, 3, H, W])."""
    maps, _ = sample_maps(crm, rnd, p, radius, radius_inv, base_ratio)
    sampled = WarpFn.apply(x.detach(), GridFn.apply(maps, filt))
    N = x.shape[0]
    return sampled[:N], sampled[N:]
