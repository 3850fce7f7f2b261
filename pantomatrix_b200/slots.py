"""What the GPU encoders (png, video, flac) share: their frame input, their output slots and the copy of the slots'
used bytes to the host (DESIGN.md section 11).

An encoder writes item i into row i of a (n, cap) uint8 slot tensor and its byte count into nbytes[i]; cap is at
least the encoder's size bound and a multiple of 4, since the kernels write 32-bit words."""
from __future__ import annotations

import torch


def frames(x):
    """Checks frames (N, H, W, 3) or (B, T, H, W, 3) uint8 CUDA, each frame dense, clips evenly spaced, frames not
    overlapping.  Returns the (N, H, W, 3) view of the same memory (N = B T) and the clip length (T, or N for
    (N, ...) input; at least 1).  Raises ValueError otherwise; each encoder then checks its own size rule."""
    if not torch.is_tensor(x):
        raise ValueError(f"frames must be a tensor, got {type(x).__name__}")
    if not x.is_cuda:
        raise ValueError("frames must be a CUDA tensor")
    if x.dtype != torch.uint8:
        raise ValueError(f"frames must be uint8, got {x.dtype}")
    if x.dim() not in (4, 5) or x.shape[-1] != 3 or x.shape[-2] < 1 or x.shape[-3] < 1:
        raise ValueError(f"frames must be (N, H, W, 3) or (B, T, H, W, 3) with H, W >= 1, got {tuple(x.shape)}")
    h, w = x.shape[-3:-1]
    if x.stride(-1) != 1 or x.stride(-2) != 3 or x.stride(-3) != 3 * w:
        raise ValueError("frames: each frame must be dense")
    clip_len = x.shape[-4]
    if x.dim() == 5:
        b, t = x.shape[:2]
        if b > 1 and t > 1 and x.stride(0) != t * x.stride(1):
            raise ValueError("frames (B, T, H, W, 3): the clips' frames must be evenly spaced")
        fs = x.stride(1) if t > 1 else x.stride(0)
        x = x.as_strided((b * t, h, w, 3), (fs, 3 * w, 3, 1))
    if x.shape[0] > 1 and x.stride(0) < 3 * h * w:
        raise ValueError("frames: frames must not overlap")
    return x, max(clip_len, 1)


def output(n: int, need: int, slot: int, device, out):
    """The (data, nbytes) pair an encoder of n items fills: new (n, slot) uint8 and (n,) int64 tensors on device when
    out is None, else out itself once checked: data (n, cap) uint8 contiguous with cap >= need and a multiple of 4,
    nbytes (n,) int64 contiguous, both on device.  Raises ValueError on any other out."""
    if out is None:
        return (torch.empty(n, slot, dtype=torch.uint8, device=device),
                torch.empty(n, dtype=torch.int64, device=device))
    data, nbytes = out
    if not (torch.is_tensor(data) and data.device == device and data.dtype == torch.uint8 and data.dim() == 2
            and data.shape[0] == n and data.shape[1] >= need and data.shape[1] % 4 == 0 and data.is_contiguous()):
        raise ValueError(f"out data must be a contiguous ({n}, cap) uint8 tensor on {device} with cap >= "
                         f"{need} a multiple of 4")
    if not (torch.is_tensor(nbytes) and nbytes.device == device and nbytes.dtype == torch.int64
            and tuple(nbytes.shape) == (n,) and nbytes.is_contiguous()):
        raise ValueError(f"out nbytes must be a contiguous ({n},) int64 tensor on {device}")
    return data, nbytes


def to_host(*pairs):
    """The used bytes of slot tensors on one device: each pair (data, sizes) gives data[i, :sizes[i]] for the host
    ints sizes.  Every item goes straight from its slot into one pinned host buffer by a non-blocking copy on the
    current stream, and that stream is synchronised once, so copies queued on it before the call are done as well.
    Returns one list of memoryviews per pair."""
    host = torch.empty(sum(sum(sizes) for _, sizes in pairs), dtype=torch.uint8, pin_memory=True)
    at = 0
    for data, sizes in pairs:
        for i, k in enumerate(sizes):
            host[at:at + k].copy_(data[i, :k], non_blocking=True)
            at += k
    torch.cuda.current_stream(pairs[0][0].device).synchronize()
    flat = memoryview(host.numpy())
    out, at = [], 0
    for _, sizes in pairs:
        views = []
        for k in sizes:
            views.append(flat[at:at + k])
            at += k
        out.append(views)
    return out
