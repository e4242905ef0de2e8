"""Poisoned device buffers for kernel tests (test_gpu_gemm.py, test_gpu_graph_kernels.py).

Inputs are views inside NaN-filled allocations (row stride past the extent, rows and slack past the end), so an over-read shows
up as NaN in a result; outputs are views inside sentinel-filled allocations, so an over-write shows up as a broken sentinel
(Region.outside_intact)."""
import subprocess

import torch

DEV = "cuda:0"
SENT = -7777.25  # output sentinel
NAN = float("nan")


def ceil4(n):
    return (n + 3) // 4 * 4


class Region:
    """A [rows, cols] view with row stride ld inside a device allocation filled with `fill`: columns past cols, two rows past
    the view and some slack after them hold `fill`; `shift` elements precede the view."""

    def __init__(self, rows, cols, ld, fill, shift=0, dtype=torch.float32):
        self.shape, self.fill = (rows, cols, ld, shift), fill
        self.buf = torch.full((shift + (rows + 2) * ld + 7,), fill, dtype=dtype, device=DEV)
        self.view = self._view(self.buf)
        self.ld = ld

    def _view(self, buf):
        rows, cols, ld, shift = self.shape
        return buf[shift:shift + rows * ld].view(rows, ld)[:, :cols]

    def ptr(self):
        return self.view.data_ptr()

    def outside_intact(self):
        c = self.buf.clone()
        self._view(c).fill_(self.fill)
        return bool((c == self.fill).all())


def filled(t, ld=None, fill=NAN, shift=0):
    """CPU tensor [rows, cols] copied into a Region filled with `fill` (row stride ld, default cols)."""
    t = t if t.dim() == 2 else t.reshape(t.shape[0], -1)
    r = Region(t.shape[0], t.shape[1], t.shape[1] if ld is None else ld, fill, shift=shift, dtype=t.dtype)
    r.view.copy_(t)
    return r


def operand(t, kc, pad=4, shift=0):
    """Logical [R, K] operand (CPU fp32) stored reduction-contiguous (kc) or as its transpose, in a NaN-poisoned region."""
    s = t if kc else t.t()
    r = Region(s.shape[0], s.shape[1], ceil4(s.shape[1]) + pad, NAN, shift=shift)
    r.view.copy_(s)
    return r


def zeroed(rows, cols, ld, dtype=torch.float32):
    r = Region(rows, cols, ld, SENT, dtype=dtype)
    r.view.zero_()
    return r


def card():
    """Name and power limit of the card the measurements were taken on."""
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return dict(card=name, power_limit=pl)
