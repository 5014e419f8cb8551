"""N1: JPEG decode on the device in place of the loader's host decode (voc12/dataloader.py:101).

``ExactJpegDecoder`` (``--device_jpeg True``): our own kernels (csrc/jpeg_exact.cu, include/irn_b200.h irn_jpeg_exact_*), bit-identical
to ``np.asarray(Image.open(f).convert("RGB"))`` on libjpeg-turbo for the baseline streams ``inspect`` accepts; images of any sizes in
one call."""
import ctypes
from collections import deque

import numpy as np
import torch

from . import _lib


class UnsupportedJpeg(_lib.IrnError):
    """A stream outside the exact decoder's supported set (progressive, arithmetic, 12-bit, CMYK / RGB, other samplings, DNL)."""


def _buf(data):
    if isinstance(data, torch.Tensor):
        return data.numpy()
    return data if isinstance(data, np.ndarray) else np.frombuffer(data, dtype=np.uint8)


def inspect(data):
    """Header of one JPEG stream, host only (no GPU needed): (H, W, components, luma h sampling, luma v sampling, restart
    interval).  Raises UnsupportedJpeg for a stream the exact decoder does not take, IrnError for a malformed or truncated header."""
    buf = _buf(data)
    info = (ctypes.c_int * 6)()
    rc = _lib.lib().irn_jpeg_exact_inspect(buf.ctypes.data, buf.size, info)
    if rc == -4:
        raise UnsupportedJpeg("unsupported JPEG stream: %s" % _lib.lib().irn_last_error().decode())
    _lib.check(rc, "irn_jpeg_exact_inspect")
    return tuple(info)


class DecodeStatus:
    """The per-image status words of one exact decode, copied to pinned host memory in stream order.  `check()` reads them: call it
    once the stream has passed the decode (after an event recorded later on the same stream); raises IrnError naming the first bad
    image."""

    _BITS = {1: "stray marker", 2: "missing or surplus restart marker", 4: "invalid Huffman code", 8: "entropy-coded data ends early",
             16: "AC run past the block"}

    def __init__(self, status_host, names):
        self.status, self.names = status_host, names

    def check(self):
        st = self.status.numpy()
        for i in np.flatnonzero(st):
            why = ", ".join(v for k, v in self._BITS.items() if int(st[i]) & k)
            raise _lib.IrnError("exact JPEG decode of %s failed: %s (status 0x%x)" % (self.names[i], why, int(st[i])))


class ExactJpegDecoder:
    """Exact device decode of JPEG file bytes (see the module docstring).  Images of any sizes go in one call; the work is enqueued on
    the current stream.  The host work is header parsing and one staging copy of the entropy-coded bytes."""

    inspect = staticmethod(inspect)

    def __init__(self, device):
        self.device = torch.device(device)
        self._inflight = deque()      # (event, pinned staging) of decodes whose upload may not have run yet

    def decode_into(self, streams, offsets, out, names=None):
        """Decode streams of any sizes into the device uint8 buffer `out`, image i's [H_i,W_i,3] RGB bytes at offsets[i] (host
        int64).  Returns the DecodeStatus to check once the stream has passed the decode."""
        bufs = [_buf(s) for s in streams]
        n = len(bufs)
        if n == 0:
            raise _lib.IrnError("ExactJpegDecoder: empty batch")
        L = _lib.lib()
        ptrs = (ctypes.c_void_p * n)(*[b.ctypes.data for b in bufs])
        lens = (ctypes.c_size_t * n)(*[b.size for b in bufs])
        dev_bytes, host_bytes = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.irn_jpeg_exact_workspace_bytes(ptrs, lens, n, ctypes.byref(dev_bytes), ctypes.byref(host_bytes)),
                   "irn_jpeg_exact_workspace_bytes")
        while self._inflight and self._inflight[0][0].query():
            self._inflight.popleft()
        staging = torch.empty(max(host_bytes.value, 1), dtype=torch.uint8, pin_memory=True)
        ws = torch.empty(dev_bytes.value, dtype=torch.uint8, device=self.device)
        status = torch.empty(n, dtype=torch.int32, device=self.device)
        offs = np.ascontiguousarray(offsets, dtype=np.int64)
        with torch.cuda.device(self.device):
            _lib.check(L.irn_jpeg_exact_decode(ptrs, lens, n, offs.ctypes.data, _lib.ptr(out), _lib.ptr(status), _lib.ptr(ws), dev_bytes.value,
                                               staging.data_ptr(), host_bytes.value, _lib.stream_ptr()), "irn_jpeg_exact_decode")
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.device))
            self._inflight.append((ev, staging))
            status_host = torch.empty(n, dtype=torch.int32, pin_memory=True)
            status_host.copy_(status, non_blocking=True)
        return DecodeStatus(status_host, list(names) if names is not None else ["image %d" % i for i in range(n)])

    def _sizes(self, streams):
        return [inspect(s)[:2] for s in streams]

    def decode_packed(self, streams, names=None, check=True):
        """streams: bytes-like / uint8 arrays / uint8 CPU tensors of JPEG files of any sizes.  Returns (flat uint8 cuda, [(H_i, W_i)]),
        image i's [H_i,W_i,3] RGB bytes back to back in order: StepContext.pack_images' layout.  check=True waits for the decode and
        raises on a bad image; check=False returns a third value, the DecodeStatus to check later."""
        sizes = self._sizes(streams)
        nbytes = [3 * h * w for h, w in sizes]
        offs = np.concatenate([[0], np.cumsum(nbytes)[:-1]]).astype(np.int64)
        out = torch.empty(int(sum(nbytes)), dtype=torch.uint8, device=self.device)
        st = self.decode_into(streams, offs, out, names)
        if not check:
            return out, sizes, st
        torch.cuda.current_stream(self.device).synchronize()
        st.check()
        return out, sizes

    def decode(self, streams, names=None, check=True):
        """JPEG files of ONE size -> uint8 cuda [n,H,W,3] RGB (check as in decode_packed)."""
        sizes = self._sizes(streams)
        if len(set(sizes)) != 1:
            raise _lib.IrnError("ExactJpegDecoder.decode: images of different sizes %s (decode_packed takes them)" % sorted(set(sizes)))
        (H, W), n = sizes[0], len(sizes)
        out = torch.empty((n, H, W, 3), dtype=torch.uint8, device=self.device)
        st = self.decode_into(streams, np.arange(n, dtype=np.int64) * (3 * H * W), out, names)
        if not check:
            return out, st
        torch.cuda.current_stream(self.device).synchronize()
        st.check()
        return out
