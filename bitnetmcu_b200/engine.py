"""Host-side mirror of the reference interface for the hot path, on top of the C ABI.

Reference                                              here
-------------------------------------------------------------------------------------------------
lib.Inference(ptr) per image (test_inference.py:146)   Engine.infer(images) / Engine.inference(image)
processfclayer / ReLUNorm / processconv33ReLU /        processfclayer / relunorm / conv33relu / maxpool22
processmaxpool22 (BitNetMCU_inference.h:15-60)         (same argument meaning, batched over a leading axis)
model = whichever header is named BitNetMCU_model.h    Engine(Model) from parse_header() / a .bnm blob

Nothing here computes on the CPU: every call goes through libbitnetmcu_b200.so (hand-written sm_90a CUDA).
torch is used only as plumbing for device memory / streams in ``infer_device``.
"""
from __future__ import annotations

import ctypes as C
import sys
from typing import Optional, Tuple

import numpy as np

from . import _lib
from .model import Model


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else C.c_void_p(a.ctypes.data)


N = "n"   # in the shape of a tensor argument of Engine._device_call: the number of images


def _half_format(dtype) -> Optional[int]:
    """The 16-bit format (include/bitnetmcu_b200.h section 11) of a torch dtype: FLOAT16, BFLOAT16, or None for float32"""
    import torch
    return {torch.float32: None, torch.float16: _lib.FLOAT16, torch.bfloat16: _lib.BFLOAT16}[dtype]


def _pad_sides(padding) -> Tuple[int, int, int, int]:
    """(left, right, top, bottom) of a window scan's padding: an int for all four sides, or a 4-sequence in F.pad's order"""
    if isinstance(padding, int):
        return (padding,) * 4
    sides = tuple(int(v) for v in padding)
    if len(sides) != 4:
        raise ValueError(f"padding: an int or (left, right, top, bottom), got {padding!r}")
    return sides


_PAD_MODES = {"constant": _lib.PAD_CONSTANT, "replicate": _lib.PAD_REPLICATE, "reflect": _lib.PAD_REFLECT}


def _host_pages(pages):
    """(format, pointer, the array that owns the pixels, (P, H, W), pitch, plane pitch) of host pages (section 14): a NumPy float32 /
    float16 array or a CPU torch tensor of float32, float16 or bfloat16, [P, H, W] or [H, W].  A view whose column stride is not
    one element, whose rows overlap (a row stride under the width, as a broadcast row has), or with a negative or partial-element
    stride is copied to a contiguous array first."""
    torch = sys.modules.get("torch")
    if torch is not None and isinstance(pages, torch.Tensor):
        if pages.device.type != "cpu":
            raise ValueError(f"host pages must be a CPU tensor, got one on {pages.device}: use the *_device methods")
        fmt = {torch.float32: _lib.FLOAT32, torch.float16: _lib.FLOAT16, torch.bfloat16: _lib.BFLOAT16}.get(pages.dtype)
        if fmt is None:
            raise TypeError(f"host pages: float32, float16 or bfloat16, got {pages.dtype}")
        p = pages if pages.dim() == 3 else pages.unsqueeze(0)
        if p.dim() != 3:
            raise ValueError(f"host pages: [P, H, W] or [H, W], got shape {tuple(pages.shape)}")
        if not _unit_columns(p.shape, p.stride(), 1):
            p = p.contiguous()
        return (fmt, p.data_ptr(), p, tuple(p.shape)) + _pitches(p.shape, p.stride())
    a = np.asarray(pages)
    fmt = {np.dtype(np.float32): _lib.FLOAT32, np.dtype(np.float16): _lib.FLOAT16}.get(a.dtype)
    if fmt is None:
        raise TypeError(f"host pages: float32 or float16, got {a.dtype}")
    a = a[None] if a.ndim == 2 else a
    if a.ndim != 3:
        raise ValueError(f"host pages: [P, H, W] or [H, W], got shape {np.shape(pages)}")
    if not _unit_columns(a.shape, a.strides, a.itemsize):
        a = np.ascontiguousarray(a)
    return (fmt, a.ctypes.data, a, a.shape) + _pitches(a.shape, [s // a.itemsize for s in a.strides])


def _unit_columns(shape, strides, unit) -> bool:
    """whether a [P, H, W] view's columns are one element (unit) apart, its rows at least a row apart (not a broadcast or
    overlapping rows) and its planes a whole number of elements >= 0 apart; a stride of an axis of one element or less is never
    used"""
    return all(n <= 1 or (s >= 0 and s % unit == 0 and (i != 1 or s >= unit * shape[2]) and (i < 2 or s == unit))
               for i, (n, s) in enumerate(zip(shape, strides)))


def _pitches(shape, strides) -> Tuple[int, int]:
    """(pitch, plane pitch) in elements of a [P, H, W] view (strides in elements), those of a compact stack on an axis of one
    element or less and for a view of no elements"""
    p, h, w = shape
    if p * h * w == 0:
        return w, h * w
    pitch = strides[1] if h > 1 else w
    return pitch, (strides[0] if p > 1 else h * pitch)


def _host_out(out: Optional[np.ndarray], want: bool, shape, dtype) -> Optional[np.ndarray]:
    """out (checked: C-contiguous, writeable, of dtype and shape), else a new array when wanted, else None"""
    if out is None:
        return np.empty(shape, dtype=dtype) if want else None
    if out.dtype != dtype or tuple(out.shape) != tuple(shape) or not out.flags.c_contiguous or not out.flags.writeable:
        raise ValueError(f"output array: a writeable C-contiguous {np.dtype(dtype)} array of shape {tuple(shape)}, got "
                         f"{out.dtype} {out.shape}")
    return out


def window_grid(height: int, width: int, stride, padding=None) -> Tuple[int, int]:
    """(out_h, out_w) of the 16x16 windows of a height x width image on a stride grid (include/bitnetmcu_b200.h section 9);
    stride is an int or (stride_y, stride_x), each >= 1.  (0, 0)-sized when the image is under 16 pixels either way.  padding:
    None, or an int / (left, right, top, bottom) as F.pad takes it (section 13): the grid over the padded image, and (0, 0) for
    an image of no pixels."""
    sy, sx = (stride, stride) if isinstance(stride, int) else (int(stride[0]), int(stride[1]))
    if sy < 1 or sx < 1:
        raise ValueError(f"window_grid: strides must be >= 1, got {(sy, sx)}")
    if padding is not None:
        if height == 0 or width == 0:
            return 0, 0
        left, right, top, bottom = _pad_sides(padding)
        height, width = height + top + bottom, width + left + right
    if height < 16 or width < 16:
        return 0, 0
    return (height - 16) // sy + 1, (width - 16) // sx + 1


class Engine:
    """One packed model resident on one GPU."""

    def __init__(self, model: Model, device: int = 0, path: int = _lib.PATH_AUTO, nf4_extension: bool = False):
        self.lib = _lib.load()
        if self.lib.bnm_device_count() == 0:
            raise _lib.BnmError("no CUDA device: bitnetmcu_b200 has no CPU fallback")
        self.model = model
        blob = model.to_blob()
        self._blob = (C.c_char * len(blob)).from_buffer_copy(blob)
        h = C.c_void_p()
        _lib.check(self.lib.bnm_model_load_blob(self._blob, len(blob), device, C.byref(h)), "bnm_model_load_blob")
        self.handle = h
        self.device = device
        self.n_classes = int(self.lib.bnm_model_n_classes(h))
        self.img_bytes = int(self.lib.bnm_model_img_bytes(h))
        if nf4_extension:
            self.set_option(_lib.OPT_NF4_EXTENSION, 1)
        if path != _lib.PATH_AUTO:
            self.set_option(_lib.OPT_PATH, path)

    def close(self) -> None:
        if getattr(self, "handle", None):
            self.lib.bnm_model_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, option: int, value: int) -> None:
        _lib.check(self.lib.bnm_model_set_option(self.handle, option, int(value)), "bnm_model_set_option")

    @property
    def active_path(self) -> int:
        return int(self.lib.bnm_model_active_path(self.handle))

    def launch_count(self, n: int) -> int:
        return int(self.lib.bnm_infer_launch_count(self.handle, n))

    # ---- batched inference over host arrays (H2D / kernels / D2H pipelined inside the library) -----------
    def infer(self, images: np.ndarray, want_labels: bool = True, want_logits: bool = True, out_logits: Optional[np.ndarray] = None,
              out_labels: Optional[np.ndarray] = None) -> Tuple[Optional[np.ndarray], Optional[np.ndarray]]:
        """images int8 [n, img_bytes] -> (logits int32 [n, n_classes], labels uint32 [n]).  ``want_logits=False`` returns
        ``(None, labels)``: the logits are neither copied back nor, on the fused path, written to GPU memory."""
        if not (want_labels or want_logits):
            raise ValueError("Engine.infer: ask for logits, labels or both")
        imgs = np.ascontiguousarray(images, dtype=np.int8).reshape(-1, self.img_bytes)
        n = imgs.shape[0]
        logits = None
        if want_logits:
            logits = out_logits if out_logits is not None else np.empty((n, self.n_classes), dtype=np.int32)
        labels = out_labels if out_labels is not None else (np.empty(n, dtype=np.uint32) if want_labels else None)
        _lib.check(self.lib.bnm_infer_batch(self.handle, _ptr(imgs), n, _ptr(logits), _ptr(labels)), "bnm_infer_batch")
        return logits, labels

    def inference(self, image: np.ndarray) -> int:
        """``uint32_t Inference(int8_t *input)`` (BitNetMCU_MNIST_dll.c:24): predicted class of one image."""
        _, labels = self.infer(np.asarray(image, dtype=np.int8).reshape(1, self.img_bytes), want_logits=False)
        return int(labels[0])

    # ---- device pointers (torch tensors as plumbing) ---------------------------------------------------
    def infer_device(self, images, logits, labels=None, stream: Optional[int] = None) -> None:
        """images: torch.int8 [n, img_bytes] on this GPU; logits: torch.int32 [n, n_classes] or None; labels: torch.int32/uint32
        [n] or None (not both None).  Asynchronous on ``stream`` (a cudaStream_t as int; default: torch's current stream).

        With ``OPT_LAUNCH_OVERLAP`` = 2 a launch whose buffers differ from the previous call's is NOT ordered against earlier
        work on the stream (include/bitnetmcu_b200.h): its images must already be complete when the previous call was
        enqueued.  Chains such as ``quantize_images_device`` -> ``infer_device`` on one stream need mode 0 or 1.

        Inside ``torch.cuda.graph`` the current stream is the capture stream, so the call is captured, and every replay gives what
        the same call would give on the buffers' contents at replay time (INTEGRATION.md section 4)."""
        import torch
        self._device_call(self.lib.bnm_infer_batch_device, images, torch.int8,
                          [(logits, torch.int32, (N, self.n_classes)), (labels, 4, N)], stream)

    def _float_call(self, fn, fn16, images, args, stream) -> None:
        """fn on torch.float32 images, or its 16-bit sibling fn16 (section 11) with the tensor's format on torch.float16 or
        torch.bfloat16 images: bit for bit what fn gives on ``images.float()``."""
        fmt = _half_format(images.dtype)
        self._device_call(fn if fmt is None else fn16, images, images.dtype, args, stream, fmt=fmt)

    def _device_call(self, fn, images, in_dtype, args, stream, lead=None, fmt=None) -> None:
        """fn(handle, images, n, *args, stream) on this GPU, images a contiguous in_dtype [n, img_bytes] tensor.  A tensor argument
        is given as (tensor or None, its dtype or element size, its shape with N for n, or N alone for n elements of any shape):
        asserted contiguous and of that type and shape, it passes as its pointer, None as NULL.  Other arguments pass as they are.
        stream: a cudaStream_t as int, None for torch's current stream.  lead: instead of images and n, these arguments
        (images is then an in_dtype tensor of any shape, N counts its elements).  fmt: a 16-bit entry's format, passed after images."""
        import torch
        if stream is None:
            stream = torch.cuda.current_stream(images.device).cuda_stream
        assert images.dtype == in_dtype and (lead is not None or images.dim() == 2)
        assert lead is not None or (images.is_contiguous() and images.shape[1] == self.img_bytes)
        n = images.shape[0] if lead is None else images.numel()
        vals = []
        for a in args:
            if isinstance(a, tuple):
                t, kind, shape = a
                if t is not None:
                    assert t.is_contiguous() and (t.dtype == kind if isinstance(kind, torch.dtype) else t.element_size() == kind)
                    assert t.numel() == n if shape is N else tuple(t.shape) == tuple(n if d is N else d for d in shape)
                a = None if t is None else C.c_void_p(t.data_ptr())
            vals.append(a)
        head = ([C.c_void_p(images.data_ptr()), n] if fmt is None else [C.c_void_p(images.data_ptr()), fmt, n]) if lead is None else list(lead)
        _lib.check(fn(self.handle, *head, *vals, C.c_void_p(stream)), fn.__name__)

    def inference_quantized(self, input_data: np.ndarray) -> np.ndarray:
        """``QuantizedModel.inference_quantized`` (/root/reference/BitNetMCU.py:420-535) on the GPU: float32 images [n, img_bytes]
        -> float64 logits [n, n_classes] with the Python emulator's normalisation rules (not the C engine's): what
        ``np.argmax`` is taken of in test_inference.py:153-154 and exportquant.py:537-559."""
        x = np.ascontiguousarray(input_data, dtype=np.float32).reshape(-1, self.img_bytes)
        out = np.empty((x.shape[0], self.n_classes), dtype=np.float64)
        _lib.check(self.lib.bnm_emulate_inference_quantized(self.handle, _ptr(x), x.shape[0], _ptr(out)), "bnm_emulate_inference_quantized")
        return out

    def inference_quantized_device(self, images, logits=None, labels=None, stream: Optional[int] = None) -> None:
        """``inference_quantized`` on device buffers: images torch.float32 [n, img_bytes] on this GPU -> logits torch.float64
        [n, n_classes] or None, labels [n] (4-byte elements: ``np.argmax`` of the logits) or None (not both None).  Asynchronous on
        ``stream`` (a cudaStream_t as int; default: torch's current stream).  FC models up to 64 wide: one kernel.
        torch.float16 / torch.bfloat16 images: what float32 gives on ``images.float()``, reading 2 bytes per pixel."""
        import torch
        self._float_call(self.lib.bnm_emulate_batch_device, self.lib.bnm_emulate_batch_device_f16, images,
                         [(logits, torch.float64, (N, self.n_classes)), (labels, 4, N)], stream)

    def infer_device_f32(self, images, logits, labels=None, stream: Optional[int] = None) -> None:
        """images: torch.float32 [n, img_bytes] on this GPU (un-normalised pixels, as test_inference.py:140 sees them) -> logits
        torch.int32 [n, n_classes] or None, labels [n] or None (not both None).  FC models: one kernel with the input scaling fused
        into its load stage.  torch.float16 / torch.bfloat16 images: what float32 gives on ``images.float()``, reading 2 bytes per
        pixel."""
        import torch
        self._float_call(self.lib.bnm_infer_batch_device_f32, self.lib.bnm_infer_batch_device_f16, images,
                         [(logits, torch.int32, (N, self.n_classes)), (labels, 4, N)], stream)

    def infer_windows_device(self, image, stride, logits=None, labels=None, stream: Optional[int] = None) -> None:
        """Window scan (include/bitnetmcu_b200.h section 9): every 16x16 window of image, a torch.float32 [height, width] plane on
        this GPU with unit column stride (its row stride is the pitch, a multiple of 4), on a stride grid (an int or (sy, sx)) ->
        logits torch.int32 [out_h, out_w, n_classes] or None, labels [out_h, out_w] (4-byte elements) or None (not both None), where
        (out_h, out_w) = window_grid(height, width, stride).  Window (r, c) covers image[r*sy : r*sy+16, c*sx : c*sx+16]; its
        results are what ``infer_device_f32`` returns for that window flattened.  Asynchronous on ``stream`` (default: torch's
        current stream).  A torch.float16 / torch.bfloat16 plane (pitch a multiple of 8): what float32 gives on ``image.float()``,
        through ``bnm_scan_windows_device_f16`` with one plane."""
        import torch
        assert image.dim() == 2 and image.stride(1) == 1
        if _half_format(image.dtype) is not None:
            one = [None if t is None else t.unsqueeze(0) for t in (logits, labels)]
            self._windows_call("bnm_scan_windows", image, stride, [(one[0], torch.int32, (self.n_classes,)), (one[1], 4, ())], stream)
            return
        sy, sx = (stride, stride) if isinstance(stride, int) else (int(stride[0]), int(stride[1]))
        h, w = image.shape
        out_h, out_w = window_grid(h, w, (sy, sx))
        lead = (C.c_void_p(image.data_ptr()), h, w, image.stride(0), sy, sx)
        self._device_call(self.lib.bnm_infer_windows_device_f32, image, torch.float32,
                          [(logits, torch.int32, (out_h, out_w, self.n_classes)), (labels, 4, (out_h, out_w))], stream, lead=lead)

    # ---- window scan of a stack of pages (include/bitnetmcu_b200.h sections 10, 12 and 13) ---------------------------------------
    # pages: a torch.float32 [P, H, W] stack on this GPU ([H, W]: one page) with unit column stride; its row stride is the pitch
    # and its plane stride the plane pitch (multiples of 4).  stride: an int or (sy, sx).  Every output is [P, out_h, out_w, ...]
    # with (out_h, out_w) = window_grid(H, W, stride, padding); window (p, r, c) covers pages[p, r*sy : r*sy+16, c*sx : c*sx+16],
    # and its results are those of the matching entry on that window flattened.  torch.float16 / torch.bfloat16 pages (section 12;
    # pitches multiples of 8): what float32 gives on ``pages.float()``, reading 2 bytes per pixel.  padding (section 13): None
    # (the unpadded entry), or an int / (left, right, top, bottom) of at most 15 each, with pad_mode "constant", "replicate" or
    # "reflect" and pad_value the constant mode's float32 fill: what the unpadded call gives on
    # ``F.pad(pages.float(), padding, pad_mode, pad_value)``, without that copy.  Asynchronous on ``stream`` (default: torch's
    # current stream).
    def _windows_call(self, stem, pages, stride, args, stream, padding=None, pad_mode="constant", pad_value=0.0) -> None:
        """The window entry named stem + ("_padded" with a padding) + "_device" (+ "_f16" on 16-bit pages): fn(handle, the stack's
        bnm_windows[, format][, its bnm_window_padding], *args, stream), as _device_call passes args, a tensor argument's shape
        given past the window grid [P, out_h, out_w]"""
        p = pages if pages.dim() == 3 else pages.unsqueeze(0)
        assert p.dim() == 3 and p.stride(2) == 1
        fmt = _half_format(p.dtype)
        sy, sx = (stride, stride) if isinstance(stride, int) else (int(stride[0]), int(stride[1]))
        n_p, h, w = p.shape
        desc = _lib.BnmWindows(p.data_ptr(), n_p, h, w, p.stride(1), p.stride(0), sy, sx)
        grid = (n_p,) + window_grid(h, w, (sy, sx), padding)
        args = [(a[0], a[1], grid + a[2]) if isinstance(a, tuple) else a for a in args]
        lead = [C.byref(desc)] if fmt is None else [C.byref(desc), fmt]
        if padding is not None:
            if pad_mode not in _PAD_MODES:
                raise ValueError(f"pad_mode must be one of {sorted(_PAD_MODES)}, got {pad_mode!r}")
            pad = _lib.BnmWindowPadding(*_pad_sides(padding), _PAD_MODES[pad_mode], float(pad_value))
            lead.append(C.byref(pad))
        name = stem + ("_padded" if padding is not None else "") + "_device" + ("_f16" if fmt is not None else "")
        self._device_call(getattr(self.lib, name), p, p.dtype, args, stream, lead=tuple(lead))

    def scan_windows_device(self, pages, stride, logits=None, labels=None, stream: Optional[int] = None, *, padding=None,
                            pad_mode: str = "constant", pad_value: float = 0.0) -> None:
        """The C engine on every window of a stack of pages: logits torch.int32 [P, out_h, out_w, n_classes] or None, labels
        [P, out_h, out_w] (4-byte elements) or None (not both None); ``infer_device_f32`` on each window."""
        import torch
        self._windows_call("bnm_scan_windows", pages, stride, [(logits, torch.int32, (self.n_classes,)), (labels, 4, ())], stream,
                           padding, pad_mode, pad_value)

    def scan_windows_topk_device(self, pages, stride, k: int, classes, scores=None, stream: Optional[int] = None, *, padding=None,
                                 pad_mode: str = "constant", pad_value: float = 0.0) -> None:
        """The C engine's top-k of every window: classes [P, out_h, out_w, k] (4-byte elements), scores torch.int32
        [P, out_h, out_w, k] or None; ``topk_device_f32`` on each window."""
        import torch
        self._windows_call("bnm_scan_windows_topk", pages, stride, [int(k), (classes, 4, (k,)), (scores, torch.int32, (k,))], stream,
                           padding, pad_mode, pad_value)

    def emulate_windows_device(self, pages, stride, logits=None, labels=None, stream: Optional[int] = None, *, padding=None,
                               pad_mode: str = "constant", pad_value: float = 0.0) -> None:
        """The emulator on every window: logits torch.float64 [P, out_h, out_w, n_classes] or None, labels [P, out_h, out_w]
        or None (not both None); ``inference_quantized_device`` on each window."""
        import torch
        self._windows_call("bnm_emulate_windows", pages, stride, [(logits, torch.float64, (self.n_classes,)), (labels, 4, ())], stream,
                           padding, pad_mode, pad_value)

    def emulate_windows_topk_device(self, pages, stride, k: int, classes, scores=None, stream: Optional[int] = None, *, padding=None,
                                    pad_mode: str = "constant", pad_value: float = 0.0) -> None:
        """The emulator's top-k of every window: classes [P, out_h, out_w, k], scores torch.float64 [P, out_h, out_w, k] or
        None; ``emulate_topk_device`` on each window."""
        import torch
        self._windows_call("bnm_emulate_windows_topk", pages, stride, [int(k), (classes, 4, (k,)), (scores, torch.float64, (k,))],
                           stream, padding, pad_mode, pad_value)

    # ---- window scan of host pages (include/bitnetmcu_b200.h section 14) ----------------------------------------------------------
    # pages: a [P, H, W] stack ([H, W]: one page) in host memory, a NumPy float32 / float16 array or a CPU torch tensor of
    # torch.float32, torch.float16 or torch.bfloat16 (pinned or not), any strided view with unit column stride (others are copied
    # to a contiguous array first).  The library copies it to the GPU band by band, scanning one band while the next is copied,
    # and returns NumPy arrays [P, out_h, out_w, ...] with (out_h, out_w) = window_grid(H, W, stride, padding): bit for bit what
    # the matching ``*_device`` method returns on the same stack copied to the GPU.  stride, padding, pad_mode and pad_value are
    # those of the device methods.  out_*: NumPy arrays of the output's dtype and shape, C-contiguous, to write into instead.
    def _host_windows_call(self, stem, pages, stride, args, padding, pad_mode, pad_value) -> None:
        """the host window entry stem(handle, the stack's bnm_windows_host, its bnm_window_padding or NULL, *args)"""
        fmt, ptr, _keep, shape, pitch, plane_pitch = _host_pages(pages)
        sy, sx = (stride, stride) if isinstance(stride, int) else (int(stride[0]), int(stride[1]))
        desc = _lib.BnmWindowsHost(ptr, fmt, shape[0], shape[1], shape[2], pitch, plane_pitch, sy, sx)
        pad = None
        if padding is not None:
            if pad_mode not in _PAD_MODES:
                raise ValueError(f"pad_mode must be one of {sorted(_PAD_MODES)}, got {pad_mode!r}")
            pad = C.byref(_lib.BnmWindowPadding(*_pad_sides(padding), _PAD_MODES[pad_mode], float(pad_value)))
        _lib.check(getattr(self.lib, stem)(self.handle, C.byref(desc), pad, *args), stem)

    def _host_grid(self, pages, stride, padding) -> Tuple[int, int, int]:
        shape = tuple(np.shape(pages))
        return (shape[0] if len(shape) == 3 else 1,) + window_grid(shape[-2], shape[-1], stride, padding)

    def scan_windows(self, pages, stride, want_labels: bool = True, want_logits: bool = True, out_logits: Optional[np.ndarray] = None,
                     out_labels: Optional[np.ndarray] = None, *, padding=None, pad_mode: str = "constant",
                     pad_value: float = 0.0) -> Tuple[Optional[np.ndarray], Optional[np.ndarray]]:
        """The C engine on every window of host pages -> (logits int32 [P, out_h, out_w, n_classes], labels uint32
        [P, out_h, out_w]), either None when not asked for; ``scan_windows_device`` on the pages copied to the GPU."""
        grid = self._host_grid(pages, stride, padding)
        logits = _host_out(out_logits, want_logits, grid + (self.n_classes,), np.int32)
        labels = _host_out(out_labels, want_labels, grid, np.uint32)
        if logits is None and labels is None:
            raise ValueError("Engine.scan_windows: ask for logits, labels or both")
        self._host_windows_call("bnm_scan_windows", pages, stride, [_ptr(logits), _ptr(labels)], padding, pad_mode, pad_value)
        return logits, labels

    def scan_windows_topk(self, pages, stride, k: int, want_scores: bool = True, out_classes: Optional[np.ndarray] = None,
                          out_scores: Optional[np.ndarray] = None, *, padding=None, pad_mode: str = "constant",
                          pad_value: float = 0.0) -> Tuple[np.ndarray, Optional[np.ndarray]]:
        """The C engine's top-k of every window of host pages -> (classes uint32 [P, out_h, out_w, k], scores int32
        [P, out_h, out_w, k] or None with ``want_scores=False``); ``scan_windows_topk_device`` on the pages copied to the GPU."""
        grid = self._host_grid(pages, stride, padding)
        classes = _host_out(out_classes, True, grid + (k,), np.uint32)
        scores = _host_out(out_scores, want_scores, grid + (k,), np.int32)
        self._host_windows_call("bnm_scan_windows_topk", pages, stride, [int(k), _ptr(classes), _ptr(scores)], padding, pad_mode,
                                pad_value)
        return classes, scores

    def emulate_windows(self, pages, stride, want_labels: bool = True, want_logits: bool = True,
                        out_logits: Optional[np.ndarray] = None, out_labels: Optional[np.ndarray] = None, *, padding=None,
                        pad_mode: str = "constant", pad_value: float = 0.0) -> Tuple[Optional[np.ndarray], Optional[np.ndarray]]:
        """The emulator on every window of host pages -> (logits float64 [P, out_h, out_w, n_classes], labels uint32
        [P, out_h, out_w]), either None when not asked for; ``emulate_windows_device`` on the pages copied to the GPU."""
        grid = self._host_grid(pages, stride, padding)
        logits = _host_out(out_logits, want_logits, grid + (self.n_classes,), np.float64)
        labels = _host_out(out_labels, want_labels, grid, np.uint32)
        if logits is None and labels is None:
            raise ValueError("Engine.emulate_windows: ask for logits, labels or both")
        self._host_windows_call("bnm_emulate_windows", pages, stride, [_ptr(logits), _ptr(labels)], padding, pad_mode, pad_value)
        return logits, labels

    def emulate_windows_topk(self, pages, stride, k: int, want_scores: bool = True, out_classes: Optional[np.ndarray] = None,
                             out_scores: Optional[np.ndarray] = None, *, padding=None, pad_mode: str = "constant",
                             pad_value: float = 0.0) -> Tuple[np.ndarray, Optional[np.ndarray]]:
        """The emulator's top-k of every window of host pages -> (classes uint32 [P, out_h, out_w, k], scores float64
        [P, out_h, out_w, k] or None with ``want_scores=False``); ``emulate_windows_topk_device`` on the pages copied to the GPU."""
        grid = self._host_grid(pages, stride, padding)
        classes = _host_out(out_classes, True, grid + (k,), np.uint32)
        scores = _host_out(out_scores, want_scores, grid + (k,), np.float64)
        self._host_windows_call("bnm_emulate_windows_topk", pages, stride, [int(k), _ptr(classes), _ptr(scores)], padding, pad_mode,
                                pad_value)
        return classes, scores

    def compare_engines_device(self, images, truth=None, labels_c=None, labels_py=None, counts=None, stream: Optional[int] = None) -> None:
        """Both engines on the same float images in one call (test_inference.py:130-175): images torch.float32 [n, img_bytes] on
        this GPU -> labels_c [n] (what ``infer_device_f32`` returns), labels_py [n] (what ``inference_quantized_device`` returns)
        and counts, a torch.int64 [4] tensor (images, correct_c, correct_py, mismatches) that the call ADDS to.  truth: [n] true
        classes (4-byte elements), counted into correct_c / correct_py, and only with counts.  Any of labels_c, labels_py and
        counts may be None, not all three.  Asynchronous on ``stream`` (default: torch's current stream).  FC models up to 64
        wide: one kernel.  torch.float16 / torch.bfloat16 images: what float32 gives on ``images.float()``."""
        import torch
        self._float_call(self.lib.bnm_compare_engines_device, self.lib.bnm_compare_engines_device_f16, images,
                         [(truth, 4, N), (labels_c, 4, N), (labels_py, 4, N), (counts, torch.int64, (4,))], stream)

    # ---- top-k: each image's k best classes and their scores (include/bitnetmcu_b200.h section 8) ------------------------------
    # Classes are ranked by logit, highest first, ties to the lower class: np.argsort(-logits, kind="stable")[:, :k].  Rank 0 is
    # the label of the matching entry.  1 <= k <= min(n_classes, 16).
    def topk(self, images: np.ndarray, k: int, want_scores: bool = True) -> Tuple[np.ndarray, Optional[np.ndarray]]:
        """images int8 [n, img_bytes] (host) -> (classes uint32 [n, k], scores int32 [n, k] = the C engine's logits of those
        classes, or None with ``want_scores=False``).  No logits are written or copied back."""
        imgs = np.ascontiguousarray(images, dtype=np.int8).reshape(-1, self.img_bytes)
        n = imgs.shape[0]
        classes = np.empty((n, k), dtype=np.uint32)
        scores = np.empty((n, k), dtype=np.int32) if want_scores else None
        _lib.check(self.lib.bnm_infer_topk(self.handle, _ptr(imgs), n, int(k), _ptr(classes), _ptr(scores)), "bnm_infer_topk")
        return classes, scores

    def topk_device(self, images, k: int, classes, scores=None, stream: Optional[int] = None) -> None:
        """images torch.int8 [n, img_bytes] on this GPU -> classes [n, k] (torch.int32 / uint32) and scores torch.int32 [n, k] or
        None.  Asynchronous on ``stream`` (a cudaStream_t as int; default: torch's current stream)."""
        import torch
        self._device_call(self.lib.bnm_infer_topk_device, images, torch.int8,
                          [int(k), (classes, 4, (N, k)), (scores, torch.int32, (N, k))], stream)

    def topk_device_f32(self, images, k: int, classes, scores=None, stream: Optional[int] = None) -> None:
        """``topk_device`` on torch.float32 [n, img_bytes] images, scaled to int8 as ``infer_device_f32`` does (torch.float16 /
        torch.bfloat16 images: what float32 gives on ``images.float()``)."""
        import torch
        self._float_call(self.lib.bnm_infer_topk_device_f32, self.lib.bnm_infer_topk_device_f16, images,
                         [int(k), (classes, 4, (N, k)), (scores, torch.int32, (N, k))], stream)

    def emulate_topk_device(self, images, k: int, classes, scores=None, stream: Optional[int] = None) -> None:
        """The emulator's top-k: images torch.float32 [n, img_bytes] -> classes [n, k] and scores torch.float64 [n, k] (the
        logits ``inference_quantized_device`` writes, at those classes) or None.  torch.float16 / torch.bfloat16 images: what
        float32 gives on ``images.float()``."""
        import torch
        self._float_call(self.lib.bnm_emulate_topk_device, self.lib.bnm_emulate_topk_device_f16, images,
                         [int(k), (classes, 4, (N, k)), (scores, torch.float64, (N, k))], stream)

    def infer_tensor(self, images, want_logits: bool = True):
        """images: torch.int8 [n, img_bytes] on this engine's GPU -> (logits torch.int32 [n, n_classes], labels torch.int32 [n]) on
        the same GPU, asynchronous on torch's current stream (device memory end to end; plumbing for ``dist.sharded_infer``).
        ``want_logits=False`` returns ``(None, labels)``."""
        import torch
        n = images.shape[0]
        logits = torch.empty((n, self.n_classes), dtype=torch.int32, device=images.device) if want_logits else None
        labels = torch.empty(n, dtype=torch.int32, device=images.device)
        if n:
            self.infer_device(images.contiguous(), logits, labels)
        return logits, labels


# ---- the four reference kernels, batched (host arrays) --------------------------------------------------------

def processfclayer(activations: np.ndarray, weights: np.ndarray, bits_per_weight: int, n_input: int, n_output: int,
                   nf4_extension: bool = False) -> np.ndarray:
    """inference.c:88-208 over a batch: activations int8 [n, n_input] -> int32 [n, n_output]."""
    lib = _lib.load()
    act = np.ascontiguousarray(activations, dtype=np.int8).reshape(-1, n_input)
    w = np.ascontiguousarray(weights)
    out = np.empty((act.shape[0], n_output), dtype=np.int32)
    _lib.check(lib.bnm_processfclayer_batch(_ptr(act), _ptr(w), bits_per_weight, n_input, n_output, _ptr(out), act.shape[0],
                                            int(nf4_extension)), "bnm_processfclayer_batch")
    return out


def relunorm(x: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """inference.c:23-72 over a batch: int32 [n, n_input] -> (int8 [n, n_input], argmax uint32 [n])."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.int32)
    x2 = x.reshape(-1, x.shape[-1]) if x.ndim > 1 else x.reshape(1, -1)
    out = np.empty(x2.shape, dtype=np.int8)
    pos = np.empty(x2.shape[0], dtype=np.uint32)
    _lib.check(lib.bnm_relunorm_batch(_ptr(x2), _ptr(out), _ptr(pos), x2.shape[1], x2.shape[0]), "bnm_relunorm_batch")
    return out, pos


def conv33relu(activations: np.ndarray, weights: np.ndarray, xy: int, n_shift: int = 4) -> np.ndarray:
    """inference.c:238-277 over a batch: int32 [n, xy*xy], int8 [n_w, 9] (item i uses weights[i % n_w])."""
    lib = _lib.load()
    a = np.ascontiguousarray(activations, dtype=np.int32).reshape(-1, xy * xy)
    w = np.ascontiguousarray(weights, dtype=np.int8).reshape(-1, 9)
    out = np.empty((a.shape[0], (xy - 2) * (xy - 2)), dtype=np.int32)
    _lib.check(lib.bnm_conv33relu_batch(_ptr(a), _ptr(w), w.shape[0], xy, n_shift, _ptr(out), a.shape[0]), "bnm_conv33relu_batch")
    return out


def maxpool22(activations: np.ndarray, xy: int) -> np.ndarray:
    """inference.c:300-322 over a batch: int32 [n, xy*xy] -> int32 [n, (xy/2)^2]."""
    lib = _lib.load()
    a = np.ascontiguousarray(activations, dtype=np.int32).reshape(-1, xy * xy)
    out = np.empty((a.shape[0], (xy // 2) * (xy // 2)), dtype=np.int32)
    _lib.check(lib.bnm_maxpool22_batch(_ptr(a), xy, _ptr(out), a.shape[0]), "bnm_maxpool22_batch")
    return out


def quantize_images(images: np.ndarray) -> np.ndarray:
    """The step right before the path (test_inference.py:140-141): float32 [n, elems] -> int8 [n, elems],
    ``np.round(x * (127 / max(|x|.max(-1), 1e-5))).clip(-128, 127)`` computed on the GPU, bit-identical to NumPy float32."""
    lib = _lib.load()
    x = np.ascontiguousarray(images, dtype=np.float32)
    x2 = x.reshape(-1, x.shape[-1]) if x.ndim > 1 else x.reshape(1, -1)
    out = np.empty(x2.shape, dtype=np.int8)
    _lib.check(lib.bnm_quantize_images(_ptr(x2), x2.shape[0], x2.shape[1], _ptr(out)), "bnm_quantize_images")
    return out


def quantize_images_device(images, out, stream: Optional[int] = None) -> None:
    """Device-buffer form: images torch.float32 [n, elems] -> out torch.int8 [n, elems] on the same GPU, asynchronous on
    ``stream`` (default: torch's current stream), so it chains with ``Engine.infer_device`` without a host pass.
    torch.float16 / torch.bfloat16 images: what float32 gives on ``images.float()``."""
    import torch
    lib = _lib.load()
    fmt = _half_format(images.dtype)
    assert images.is_contiguous() and out.is_contiguous() and out.dtype == torch.int8
    assert images.dim() == 2 and tuple(out.shape) == tuple(images.shape)
    if stream is None:
        stream = torch.cuda.current_stream(images.device).cuda_stream
    head = [C.c_void_p(images.data_ptr())] if fmt is None else [C.c_void_p(images.data_ptr()), fmt]
    fn = lib.bnm_quantize_images_device if fmt is None else lib.bnm_quantize_images_device_f16
    _lib.check(fn(*head, images.shape[0], images.shape[1], C.c_void_p(out.data_ptr()), C.c_void_p(stream)), fn.__name__)
