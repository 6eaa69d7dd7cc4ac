"""Host-side mirror of ``3_style_translator/training/models.py`` for the inference hot path.

``GeneratorJ_RIC`` (stage 1, models.py:200-356) and ``GeneratorJ`` (stage 2, models.py:24-129)
with the reference constructor signature, the same 89-key ``state_dict`` layout (SURVEY.md 8a
row a8) and the same ``forward(x)`` contract (fp32 NCHW in / out on the module's CUDA device), so
``training.trainers.build_model`` + ``load_state_dict`` + ``.eval()`` + ``generator(x)`` in the
reference's ``test_stage1.py`` / ``test_stage2.py`` work unchanged once
``drawingspinup_b200.install()`` has rebound the two class names.

The modules hold only parameters; ``forward`` hands raw device pointers to the hand-written
sm_90a kernels through the C ABI (``include/dsu_b200.h``, ctypes).  No ``torch.nn.Conv2d``, no
torch compute on the path, no CPU fallback: a missing library or a device other than sm_90 (H100) raises.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Optional, Sequence

import torch
import torch.nn as nn

from . import capi


def ric_offsets(height: int, width: int) -> torch.Tensor:
    """Offset field of ``generate_coordinates`` (models.py:551-598) as fp32 ``[18, h, w]`` on the
    CPU: every non-centre tap k of the 3x3 window samples on the unit circle around the pixel at
    angle theta + k*pi/4, theta = polar angle of the pixel about the image centre rounded to 1e-4.
    Computed with the same torch ops / dtypes as the reference so the bilinear stencil the kernels
    use is bit-identical to the one torchvision would derive.  (Batch expand :600 and the
    unconditional ``.cuda()`` :602 are not needed: the field is data independent.)"""
    hw = torch.zeros(2)
    hw[0] = height
    hw[1] = width
    c_row = torch.sub(torch.div(hw[0], 2.0), 0.5)
    c_col = torch.sub(torch.div(hw[1], 2.0), 0.5)
    row, col = torch.meshgrid(torch.arange(0, hw[0]), torch.arange(0, hw[1]), indexing="ij")
    full = torch.mul(torch.Tensor([math.pi]), 2.0)[0]
    theta = torch.atan2(torch.sub(col, c_col), torch.sub(row, c_row)) % full
    theta = torch.round(10000.0 * theta) / 10000.0
    eighth = torch.div(full, 8.0)
    field = torch.zeros(18, height, width)
    for rot in range(8):
        tap = rot + (rot >= 4)
        ang = torch.add(theta, torch.mul(eighth, float(rot)))
        field[2 * tap] = torch.add(torch.cos(ang), float(1 - tap // 3))
        field[2 * tap + 1] = torch.add(torch.sin(ang), float(1 - tap % 3))
    return field.contiguous()


class _ConvParams(nn.Module):
    """Holder of a convolution's ``weight`` (and optional ``bias``) under the reference key names;
    initialised like ``nn.Conv2d`` (kaiming-uniform a=sqrt(5), bias U(-1/sqrt(fan_in), ..))."""

    def __init__(self, cin: int, cout: int, k: int, bias: bool):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, k, k))
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if bias:
            bound = 1.0 / math.sqrt(cin * k * k)
            self.bias = nn.Parameter(torch.empty(cout).uniform_(-bound, bound))
        else:
            self.register_parameter("bias", None)


class _BatchNormStats(nn.Module):
    """Holder of BatchNorm2d parameters and running statistics (eval-mode affine)."""

    def __init__(self, c: int):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))
        self.register_buffer("running_mean", torch.zeros(c))
        self.register_buffer("running_var", torch.ones(c))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))


class _Named(nn.Module):
    """Container whose children carry the reference's sub-module names (``conv``, ``1``, ...)."""

    def __init__(self, **children):
        super().__init__()
        for name, mod in children.items():
            self.add_module(name.lstrip("_"), mod)


class _Generator(nn.Module):
    _KIND = 0
    _FIRST_K = 7

    def __init__(self, norm_layer='batch_norm', gpu_ids=None, use_bias=False, resnet_blocks=9, tanh=False,
                 filters=(64, 128, 128, 128, 128, 64), input_channels=3, append_smoothers=False,
                 precision: Optional[str] = None, deterministic: Optional[bool] = None):
        super().__init__()
        assert norm_layer in [None, 'batch_norm', 'instance_norm'], \
            "norm_layer should be None, 'batch_norm' or 'instance_norm', not {}".format(norm_layer)
        self.norm_layer = norm_layer
        self.gpu_ids = gpu_ids
        self.use_bias = bool(use_bias)
        self.resnet_blocks = int(resnet_blocks)
        self.append_smoothers = bool(append_smoothers)
        self.tanh = bool(tanh)
        self.filters = tuple(int(v) for v in filters)
        self.input_channels = int(input_channels)
        # deterministic=True: bit-reproducible results run to run.  Every CTA accumulates its K chunks in a fixed order and
        # the instance-norm statistics add their slices in slice order, so the engine is deterministic in both settings; the
        # flag is kept for callers that request it explicitly.
        self.deterministic = bool(int(os.environ.get("DSU_DETERMINISTIC", "0"))) if deterministic is None else bool(deterministic)
        self.precision = precision or os.environ.get("DSU_PRECISION", "fp16x3")
        if self.precision not in capi.PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(capi.PRECISIONS))
        f, k0, bn = self.filters, self._FIRST_K, norm_layer == 'batch_norm'

        def relu_layer(cin, cout, k):
            kids = {"conv": _ConvParams(cin, cout, k, self.use_bias)}
            if bn:
                kids["normalization"] = _BatchNormStats(cout)
            return _Named(**kids)

        self.conv0 = relu_layer(self.input_channels, f[0], k0)
        self.conv1 = relu_layer(f[0], f[1], 3)
        self.conv2 = relu_layer(f[1], f[2], 3)
        self.resnets = nn.ModuleList()
        for _ in range(self.resnet_blocks):
            kids = {"conv_0": _ConvParams(f[2], f[2], 3, self.use_bias)}
            if bn:
                kids["normalization"] = _BatchNormStats(f[2])
            kids["conv_1"] = _ConvParams(f[2], f[2], 3, self.use_bias)
            self.resnets.append(_Named(**kids))

        def upconv(cin, cout):
            kids = {"_1": _ConvParams(cin, cout, 3, False)}
            if bn:
                kids["_2"] = _BatchNormStats(cout)
            return _Named(**kids)

        self.upconv2 = upconv(f[3] + f[2], f[4])
        self.upconv1 = upconv(f[4] + f[1], f[4])
        self.conv_11 = _Named(_0=_ConvParams(f[0] + f[4] + self.input_channels, f[5], k0, self.use_bias))
        if self.append_smoothers:
            self.conv_11_a = _Named(_0=_ConvParams(f[5], f[5], 3, self.use_bias), _2=_BatchNormStats(f[5]),
                                    _3=_ConvParams(f[5], f[5], 3, self.use_bias))
        self.conv_12 = _Named(_0=_ConvParams(f[5], 3, 1, True)) if self.tanh else _ConvParams(f[5], 3, 1, True)

        self._handle = None
        self._handle_dev = None
        self._loaded_sig = None
        self._offset_dims = set()

    # ------------------------------------------------------------------ engine plumbing
    def _release(self):
        if getattr(self, "_handle", None):
            capi.lib().dsu_destroy(self._handle)
        self._handle = None
        self._loaded_sig = None
        self._offset_dims = set()

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _signature(self):
        # identity + version of every state-dict tensor: a changed weight (load_state_dict, in-place edit, .to()) re-packs.
        # The tensor list is cached - walking state_dict() costs ~0.2 ms per forward on the batch-1 script path - and dropped
        # whenever .to() / .cuda() / .half() may have replaced buffer objects (_apply).
        ts = self.__dict__.get("_sig_tensors")
        if ts is None:
            ts = self.__dict__["_sig_tensors"] = list(self.state_dict(keep_vars=True).values())
        return tuple((v.data_ptr(), v._version) for v in ts)

    def _apply(self, fn, *args, **kwargs):
        self.__dict__.pop("_sig_tensors", None)
        return super()._apply(fn, *args, **kwargs)

    def _engine(self, device: torch.device):
        """Create the engine for ``device`` if needed and (re)upload weights when any changed."""
        lib = capi.lib()
        if device.type != "cuda":
            raise RuntimeError("drawingspinup_b200 generators run on a CUDA (H100, sm_90) device only; got tensor on %s "
                               "(no CPU fallback)" % device)
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if self._handle is None or self._handle_dev != idx:
            self._release()
            cfg = capi.DsuConfig()
            cfg.kind = self._KIND
            cfg.input_channels = self.input_channels
            for i in range(6):
                cfg.filters[i] = self.filters[i]
            cfg.resnet_blocks = self.resnet_blocks
            cfg.use_bias = int(self.use_bias)
            cfg.tanh = int(self.tanh)
            cfg.append_smoothers = int(self.append_smoothers)
            cfg.norm = {'batch_norm': capi.NORM_BATCH, 'instance_norm': capi.NORM_INSTANCE}.get(self.norm_layer, capi.NORM_NONE)
            cfg.precision = capi.PRECISIONS[self.precision]
            cfg.device = idx
            h = C.c_void_p()
            capi.check(lib.dsu_create(C.byref(cfg), C.byref(h)), "dsu_create")
            self._handle, self._handle_dev = h, idx
        sig = self._signature()
        if sig != self._loaded_sig:
            for key, t in self.state_dict().items():
                t = t.detach()
                if t.dtype == torch.int64:
                    host, dtype = t.cpu().contiguous(), 1
                else:
                    host, dtype = t.to(device="cpu", dtype=torch.float32).contiguous(), 0
                shape = (C.c_int64 * max(1, host.dim()))(*host.shape)
                capi.check(lib.dsu_load_weights(self._handle, key.encode(), C.c_void_p(host.data_ptr()), shape,
                                                host.dim(), dtype, 0), "dsu_load_weights(%s)" % key)
            capi.check(lib.dsu_finalize(self._handle, None), "dsu_finalize")
            self._loaded_sig = sig
        return self._handle

    def _prepare_shape(self, h: int, w: int):
        pass

    def set_knob(self, name: str, value: int, device=None):
        """Development / test hook (C ABI ``dsu_set_knob``): kernel-selection knob of this module's engine handle."""
        dev = torch.device(device) if device is not None else (
            torch.device("cuda", self._handle_dev) if self._handle_dev is not None else next(self.parameters()).device)
        capi.check(capi.lib().dsu_set_knob(self._engine(dev), name.encode(), int(value)), "dsu_set_knob(%s)" % name)

    def _check_mode(self):
        # train() mode would mean batch-statistics BatchNorm in the reference (even under no_grad); the engine only
        # implements the eval-mode affine, so a module left in train() fails loudly instead of diverging silently
        if self.training:
            raise RuntimeError("drawingspinup_b200 generators are inference-only: call .eval() first (the reference scripts do, "
                               "test_stage1.py:48); training, trainers.py:90-108, is out of scope")
        if self._KIND == capi.KIND_GENERATORJ_RIC and self.norm_layer is None:
            # same failure as the reference: GeneratorJ_RIC.forward indexes self.conv0[2] (models.py:303), which does not
            # exist without a norm module - norm_layer=None is only a runnable configuration for GeneratorJ
            raise IndexError("index 2 is out of range (GeneratorJ_RIC.forward with norm_layer=None, models.py:303)")

    # ------------------------------------------------------------------ reference API
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """``generator(x)``: fp32 NCHW ``[B, input_channels, H, W]`` -> fp32 NCHW ``[B, 3, H, W]``
        (models.py:113-129 / 293-356), H and W multiples of 4."""
        self._check_mode()
        if x.dim() != 4 or x.shape[1] != self.input_channels:
            raise RuntimeError("expected input [B, %d, H, W], got %s" % (self.input_channels, tuple(x.shape)))
        handle = self._engine(x.device)
        x = x.detach().to(torch.float32).contiguous()
        b, _, h, w = x.shape
        self._prepare_shape(h, w)
        y = torch.empty((b, 3, h, w), dtype=torch.float32, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        with torch.cuda.device(x.device):
            capi.check(capi.lib().dsu_forward(handle, C.c_void_p(x.data_ptr()), b, h, w, C.c_void_p(y.data_ptr()),
                                              C.c_void_p(stream)), "dsu_forward")
        return y

    # ------------------------------------------------------------------ fused frame path
    def forward_frames(self, color: torch.Tensor, pos: torch.Tensor, edge: Optional[torch.Tensor] = None,
                       return_float: bool = False):
        """Device-resident frame loop body of test_stage1.py:60-70 / test_stage2.py:67-78:
        uint8 RGBA colour ``[B,H,W,4]`` + pos ``[B,H,W,4]`` (+ edge ``[B,H,W]`` for stage 2)
        -> uint8 RGBA result ``[B,H,W,4]`` (and optionally the fp32 network output)."""
        self._check_mode()
        for name, t in (("color", color), ("pos", pos)):
            if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[-1] != 4:
                raise RuntimeError("%s must be uint8 [B,H,W,4]" % name)
        handle = self._engine(color.device)
        color, pos = color.contiguous(), pos.contiguous()
        b, h, w, _ = color.shape
        self._prepare_shape(h, w)
        out = torch.empty((b, h, w, 4), dtype=torch.uint8, device=color.device)
        y = torch.empty((b, 3, h, w), dtype=torch.float32, device=color.device) if return_float else None
        edge_p = None
        if edge is not None:
            edge = edge.contiguous()
            edge_p = C.c_void_p(edge.data_ptr())
        stream = torch.cuda.current_stream(color.device).cuda_stream
        with torch.cuda.device(color.device):
            capi.check(capi.lib().dsu_forward_u8(handle, C.c_void_p(color.data_ptr()), C.c_void_p(pos.data_ptr()), edge_p,
                                                 b, h, w, C.c_void_p(out.data_ptr()),
                                                 C.c_void_p(y.data_ptr()) if y is not None else None,
                                                 C.c_void_p(stream)), "dsu_forward_u8")
        return (out, y) if return_float else out

    def forward_frames_host(self, color, pos, edge, out, device: torch.device):
        """Same with HOST (ideally pinned) uint8 tensors; copies in, runs, copies the RGBA result
        into ``out`` and synchronises (C ABI ``dsu_forward_u8_host``)."""
        self._check_mode()
        handle = self._engine(device)
        b, h, w, _ = color.shape
        self._prepare_shape(h, w)
        stream = torch.cuda.current_stream(device).cuda_stream
        with torch.cuda.device(device):
            capi.check(capi.lib().dsu_forward_u8_host(handle, C.c_void_p(color.data_ptr()), C.c_void_p(pos.data_ptr()),
                                                      C.c_void_p(edge.data_ptr()) if edge is not None else None,
                                                      b, h, w, C.c_void_p(out.data_ptr()), C.c_void_p(stream)),
                       "dsu_forward_u8_host")
        return out

    def algorithmic_flops(self, b: int, h: int, w: int) -> float:
        """2 x live MACs of one forward (SURVEY.md 8d; the dead stage-1 smoother conv excluded)."""
        dev = torch.device("cuda", self._handle_dev) if self._handle_dev is not None else next(self.parameters()).device
        return float(capi.lib().dsu_forward_flops(self._engine(dev), b, h, w))

    def workspace_bytes(self, b: int, h: int, w: int) -> int:
        dev = torch.device("cuda", self._handle_dev) if self._handle_dev is not None else next(self.parameters()).device
        return int(capi.lib().dsu_workspace_bytes(self._engine(dev), b, h, w))

    def kernel_launches(self, b: int, h: int, w: int) -> int:
        dev = torch.device("cuda", self._handle_dev) if self._handle_dev is not None else next(self.parameters()).device
        return int(capi.lib().dsu_forward_launches(self._engine(dev), b, h, w))

    def profile_layers(self, b: int, h: int, w: int, reps: int = 3):
        """Per-launch device time of one forward of this shape, measured with CUDA events around
        every launch on the current stream (C ABI ``dsu_profile_forward``).  Returns a list of
        ``(name, ms, algorithmic_flops)``; run a real forward of the same shape first so the
        workspace holds meaningful activations."""
        dev = torch.device("cuda", self._handle_dev)
        handle = self._engine(dev)
        self._prepare_shape(h, w)
        cap = 256
        ms = (C.c_double * cap)()
        fl = (C.c_double * cap)()
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            n = capi.lib().dsu_profile_forward(handle, b, h, w, reps, C.c_void_p(stream), ms, fl, cap)
        if n < 0:
            capi.check(n, "dsu_profile_forward")
        return [(capi.lib().dsu_step_name(handle, i).decode(), ms[i], fl[i]) for i in range(min(n, cap))]

    def step_kernels(self):
        """``(name, kernel)`` of every launch of the current plan (C ABI ``dsu_step_kernel``: "halo", "tap", "ric_halo"
        (stage-1 RIC with stencil and input staged in shared memory), "ric" (stage-1 RIC gathering from global memory), ...);
        valid after the first forward."""
        lib = capi.lib()
        out, i = [], 0
        while True:
            name = lib.dsu_step_name(self._handle, i).decode()
            if not name:
                return out
            out.append((name, lib.dsu_step_kernel(self._handle, i).decode()))
            i += 1

    def debug_buffer(self, buffer: int, plane: int, shape, dtype=torch.float16) -> torch.Tensor:
        """Test hook: host copy of an internal activation buffer (see dsu_debug_read)."""
        t = torch.empty(shape, dtype=dtype)
        capi.check(capi.lib().dsu_debug_read(self._handle, buffer, plane, C.c_void_p(t.data_ptr()),
                                             t.numel() * t.element_size()), "dsu_debug_read")
        return t


class GeneratorJ(_Generator):
    """Stage-2 contour restorer (training/models.py:24-129): plain 7x7 / 3x3 convolutions."""
    _KIND = capi.KIND_GENERATORJ
    _FIRST_K = 7


class GeneratorJ_RIC(_Generator):
    """Stage-1 geometry-aware stylizer (training/models.py:200-356): every convolution except the
    final 1x1 is a deformable conv with the fixed rotation-invariant offset field."""
    _KIND = capi.KIND_GENERATORJ_RIC
    _FIRST_K = 3

    def _prepare_shape(self, h: int, w: int):
        # the reference regenerates its coords when x.shape changes (models.py:296-300); the field
        # is batch independent, so it is handed to the engine once per (h, w)
        for lh, lw in ((h, w), (int(h / 2), int(w / 2)), (int(h / 4), int(w / 4))):
            if (lh, lw) not in self._offset_dims:
                field = ric_offsets(lh, lw)
                capi.check(capi.lib().dsu_set_ric_offsets(self._handle, lh, lw, C.c_void_p(field.data_ptr())),
                           "dsu_set_ric_offsets")
                self._offset_dims.add((lh, lw))
