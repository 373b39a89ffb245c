"""Device runtime: uploads a Plan, owns the workspace, runs / graph-replays op-table programs.

PyTorch is plumbing only: it allocates the two device buffers (weight arena, workspace), provides
the stream and moves I/O tensors.  Every kernel that touches the mel-latent tensor is launched by
libaldm_b200.so through the C-ABI; there is no torch fallback on this path.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .plan import Plan

_TORCH_DT = {"f32": torch.float32, "i64": torch.int64, "i32": torch.int32}


def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


class DeviceProgram:
    """A Plan resident on one GPU.  ``ranges`` maps a name to an (first, last) op range; each range
    is its own aldm_program so it can be run eagerly or replayed as a CUDA graph."""

    def __init__(self, plan: Plan, device: torch.device, ranges: Dict[str, Tuple[int, int]],
                 arena_dev: Optional[torch.Tensor] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("the native engine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.L = _lib.lib()
        self.plan = plan
        self.device = torch.device(device)
        _lib.check(self.L.aldm_device_check(self.device.index or 0), "device_check")
        self.arena = arena_dev if arena_dev is not None else plan.arena.to(self.device, non_blocking=False)
        assert self.arena.numel() >= plan.arena.numel()
        self.ws = torch.zeros(plan.ws_bytes + 4096, dtype=torch.uint8, device=self.device)
        self.handles: Dict[str, C.c_void_p] = {}
        self.captured: Dict[str, bool] = {}
        self._keep = []
        for name, (a, b) in ranges.items():
            arr = plan.resolve(self.arena.data_ptr(), self.ws.data_ptr(), a, b)
            h = C.c_void_p()
            _lib.check(self.L.aldm_program_create(arr, len(arr), C.byref(h)), f"program_create[{name}]")
            self.handles[name] = h
            self.captured[name] = False
        self._capture_stream = torch.cuda.Stream(device=self.device)

    # ---- I/O views into the workspace ----------------------------------------------------
    def view(self, name: str) -> torch.Tensor:
        kind, ref, shape = self.plan.io[name]
        dt = _TORCH_DT[kind]
        n = int(np.prod(shape)) * (8 if kind == "i64" else 4)
        assert ref.region == "ws"
        return self.ws[ref.off:ref.off + n].view(dt).reshape(shape)

    # ---- execution -----------------------------------------------------------------------
    def run(self, name: str):
        _lib.check(self.L.aldm_program_run(self.handles[name], _stream_ptr()), f"run[{name}]")

    def capture(self, name: str):
        """Run once eagerly (loads modules, sets smem attributes), then capture into a CUDA graph."""
        self.run(name)
        torch.cuda.current_stream().synchronize()
        s = self._capture_stream
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _lib.check(self.L.aldm_program_capture(self.handles[name], s.cuda_stream), f"capture[{name}]")
        torch.cuda.current_stream().wait_stream(s)
        self.captured[name] = True

    def replay(self, name: str):
        if not self.captured[name]:
            self.capture(name)
        _lib.check(self.L.aldm_program_replay(self.handles[name], _stream_ptr()), f"replay[{name}]")

    def num_launches(self, name: str) -> int:
        return int(self.L.aldm_program_num_launches(self.handles[name]))

    def close(self):
        for h in self.handles.values():
            self.L.aldm_program_destroy(h)
        self.handles = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# --------------------------------------------------------------------------------------------------
# thin wrappers over the stand-alone entry points (used by the sampler and by the tests)
# --------------------------------------------------------------------------------------------------
def ddim_step(x, eps_u, eps_c, noise, x_prev, a_t, a_prev, sigma_t, sqrt_one_minus_at, guidance, pred_x0=None):
    """aldm_ddim_step: p_sample_ddim's CFG combine + update (ddim.py:298-300,339-354)."""
    L = _lib.lib()
    for t in (x, eps_u, eps_c, noise, x_prev):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    _lib.check(L.aldm_ddim_step(x.data_ptr(), eps_u.data_ptr(), eps_c.data_ptr(), noise.data_ptr(), x_prev.data_ptr(),
                                pred_x0.data_ptr() if pred_x0 is not None else None, x.numel(),
                                a_t, a_prev, sigma_t, sqrt_one_minus_at, guidance, _stream_ptr()), "ddim_step")
    return x_prev


def stochastic_encode(x0, noise, c0: float, c1: float, clip_flag=None, out=None):
    """aldm_stochastic_encode: c0 * x0' + c1 * noise (ddim.py:434-449), x0' = clip(x0, -10, 10) when the device int32
    ``clip_flag`` is non-zero (AudioLDM 1's latent guard; None: no guard)."""
    L = _lib.lib()
    out = torch.empty_like(x0) if out is None else out
    for t in (x0, noise, out):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.shape == x0.shape
    if clip_flag is not None:
        assert clip_flag.is_cuda and clip_flag.dtype == torch.int32 and clip_flag.numel() == 1
    _lib.check(L.aldm_stochastic_encode(x0.data_ptr(), noise.data_ptr(), out.data_ptr(), x0.numel(), c0, c1,
                                        clip_flag.data_ptr() if clip_flag is not None else None, _stream_ptr()),
               "stochastic_encode")
    return out


def masked_blend(img, x0, mask, q_noise, sqrt_acp, sqrt_1m_acp):
    L = _lib.lib()
    B, Cc, T, Fq = img.shape
    _lib.check(L.aldm_masked_blend(img.data_ptr(), x0.data_ptr(), mask.data_ptr(), q_noise.data_ptr(), B, Cc, T * Fq,
                                   sqrt_acp, sqrt_1m_acp, _stream_ptr()), "masked_blend")
    return img


def stft_mel(wav: torch.Tensor, n_fft: int, hop: int, mel_basis: torch.Tensor, out_frames: Optional[int] = None):
    """aldm_stft_mel: TacotronSTFT.mel_spectrogram (stft.py:159-178) -> [B, frames, n_mels] log-mel."""
    L = _lib.lib()
    assert wav.is_cuda and wav.dtype == torch.float32 and wav.is_contiguous() and wav.dim() == 2
    B, T = wav.shape
    frames = T // hop + 1
    out_frames = frames if out_frames is None else out_frames
    n_mels = mel_basis.shape[0]
    out = torch.empty(B, out_frames, n_mels, dtype=torch.float32, device=wav.device)
    _lib.check(L.aldm_stft_mel(wav.data_ptr(), B, T, n_fft, hop, mel_basis.data_ptr(), n_mels, out.data_ptr(), out_frames,
                               _stream_ptr()), "stft_mel")
    return out


def posterior_sample(moments_nhwc: torch.Tensor, noise_nchw: torch.Tensor, scale: float):
    L = _lib.lib()
    B, H, W, C2 = moments_nhwc.shape
    zc = C2 // 2
    z = torch.empty(B, zc, H, W, dtype=torch.float32, device=moments_nhwc.device)
    _lib.check(L.aldm_posterior_sample(moments_nhwc.data_ptr(), noise_nchw.data_ptr(), z.data_ptr(), B, zc, H * W, scale,
                                       _stream_ptr()), "posterior_sample")
    return z
