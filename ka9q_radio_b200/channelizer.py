"""Torch-tensor convenience wrapper over the C-ABI: device memory, streams and nothing else.

Mirrors how radiod drives filter.h (reference radio.c:582-620 setup, rx888.c:800-826 producer,
radio.c:1460 consumer) but batched: one forward launch pair and one channel launch per group of
blocks.  All arithmetic happens in libka9qgpu.so; torch only owns the buffers.
"""
from __future__ import annotations

import numpy as np
import torch

from . import capi


class Channelizer:
    def __init__(self, L: int, M: int, in_type: int, device: str | torch.device = "cuda:0", capacity: int = 1024,
                 extended: bool = False):
        """extended: also serve masters whose transform length has prime factors up to 23 (capi.Master)"""
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise capi.KgpuError("Channelizer needs a CUDA device; there is no CPU fallback")
        torch.cuda.set_device(self.device)
        capi.check(capi.load().kgpu_set_device(self.device.index or 0), "kgpu_set_device")
        self.master = capi.Master(L, M, in_type, extended)
        self.bank = capi.Bank(self.master, capacity)
        self.L, self.M, self.N, self.in_type = L, M, L + M - 1, in_type
        self.nchan = 0
        self._olen = {}
        self._real = {}
        self._tune = {}
        self.capacity = capacity

    # ---- channel management (create_filter_output + set_filter + shift) -------------------
    def add_channel(self, olen, shift, low=None, high=None, beta=None, response=None, isb=False, out_type=capi.KGPU_COMPLEX,
                    beam=None) -> int:
        """out_type KGPU_REAL: REAL-output slave (olen floats per block); beam=(i_weight, q_weight): beam synthesis."""
        idx = self.nchan
        pts = self.bank.define_any(idx, olen, out_type)
        if response is not None:
            self.bank.set_response(idx, response)
        else:
            self.bank.set_filter(idx, low, high, beta)
        self.bank.set_shift(idx, shift)
        if isb:
            self.bank.set_flags(idx, capi.KGPU_CHAN_ISB)
        if beam is not None:
            self.bank.set_weights(idx, beam[0], beam[1])
            self.bank.set_flags(idx, capi.KGPU_CHAN_BEAM)
        self._olen[idx] = (olen, pts)
        self._real[idx] = out_type == capi.KGPU_REAL
        self.nchan += 1
        return idx

    def tune(self, idx: int, shift: int, remainder: float, out_samprate: float, doppler_rate: float = 0.0) -> None:
        """Fine tuning fused into the channel kernel: the bookkeeping of radio.c:1476-1497 (set_osc on a new
        remainder, per-block phase step (shift % V)/V, one-time phase term on a shift change) expressed as
        kgpu_bank_set_osc parameters.  Call before channels() whenever compute_tuning's (shift, remainder) may
        have moved; a call with unchanged values is free."""
        import math

        st = self._tune.setdefault(idx, dict(bin_shift=-1000999, remainder=float("nan"), freq=0.0, rate=0.0, adj=0.0, on=False))
        changed, jump = False, 0.0
        if shift != st["bin_shift"] or math.isnan(st["remainder"]) or remainder != st["remainder"]:
            st["freq"] = -remainder / out_samprate                      # radio.c:1481
            st["rate"] = doppler_rate / (out_samprate * out_samprate)
            st["remainder"] = remainder
            changed = True
        if shift != st["bin_shift"]:
            V = 1 + self.L // (self.M - 1)                               # radio.c:1492
            st["adj"] = math.fmod(shift, V) / V                          # cispi(2 (shift % V) / V), C remainder
            jump = math.fmod((shift - st["bin_shift"]) / (-2.0 * (V - 1)) / 2.0, 1.0)  # radio.c:1494 in cycles
            st["bin_shift"] = shift
            self.bank.set_shift(idx, shift)
            changed = True
        if changed:
            phase = self.bank.osc_phase(idx) if st["on"] else 0.0       # set_osc starts an uninitialised phasor at 1
            self.bank.set_osc(idx, True, phase + jump, st["freq"], st["rate"], st["adj"])
            st["on"] = True

    # ---- data movement helpers -------------------------------------------------------------
    def stage_stream(self, samples: np.ndarray) -> torch.Tensor:
        """Host stream of nblocks*L new samples -> device tensor with the M-1 zero history the
        reference's zeroed ring provides at start-up (filter.c:242-244, :257-259)."""
        npad = self.M - 1
        if self.in_type == capi.KGPU_COMPLEX and samples.dtype == np.int16:
            npad *= 2  # interleaved I/Q
        pad = np.zeros(npad, samples.dtype)
        t = torch.from_numpy(np.concatenate([pad, samples]))
        return t.to(self.device)

    def fmt_of(self, t: torch.Tensor) -> int:
        return capi.KGPU_FMT_I16 if t.dtype == torch.int16 else capi.KGPU_FMT_F32

    def alloc_spectra(self, nblocks) -> torch.Tensor:
        return torch.empty((nblocks, self.master.spec_stride), dtype=torch.complex64, device=self.device)

    def alloc_outputs(self, nblocks) -> torch.Tensor:
        return torch.empty((nblocks, max(self.bank.out_stride, 1)), dtype=torch.complex64, device=self.device)

    # ---- the two halves of the path ----------------------------------------------------------
    def forward(self, d_stream: torch.Tensor, nblocks: int, spectra: torch.Tensor, scale: float = 1.0,
                first_block: int = 0, derandomize: bool = False, stats: torch.Tensor | None = None) -> None:
        i16 = d_stream.dtype == torch.int16
        if self.in_type == capi.KGPU_COMPLEX:
            esz = 4 if i16 else 8   # one I/Q pair
        else:
            esz = 2 if i16 else 4
        off = first_block * self.L * esz
        st = torch.cuda.current_stream(self.device).cuda_stream
        self.master.forward(d_stream.data_ptr() + off, self.fmt_of(d_stream), scale, nblocks, spectra.data_ptr(), st,
                            derandomize, stats.data_ptr() if stats is not None else 0)

    def apply_notches(self, spectra: torch.Tensor, nblocks: int) -> None:
        st = torch.cuda.current_stream(self.device).cuda_stream
        self.master.apply_notches(spectra.data_ptr(), nblocks, st)

    def channels(self, spectra: torch.Tensor, nblocks: int, outputs: torch.Tensor, power: torch.Tensor | None = None) -> None:
        """power: optional float32 [nblocks, capacity]; channels whose oscillator is on get their block power there."""
        st = torch.cuda.current_stream(self.device).cuda_stream
        self.bank.run(spectra.data_ptr(), nblocks, outputs.data_ptr(), st, power.data_ptr() if power is not None else 0)

    def alloc_power(self, nblocks) -> torch.Tensor:
        return torch.zeros((nblocks, self.capacity), dtype=torch.float32, device=self.device)

    def noise(self, spectra: torch.Tensor, nblocks: int, samprate: float) -> torch.Tensor:
        """N0 per block and channel (estimate_noise, radio.c:1783-1866) -> float64 [nblocks, capacity]"""
        n0 = torch.zeros((nblocks, self.capacity), dtype=torch.float64, device=self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        self.bank.noise(spectra.data_ptr(), nblocks, samprate, n0.data_ptr(), st)
        return n0

    def fm_front(self, outputs: torch.Tensor, nblocks: int):
        """FM discriminator front half (fm.c:104-131, :205-231) on the outputs channels() just wrote:
        -> (baseband float32 [nblocks, 2*row], stats float64 [nblocks, capacity, 2] = mean |y|, sum of squared deviations);
        channel idx's baseband samples are baseband[:, 2*out_offset(idx) : 2*out_offset(idx) + olen]."""
        bb = torch.zeros((nblocks, 2 * outputs.shape[1]), dtype=torch.float32, device=self.device)
        stats = torch.zeros((nblocks, self.capacity, 2), dtype=torch.float64, device=self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        self.bank.fm_front(outputs.data_ptr(), nblocks, bb.data_ptr(), stats.data_ptr(), st)
        return bb, stats

    def channel_slice(self, outputs: torch.Tensor, idx: int) -> torch.Tensor:
        off = self.bank.out_offset(idx)
        olen = self._olen[idx][0]
        if self._real.get(idx):  # olen floats packed into (olen+1)/2 complex slots
            return torch.view_as_real(outputs[:, off:off + (olen + 1) // 2]).reshape(outputs.shape[0], -1)[:, :olen]
        return outputs[:, off:off + olen]

    def close(self):
        self.bank.close()
        self.master.close()
