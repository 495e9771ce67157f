"""Per-kernel CUDA-event timing used by bench.py for the roofline object.

Spans are recorded on the CURRENT torch stream — the stream every libllmc_b200 kernel is
launched on (_lib.stream_ptr) — so the events bracket exactly the kernels of one C-ABI call.
Disabled (zero cost beyond one attribute check) unless bench.py enables it.
"""
import contextlib

import torch


class KernelTimer:
    def __init__(self):
        self.enabled = False
        self.records = []       # (name, start, end, flops, bytes)

    def reset(self):
        self.records = []

    @contextlib.contextmanager
    def span(self, name, flops=0.0, nbytes=0.0):
        if not self.enabled:
            yield
            return
        # Event.record() without a stream resolves "the current device" through
        # torch.cuda.is_available() -> cudaGetDeviceCount on every call (host time on every
        # record); an explicit stream object avoids that.
        st = torch.cuda.current_stream(torch.cuda.current_device())
        s = torch.cuda.Event(enable_timing=True)
        e = torch.cuda.Event(enable_timing=True)
        s.record(st)
        try:
            yield
        finally:
            e.record(st)
            self.records.append((name, s, e, flops, nbytes))

    def summary(self):
        """-> {name: dict(calls, ms, flops, bytes)}; call after torch.cuda.synchronize()."""
        out = {}
        for name, s, e, fl, by in self.records:
            d = out.setdefault(name, dict(calls=0, ms=0.0, flops=0.0, bytes=0.0))
            d['calls'] += 1
            d['ms'] += s.elapsed_time(e)
            d['flops'] += fl
            d['bytes'] += by
        return out


TIMER = KernelTimer()
