"""Inference runtime: CUDA-graph capture of a whole network forward and a host<->device pipeline.

The reference launches ~70 framework kernels per student frame from Python (train/model_seg.py:337-366); at H100
speeds the frame is launch-bound long before it is HBM- or tensor-bound (SURVEY section 8d), so the whole forward is
captured once into a CUDA graph and replayed.  `InferencePipeline` overlaps the H2D copy of frame i+1, the graph
replay of frame i and the D2H copy of frame i-1 on three streams.
"""
from __future__ import annotations

import collections
from typing import List, Optional

import torch

from . import _lib


def bind_host_thread_to_gpu(device_index: int = 0) -> Optional[int]:
    """Pin the calling thread (and the threads / pinned allocations it creates afterwards) to the CPUs NVML reports as
    local to GPU `device_index`.  A host-driven pipeline that streams 25 MB frames over PCIe loses ~40 % of its H2D
    bandwidth when its pinned buffers sit on the other socket (1.2 k vs 2.0 k frames/s measured between otherwise
    identical boxes).  Returns the number of CPUs in the new affinity mask, or None when NVML is unavailable or refuses
    (the call is best effort and never raises)."""
    try:
        import os

        import pynvml
        pynvml.nvmlInit()
        phys = device_index
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        if vis:
            ids = [v.strip() for v in vis.split(",") if v.strip()]
            if device_index < len(ids) and ids[device_index].isdigit():
                phys = int(ids[device_index])
        handle = pynvml.nvmlDeviceGetHandleByIndex(phys)
        pynvml.nvmlDeviceSetCpuAffinity(handle)
        return len(os.sched_getaffinity(0))
    except Exception:  # noqa: BLE001 -- best effort
        return None


class LaunchCounter:
    """Counts C-ABI kernel launches (every successful `check()` of a launching call) -- used for bench.py's
    `gpu_launches` claim."""

    def __init__(self):
        self.n = 0
        self.by_name = collections.Counter()   # launches per C-ABI call name (e.g. "fsb_conv_fwd")
        self._orig = None

    def __enter__(self):
        import fasterseg_b200.functional as F_
        self._orig = F_.check
        counter = self

        def counting_check(rc, what=""):
            counter.n += 1
            counter.by_name[what] += 1
            return counter._orig(rc, what)

        F_.check = counting_check
        return self

    def __exit__(self, *exc):
        import fasterseg_b200.functional as F_
        F_.check = self._orig


class GraphedInference:
    """Capture `model` (eval mode) once for a fixed input shape; `__call__` replays it.

    mode = "logits": output is the upsampled NCHW logits tensor (dtype `logits_dtype`)
    mode = "labels": output is the uint8 argmax label map (fused upsample+argmax)
    The example input fixes the input format: an fp32 / fp16 NCHW frame, or -- after model.set_input_normalization(mean, std) --
    the uint8 HWC image itself as `img_u8.permute(0, 3, 1, 2)` (evaluator path: 4x less host->device traffic).
    The input is read from `self.static_input`; `__call__(x)` first copies x into it (device->device or
    host->device on the current stream).
    """

    def __init__(self, model, example_input: torch.Tensor, mode: str = "logits", logits_dtype=torch.float16, warmup: int = 3):
        assert mode in ("logits", "labels")
        assert example_input.is_cuda
        _lib.lib()  # fail loudly before anything else if the native library is missing
        self.model = model.eval()
        self.mode = mode
        self.static_input = example_input.clone()
        if hasattr(model, "logits_dtype"):
            model.logits_dtype = logits_dtype
        self.launches_per_replay = 0
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(1, warmup)):  # populates packed-weight / folded-BN caches outside the graph
                self._run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with LaunchCounter() as lc, torch.no_grad(), torch.cuda.graph(self.graph):
            self.static_output = self._run()
        self.launches_per_replay = lc.n
        torch.cuda.synchronize()

    def _run(self):
        if self.mode == "labels":
            return self.model.predict_labels(self.static_input)
        return self.model(self.static_input)

    def replay(self):
        self.graph.replay()
        return self.static_output

    def __call__(self, x: Optional[torch.Tensor] = None):
        if x is not None:
            self.static_input.copy_(x, non_blocking=True)
        return self.replay()


class InferencePipeline:
    """End-to-end host->device->host inference with `depth` frames in flight.

    submit(host_tensor_pinned) enqueues H2D (copy-in stream) -> graph replay (compute stream) -> D2H of the result
    into a pinned host buffer (copy-out stream); results come back in order from `collect()`.
    Each slot owns its own captured graph + static buffers, so consecutive frames do not serialise on one input buffer.
    """

    def __init__(self, model, example_input: torch.Tensor, mode: str = "labels", depth: int = 3, logits_dtype=torch.float16):
        self.slots: List[GraphedInference] = [GraphedInference(model, example_input, mode, logits_dtype) for _ in range(depth)]
        self.depth = depth
        self.h2d = torch.cuda.Stream()
        self.compute = torch.cuda.Stream()
        self.d2h = torch.cuda.Stream()
        out = self.slots[0].static_output
        self.host_out = [torch.empty(out.shape, dtype=out.dtype, pin_memory=True) for _ in range(depth)]
        self.ev_in = [torch.cuda.Event() for _ in range(depth)]
        self.ev_done = [torch.cuda.Event() for _ in range(depth)]
        self.ev_out = [torch.cuda.Event() for _ in range(depth)]
        self._next = 0
        self._pending: List[int] = []
        self.h2d_bytes = example_input.numel() * example_input.element_size()
        self.d2h_bytes = out.numel() * out.element_size()
        self.launches_per_frame = self.slots[0].launches_per_replay

    def submit(self, host_x: torch.Tensor):
        i = self._next
        self._next = (i + 1) % self.depth
        if len(self._pending) >= self.depth:
            raise RuntimeError("pipeline full: collect() before submitting more")
        slot = self.slots[i]
        with torch.cuda.stream(self.h2d):
            # slot i's previous frame was collect()ed (host waited for its D2H, which followed its compute), so
            # static_input / static_output / host_out of this slot are free to be overwritten
            slot.static_input.copy_(host_x, non_blocking=True)
            self.ev_in[i].record(self.h2d)
        with torch.cuda.stream(self.compute):
            self.compute.wait_event(self.ev_in[i])
            slot.graph.replay()
            self.ev_done[i].record(self.compute)
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(self.ev_done[i])
            self.host_out[i].copy_(slot.static_output, non_blocking=True)
            self.ev_out[i].record(self.d2h)
        self._pending.append(i)

    def collect(self) -> torch.Tensor:
        i = self._pending.pop(0)
        self.ev_out[i].synchronize()
        return self.host_out[i]

    def run(self, host_frames, consume=None):
        """Process an iterable of pinned host frames, keeping `depth` in flight; returns the number of frames."""
        n = 0
        for x in host_frames:
            if len(self._pending) >= self.depth:
                r = self.collect()
                if consume is not None:
                    consume(r)
            self.submit(x)
            n += 1
        while self._pending:
            r = self.collect()
            if consume is not None:
                consume(r)
        return n
