"""Shape-keyed CUDA-graph cache.

The hot path is launch-bound in the reference (~160 k ATen dispatches per 80-frame clip, SURVEY.md §0.4).
Every stage here has static shapes and no host-side data dependence (window masks, scan order and key
tables are resolved on the device or from shapes alone), so a stage call is captured once per shape
signature -- torch library kernels and our ctypes-launched kernels alike, both run on the capture
stream -- and replayed afterwards.  No tracing compiler: this is plain stream capture.
"""
import torch

from . import config, ops


def _switches():
    """execution switches that are baked into a capture: part of the cache key, so flipping one re-captures"""
    return (config.LINEAR_TF32, config.FUSED_EPILOGUE, config.AUTOTUNE, config.CUDNN_BENCHMARK, config.UMMA_CONV, config.SCAN_PRIORITY,
            config.HALF_OPERANDS, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)


_hp_streams = {}


def high_priority(fn):
    """Run fn() as a high-priority branch of the graph being captured (fork / join around it); outside a capture, or with
    config.SCAN_PRIORITY off, just call it.  Kernel nodes keep the priority of the stream they were captured on.  Used for
    the recurrent propagation scans: chains of small dependent kernels that otherwise queue behind the not yet dispatched
    CTAs of the big kernels other windows / clips have in flight (the work distributor hands out a kernel's CTAs in launch
    order within one priority level)."""
    if not (config.SCAN_PRIORITY and torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()):
        return fn()
    cur = torch.cuda.current_stream()
    key = (cur.device_index, cur.stream_id)
    hp = _hp_streams.get(key)
    if hp is None:
        hp = _hp_streams[key] = torch.cuda.Stream(device=cur.device, priority=-1)
    hp.wait_stream(cur)
    with torch.cuda.stream(hp):
        out = fn()
    cur.wait_stream(hp)
    return out


class GraphCache:
    """One cache per net.  max_entries bounds the number of live captures (least recently used is dropped, its private
    memory pool goes with it).  Every capture keeps its own memory pool: graphs that share a pool must never be replayed
    concurrently, and several of ours are (windows in flight on side streams, the two flow directions, two pipelines
    working on different clips) -- a shared pool was tried in round 2 and corrupted exactly those replays."""

    def __init__(self, enabled=True, warmup=2, max_entries=48):
        self.enabled, self.warmup, self.entries, self.max_entries = enabled, warmup, {}, max_entries

    def clear(self):
        self.entries = {}

    def __call__(self, key, fn, *inputs):
        """Run ``fn(*inputs)`` (tensors in, tensor / tuple of tensors out) through a captured graph.
        Returned tensors are fresh clones, so callers may keep them across replays."""
        if not (self.enabled and config.CUDA_GRAPHS) or not inputs[0].is_cuda:
            return fn(*inputs)
        if sum(x.numel() * x.element_size() for x in inputs) > config.GRAPH_MAX_INPUT_BYTES:
            # a capture pins its whole working set in a private pool; at 720p+ that is tens of GB per stage shape (a
            # 300-frame 720p clip pinned 150 GB) while the kernels are long enough for eager launches to keep up
            return fn(*inputs)
        key = (key, _switches()) + tuple((tuple(x.shape), x.dtype, x.device.index) for x in inputs)
        e = self.entries.pop(key, None)
        if e is not None:
            self.entries[key] = e                                   # re-insert: most recently used last
        if e is None:
            while len(self.entries) >= self.max_entries:
                self.entries.pop(next(iter(self.entries)))
            static_in = [x.detach().clone() for x in inputs]
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side), config.cudnn_autotune():   # lazy weight packing, cuDNN autotune, allocator warm-up
                for _ in range(self.warmup):
                    fn(*static_in)
            cur.wait_stream(side)
            torch.cuda.synchronize()
            l0 = ops.LAUNCHES
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph), config.cudnn_autotune():
                out = fn(*static_in)
            e = (graph, static_in, out, ops.LAUNCHES - l0)
            ops.LAUNCHES = l0                                   # capture records launches, it does not run them
            self.entries[key] = e
        graph, static_in, out, launches = e
        for s, x in zip(static_in, inputs):
            s.copy_(x)
        graph.replay()
        ops._count(launches)
        if isinstance(out, (tuple, list)):
            return tuple(o.clone() for o in out)
        return out.clone()
