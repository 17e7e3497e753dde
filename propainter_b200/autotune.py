"""Measured choice between numerically equivalent execution plans of one library-backed step.

cuDNN's own autotuner (config.CUDNN_BENCHMARK) picks the algorithm *inside* one conv call; it cannot decide between
different decompositions of the same math -- a grouped conv vs one dense conv per group, conv + our bias/ReLU epilogue
kernel vs cuDNN's fused conv-bias-ReLU.  `pick` times the candidates once per shape signature with CUDA events on the
current stream (during the eager warm-up runs that precede every graph capture, propainter_b200/graphs.py) and replays
the winner afterwards.  Inside a stream capture, or with config.AUTOTUNE off, an unmeasured signature runs candidate 0.
"""
import torch

from . import config

_choice = {}
_timings = {}          # (key, variant) -> ms per run of the graph-timed candidates (reported by bench.py)


def choices():
    return dict(_choice)


def pick(key, variants, *args, reps=5, graph_timed=False):
    """graph_timed: time every candidate as a captured CUDA graph (device time of the launch sequence, the way the stage
    will actually run) instead of eagerly -- for plans made of many small kernels an eager timing measures the host's
    launch rate, not the GPU."""
    if not args[0].is_cuda:                                 # choices are measured on the GPU: CPU inputs always run candidate 0
        return variants[0](*args)
    i = _choice.get(key)
    if i is None:
        if not config.AUTOTUNE or torch.cuda.is_current_stream_capturing():
            return variants[0](*args)
        best, i = None, 0
        for j, fn in enumerate(variants):
            try:
                fn(*args)
                fn(*args)                                   # cuDNN algorithm search / lazy packing happen here
                run = lambda: fn(*args)
                if graph_timed:
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        fn(*args)
                    run = g.replay
                    run()
            except RuntimeError:
                continue                                    # plan not supported for this shape by the library
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                run()
            e1.record()
            e1.synchronize()
            t = e0.elapsed_time(e1)
            if graph_timed:
                _timings[(key, j)] = t / reps
            if best is None or t < best:
                best, i = t, j
        _choice[key] = i
    return variants[i](*args)
