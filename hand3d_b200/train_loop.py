"""One CUDA graph per training iteration.

With a device-resident reader (BinaryDbReader(..., device_resident=True)) every part of a training iteration only enqueues device
work: the reader's queue, gather and augmentation, the forward, the loss, the backward and the Adam step.  GraphedIteration captures
such an iteration once and replays it, so the host does one graph launch per iteration.

    run = GraphedIteration(iteration)          # iteration() -> e.g. the loss, detached
    for i in range(max_iter):
        opt.set_lr(scheduler.get_lr(i))        # host-side changes go between replays, never inside the iteration
        loss = run()

The replays compute what the same number of eager calls computes, bit for bit.
"""
from __future__ import annotations

import gc

import torch


class GraphedIteration:
    """Calls 1..warmup run `iteration()` eagerly on a side stream: they size the operator scratch and create the gradients that the
    captured backward accumulates into.  The next call captures it into a CUDA graph and replays it; every later call replays it.
    Each call returns the outputs of the captured call, whose storage every replay overwrites.

    `iteration` must return no tensor that still holds an autograd graph (return loss.detach()): a graph of an earlier iteration that
    is alive at the capture would be reused with the stream it was made on."""

    def __init__(self, iteration, warmup=2):
        if warmup < 1:
            raise ValueError("GraphedIteration needs at least one eager warm-up call")
        self.iteration, self.warmup = iteration, int(warmup)
        self.graph, self._out, self._calls = None, None, 0

    def __call__(self):
        if self.graph is None and self._calls < self.warmup:
            self._calls += 1
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                out = self.iteration()
            torch.cuda.current_stream().wait_stream(side)
            return out
        if self.graph is None:
            gc.collect()
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._out = self.iteration()
        self.graph.replay()
        return self._out
