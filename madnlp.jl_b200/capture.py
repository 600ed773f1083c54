"""One rule for replaying a fixed launch sequence as a CUDA graph, shared by the IPM prologues, the adaptive barrier and the refinement
step: the first call for a key runs eagerly (which also lets the solver instantiate its own internal graphs), the second captures, every
later call replays.  A call with another key starts over at eager, and reset() drops the graph (e.g. when a setting baked into it
changed)."""
from __future__ import annotations

import torch


class CapturedSequence:
    """`run(fn, key)` runs fn's launch sequence eager, captured, then replayed; with enabled=False every call runs eagerly.  The key
    names what the captured sequence bakes in (buffers, scalar arguments); it is held, so the objects it names stay alive as long as
    the graph may replay them."""

    def __init__(self, enabled=True):
        self.enabled = enabled
        self.key = None
        self.graph = None           # None: not run for `key` yet; False: ran eagerly once; then the captured torch.cuda.CUDAGraph

    def reset(self):
        self.key = self.graph = None

    def run(self, fn, key=None):
        if not self.enabled:
            fn()
            return
        if key != self.key:
            self.key, self.graph = key, None
        if self.graph is None:
            fn()
            self.graph = False
        elif self.graph is False:
            g = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            with torch.cuda.graph(g):
                fn()
            self.graph = g
            g.replay()
        else:
            self.graph.replay()
