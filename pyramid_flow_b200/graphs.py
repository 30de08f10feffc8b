"""CUDA-graph capture and replay of a DiT step, shared by B200FluxTransformer and B200MMDiT.

A step is a fixed sequence of ~200-300 kernel launches.  With `use_cuda_graph = True` it is captured once per (plan, model
switches, input shapes and dtypes) and replayed, so the step does not depend on how fast the host can walk the launch
sequence (ctypes + descriptor encoding per launch).  Off by default: callers that reuse shapes for many steps (sampler,
bench) turn it on.  A model class mixes this in and supplies:

  _forward_eager(clips, timestep_ratio, enc, mask, pooled) -> [velocity]   the host-launched step
  _graph_key_fields() -> tuple        its switches that change the launch sequence (part of the capture key)
  _graph_prealloc(plan, clips)        allocates, outside the capture, everything the step uses (workspace, peer arena)
  plan_for(clip_shapes, mask)         the step's SeqPlan (the capture keeps it, and the device tables it holds, alive)
"""
from __future__ import annotations

from typing import Dict

import torch

from . import _lib

MAX_GRAPHS = 3          # every entry pins a workspace (~1.5 GB at 768p)


class GraphedStep:
    def _init_graphs(self) -> None:
        self.use_cuda_graph = False
        self._graphs: "Dict[tuple, dict]" = {}
        self._graph_warm = False
        self._graph_pool = None
        self._graph_stream = None
        self.graph_replays = 0          # bookkeeping for bench.py: replays and kernel launches replayed
        self.graph_launches_replayed = 0

    def _forward_graphed(self, clips, timestep_ratio, enc, mask, pooled):
        """Replay the step's captured launch sequence; inputs are copied into the capture's static buffers."""
        dev = self.device
        plan = self.plan_for([cl.shape for cl in clips], mask)
        ins = [*clips, timestep_ratio, enc, pooled]
        key = (id(plan), *self._graph_key_fields(), tuple((tuple(x.shape), x.dtype) for x in ins))
        ent = self._graphs.get(key)
        if ent is None:
            while len(self._graphs) >= MAX_GRAPHS:
                self._graphs.pop(next(iter(self._graphs)))
            static = [torch.empty(x.shape, dtype=x.dtype, device=dev) for x in ins]
            for st, x in zip(static, ins):
                st.copy_(x, non_blocking=True)
            nclip = len(clips)

            def run():
                return self._forward_eager(static[:nclip], static[nclip], static[nclip + 1], mask, static[nclip + 2])[0]

            # allocate outside the capture (ordinary allocator pool); a parallel layout also (re)builds its peer arena here,
            # a collective that must not happen inside stream capture
            self._graph_prealloc(plan, clips)
            # Nothing host-side may initialise inside stream capture: `_lib.require_device()` has already loaded every kernel
            # instantiation and set its shared-memory attribute on this device (pf_warmup), so a new shape that
            # dispatches to a not-yet-used template instantiation is safe to capture; the first capture of the process
            # additionally runs the step once host-launched (allocator pools, plan upload).
            if not self._graph_warm:
                run()
                self._graph_warm = True
            # Manual capture on a side stream (what torch.cuda.graph() does, minus its gc.collect() + empty_cache(), which
            # cost ~50 ms per capture and made the per-(unit, stage) captures of the sampler a net loss at 384p); all
            # graphs share one memory pool, so the buffers of an evicted graph are reused by the next capture.
            if self._graph_pool is None:
                self._graph_pool = torch.cuda.graph_pool_handle()
                self._graph_stream = torch.cuda.Stream()
            graph = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            side = self._graph_stream
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                graph.capture_begin(pool=self._graph_pool)
                try:
                    out = run()
                finally:
                    graph.capture_end()
            torch.cuda.current_stream().wait_stream(side)
            # the captured pointers must stay allocated as long as the graph lives: workspaces and plan
            ent = dict(graph=graph, static=static, out=out, launches=_lib.launch_count() - n0, plan=plan, mask=mask,
                       ws=dict(self._ws))
            self._graphs[key] = ent
        else:
            for st, x in zip(ent["static"], ins):
                st.copy_(x, non_blocking=True)
        self.last_plan = ent["plan"]
        ent["graph"].replay()
        self.graph_replays += 1
        self.graph_launches_replayed += ent["launches"]
        return [ent["out"].clone()]
