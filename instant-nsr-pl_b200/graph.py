"""CUDA-graph execution of a whole training step (replacement for launching ~40 small kernels per
step from Python: the reference's per-step host cost dominates once the kernels take well under a millisecond).

    step = GraphedStep(model, loss_fn, n_rays, batch_spec={'rgb': (3,)})
    loss = step(rays, rgb=rgb, background_color=bg)        # copies into static buffers, replays the graph
    # parameter .grad tensors are static buffers refreshed by every replay

The captured region is ``out = model.forward_(rays, static=True); loss = loss_fn(out, batch); loss.backward()``:
march, visibility pre-pass, compaction, fused forward, loss, fused backward -- no host synchronisation inside
(sample counts live on the device).  loss_fn must be capturable (no .item(), no boolean-mask indexing).
Build it BEFORE running eager steps on the same parameters, or drop every reference to earlier outputs / losses first:
autograd AccumulateGrad nodes kept alive by an old graph are bound to the default stream, which invalidates capture.
"""
import torch

from .lib import lib


class GraphedStep:
    def __init__(self, model, loss_fn, n_rays, batch_spec=None, device=None, warmup=3, refresh_half_params=False, post_backward=None):
        self.model, self.loss_fn = model, loss_fn
        self.post_backward = post_backward  # e.g. the NCCL gradient all-reduce: captured into the same graph
        dev = device or next(model.parameters()).device
        self.params = [p for p in model.parameters() if p.requires_grad]
        self.rays = torch.zeros(n_rays, 6, device=dev)
        self.rays[:, 5] = 1.0
        self.batch = {k: torch.zeros((n_rays,) + tuple(shape), device=dev) for k, shape in (batch_spec or {}).items()}
        self.background_color = torch.ones(3, device=dev)
        self.refresh_half_params = refresh_half_params
        self.graph = None
        self.loss = None
        self.out = None
        self._capture(warmup)

    def _run(self):
        m = self.model
        m.background_color = self.background_color
        if self.refresh_half_params:  # parameters changed outside the graph (optimizer step): re-derive the fp16 copies
            for mod in m.modules():
                if hasattr(mod, '_half_key'):
                    mod._half_key = None
        out = m.forward_(self.rays, static=True)
        loss = self.loss_fn(out, self.batch)
        loss.backward()
        if self.post_backward is not None:
            self.post_backward()
        return out, loss

    def _capture(self, warmup):
        m = self.model
        if not m.training:
            raise RuntimeError('GraphedStep captures a training step: call model.train() first')
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(max(1, warmup)):
                for p in self.params:
                    p.grad = None
                self._run()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        for p in self.params:
            p.grad = None
        self.graph = torch.cuda.CUDAGraph()
        before = lib.launches
        with torch.cuda.graph(self.graph):
            self.out, self.loss = self._run()
        self.launches_per_replay = lib.launches - before  # our kernels inside the graph (torch's own nodes not counted)
        fused = getattr(m, '_fused', None)   # the captured step's device-side sample counts (an eager forward later replaces last_stats)
        self._counts = fused.last_stats.get('counts_dev') if fused is not None and isinstance(getattr(fused, 'last_stats', None), dict) else None
        torch.cuda.synchronize()

    def __call__(self, rays, background_color=None, **batch):
        """rays [n_rays,6] (host pinned or device); returns the (static) loss tensor.  No host sync."""
        self.rays.copy_(rays, non_blocking=True)
        for k, v in batch.items():
            self.batch[k].copy_(v, non_blocking=True)
        if background_color is not None:
            self.background_color.copy_(background_color, non_blocking=True)
        self.graph.replay()
        lib.launches += self.launches_per_replay
        return self.loss

    def counts(self):
        """(n_marched, n_kept) of the last replay -- one device->host read."""
        c = self._counts
        if c is None:
            raise RuntimeError('GraphedStep.counts(): the captured model exposes no device-side sample counts')
        return tuple((torch.cat(list(c)) if isinstance(c, (tuple, list)) else c).tolist())
