"""CUDA-graph replay of `G.synthesis` for serving-style loops (fixed batch shape, changing latents and cameras).

One `G.synthesis` is ~250 kernel launches (libp3d.so kernels plus a few small ATen ops: affine layers, RNG draws,
casts). Captured once into a CUDA graph, a step becomes a single graph launch, so the host is off the critical
path -- the GPU-side replacement for what a tracing compiler would be used for. Random draws inside the capture
(stratified jitter, importance u) use torch's graph-safe Philox generator, so every replay draws fresh numbers.
"""
import torch


class GraphedSynthesis:
    """`gs = GraphedSynthesis(G, ws, c, noise_mode='const', neural_rendering_resolution=128)`; `out = gs(ws, c)`.

    The returned dict holds static output tensors that the next call overwrites."""

    def __init__(self, G, ws, c, warmup=2, **synthesis_kwargs):
        assert ws.is_cuda and c.is_cuda
        if G.rendering_kwargs.get('ray_start') == 'auto':
            # ImportanceRenderer.forward reads `torch.any(is_ray_valid).item()` for per-ray limits (renderer.py:94): a host
            # synchronisation, which a stream capture cannot contain
            raise ValueError("GraphedSynthesis: ray_start='auto' needs a host read-back per call; call G.synthesis directly")
        self.G = G
        self.kwargs = synthesis_kwargs
        self.ws = ws.clone()
        self.c = c.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(1, warmup)):      # allocate workspaces, build caches, JIT nothing
                G.synthesis(self.ws, self.c, **synthesis_kwargs)
        torch.cuda.current_stream().wait_stream(side)
        from . import _lib
        n0 = _lib.launch_count
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.out = G.synthesis(self.ws, self.c, **synthesis_kwargs)
        self.native_launches = _lib.launch_count - n0

    def __call__(self, ws, c):
        self.ws.copy_(ws, non_blocking=True)
        self.c.copy_(c, non_blocking=True)
        self.graph.replay()
        return self.out
