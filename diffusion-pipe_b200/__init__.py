"""diffusion-pipe_b200: a Hopper-native (sm_90a) pipeline-parallel training engine that keeps the
plugin/operator surface of tdrussell/diffusion-pipe for its Flux training hot path.

Layout
  csrc/            hand-written CUDA kernels (wgmma / TMA / mbarrier) + the C ABI (include/dpipe.h)
  _lib.py          ctypes loader for libdpipe_b200.so (fails loudly when it is missing)
  ops.py           thin tensor-level wrappers over the C ABI
  flux_blocks.py   Flux double/single stream blocks as fused autograd Functions over those ops
  flux.py          FluxPipeline mirror of the reference's models/flux.py (to_layers/prepare_inputs/loss)
  pipe/            PipelineModule + 1F1B engine (replaces the DeepSpeed surface train.py uses)
  data_feed.py     split_batch / PipelineDataLoader / batch-index bookkeeping (bit-exact)
"""
__version__ = '0.1.0'
