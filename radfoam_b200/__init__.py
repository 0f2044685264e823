"""radfoam_b200 -- H100-native drop-in for radfoam's ``src/tracing`` hot path.

Public surface mirrors what ``import radfoam`` gives the reference's Python code for
this path (torch_bindings/pipeline_bindings.cpp:626-672):

    pipeline = radfoam_b200.create_pipeline(sh_degree, attr_dtype="float32")
    pipeline.trace_forward(...) / trace_backward(...) / trace_benchmark(...)

plus ``TraceRays`` (the autograd op of radfoam_model/render.py) and the ray-sharded
multi-GPU wrapper.  Importing the package does not import torch or load the CUDA
library; both happen on first use, and a missing library is a hard error (there is
no CPU fallback).
"""
from . import foam  # noqa: F401  (numpy/scipy only)

__all__ = ["create_pipeline", "Pipeline", "TraceRays", "TraceRaysParams", "SampleField", "ShardedTracer",
           "nearest_point", "starting_points", "locate_points", "farthest_neighbor", "foam", "library_path"]


def __getattr__(name):
    if name in ("create_pipeline", "Pipeline", "nearest_point", "starting_points", "locate_points",
                "farthest_neighbor"):
        from . import pipeline as _p
        return getattr(_p, name)
    if name in ("TraceRays", "TraceRaysParams", "SampleField"):
        from . import render as _r
        return getattr(_r, name)
    if name == "ShardedTracer":
        from . import sharded as _s
        return _s.ShardedTracer
    if name == "library_path":
        from . import _lib
        return _lib.library_path
    raise AttributeError(name)
