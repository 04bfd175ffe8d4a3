"""adaptive_voice_conversion_b200 -- the AdaIN-VC (arXiv 1904.05742) forward/backward hot
path as hand-written sm_90a (H100) CUDA behind the reference's own Python API.

Public surface (mirrors the reference repo's modules):
    model.AE, solver.Solver, inference.Inferencer, utils.cc
"""
__all__ = ["AE", "Solver", "Inferencer"]


def __getattr__(name):  # lazy: importing the package must not require torch+CUDA up front
    if name == "AE":
        from .model import AE
        return AE
    if name == "Solver":
        from .solver import Solver
        return Solver
    if name == "Inferencer":
        from .inference import Inferencer
        return Inferencer
    raise AttributeError(name)
