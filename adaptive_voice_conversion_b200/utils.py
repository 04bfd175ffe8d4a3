"""cc / Logger / infinite_iter of the reference's utils.py (utils.py:8-35), H100 edition.

``cc`` moves to the local rank's CUDA device and refuses to fall back to the CPU.  The
tensorboardX writer is optional (it is not installed in this image): without it the
Logger keeps the last scalars in memory and prints nothing.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os

import numpy as np
import torch


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def upload_mels(data, keys, dev):
    """{key: data[key] as a float32 tensor on dev} of a set's arrays at the keys."""
    return {u: torch.from_numpy(np.ascontiguousarray(data[u], np.float32)).to(dev) for u in keys}


def exact_buckets(src_lens, ref_lens):
    """[((T, T_ref), pair indices)] in sorted key order: the pairs grouped by their exact lengths, each group in input
    order."""
    buckets = {}
    for i, key in enumerate(zip(src_lens, ref_lens)):
        buckets.setdefault(key, []).append(i)
    return sorted(buckets.items())


@contextlib.contextmanager
def eval_mode(model, dev):
    """Runs the block with `model` in eval mode, checks its engine's tensor-core status word on `dev` when the block
    ends normally and restores the previous training mode in any case."""
    was_training = model.training
    model.eval()
    try:
        yield
        model.engine(dev).check_tc_status()
    finally:
        model.train(was_training)


def local_device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("adaptive_voice_conversion_b200 needs a CUDA device (H100); there is no CPU fallback")
    return torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))


def cc(net):
    """utils.py:8-10 -- but always the local CUDA device."""
    return net.to(local_device())


class Logger:
    """utils.py:12-26 surface: scalar_summary / scalars_summary / text_summary."""

    def __init__(self, logdir="./log"):
        self.last = {}
        try:
            from tensorboardX import SummaryWriter  # optional
            self.writer = SummaryWriter(logdir)
        except Exception:
            self.writer = None

    def scalar_summary(self, tag, value, step):
        self.last[tag] = (value, step)
        if self.writer is not None:
            self.writer.add_scalar(tag, value, step)

    def scalars_summary(self, tag, dictionary, step):
        self.last[tag] = (dict(dictionary), step)
        if self.writer is not None:
            self.writer.add_scalars(tag, dictionary, step)

    def text_summary(self, tag, value, step):
        self.last[tag] = (value, step)
        if self.writer is not None:
            self.writer.add_text(tag, value, step)


def infinite_iter(iterable):
    """utils.py:28-35: restart the iterable forever."""
    while True:
        yielded = False
        for item in iterable:
            yielded = True
            yield item
        if not yielded:
            raise ValueError("infinite_iter over an empty iterable")
