"""cc / Logger / infinite_iter of the reference's utils.py (utils.py:8-35), H100 edition.

``cc`` moves to the local rank's CUDA device and refuses to fall back to the CPU.  The
tensorboardX writer is optional (it is not installed in this image): without it the
Logger keeps the last scalars in memory and prints nothing.
"""
from __future__ import annotations

import os

import torch


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
