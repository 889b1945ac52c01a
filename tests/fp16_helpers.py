"""Shared by tests/test_fp16_cpu.py and tests/test_fp16_gpu.py: run the existing engine test helpers (tests/engine_helpers.py) in the
opt-in fp16 tensor-core mode.

The helpers select the compute dtype with ``model.to(dtype)``, and ``.to(torch.float16)`` selects bf16 by design (the reference's
``.half()`` call sites keep the default 16-bit format).  ``literal_fp16_to`` makes ``.to(torch.float16)`` mean
``set_compute_dtype(torch.float16)`` for the duration of a test, so every helper runs unchanged in fp16.
"""
import torch

from followyourclick_b200.modeling import ParamTreeModel


def literal_fp16_to(monkeypatch):
    orig = ParamTreeModel.to

    def to(self, *args, **kwargs):
        if kwargs.get("dtype") is torch.float16 or any(a is torch.float16 for a in args):
            kwargs.pop("dtype", None)
            rest = [a for a in args if a is not torch.float16]
            if rest or kwargs:
                orig(self, *rest, **kwargs)
            return self.set_compute_dtype(torch.float16)
        return orig(self, *args, **kwargs)

    monkeypatch.setattr(ParamTreeModel, "to", to)
