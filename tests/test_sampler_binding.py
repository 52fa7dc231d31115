"""The extension's ``sample`` is keyword-only, with exactly ``ops.sample``'s parameter names and no defaults.

Several of its parameters are optional fp32 ``[rows]`` tensors (temperature, top_p, rep_penalty, min_p, presence,
frequency), so a positional slip would pass every check and sample with the wrong control; a forgotten argument must
fail rather than take a value.  None of these calls launches a kernel: a call that binds reaches the CPU-tensor check
first.  The raw module is called so that the launch counter is not bumped."""
from __future__ import annotations

import inspect
import re

import pytest
import torch

from bee2bee_b200 import ops

NAMES = list(inspect.signature(ops.sample).parameters)


def _raw_sample():
    return ops.native()._mod.sample


def _kwargs():
    # ops.sample's defaults, with a (CPU) tensor for the two parameters that have none
    return {name: (torch.zeros(1) if prm.default is inspect.Parameter.empty else prm.default)
            for name, prm in inspect.signature(ops.sample).parameters.items()}


def test_keyword_names_match_ops_sample():
    sig = _raw_sample().__doc__.splitlines()[0]
    m = re.fullmatch(r"sample\(\*, (.*)\) -> None", sig)
    assert m, sig
    names = re.findall(r"(\w+): ", m.group(1))
    assert len(names) == len(set(names)) == 26
    assert set(names) == set(NAMES)


def test_complete_keyword_call_binds():
    # every argument given: the call binds and stops at the device check, before any launch
    with pytest.raises(RuntimeError, match="logits: fp32"):
        _raw_sample()(**_kwargs())


def test_positional_call_is_refused():
    with pytest.raises(TypeError):
        _raw_sample()(*_kwargs().values())


@pytest.mark.parametrize("missing", NAMES)
def test_missing_argument_is_refused(missing):
    kw = _kwargs()
    del kw[missing]
    with pytest.raises(TypeError):
        _raw_sample()(**kw)
