"""CPU checks of `optimizer.Adam` (`--optim adam|adamw`): the ctypes mirror of mi3d_adam_cfg against the header, every refusal, and
the parameter-group keys against torch.optim.Adam's (so state dicts interchange)."""
import ctypes
import importlib
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

L = importlib.import_module("make-it-3d_b200._lib")
optim = importlib.import_module("make-it-3d_b200.optimizer")


def test_adam_cfg_mirror_matches_the_header(tmp_path):
    cls = L.AdamCfg
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mi3d.h"', 'int main(void) {',
           '  printf("size %zu\\n", sizeof(mi3d_adam_cfg));']
    src += [f'  printf("{f} %zu\\n", offsetof(mi3d_adam_cfg, {f}));' for f, _ in cls._fields_]
    src += ['  return 0;', '}']
    c = tmp_path / "cfg.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "cfg"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f
    assert "mi3d_adam_step" in L.SYMBOLS


def _param(*shape):
    return torch.nn.Parameter(torch.zeros(*shape))


@pytest.mark.parametrize("kw, match", [
    (dict(weight_decay=1e-2), "weight_decay"),
    (dict(amsgrad=True), "amsgrad"),
    (dict(maximize=True), "maximize"),
    (dict(capturable=True), "capturable"),
    (dict(differentiable=True), "differentiable"),
    (dict(fused=True), "fused"),
])
def test_unsupported_options_are_refused(kw, match, monkeypatch):
    with pytest.raises(L.Mi3dError, match=match):
        optim.Adam([_param(4)], **kw)
    # a later group with the option is refused as well (the first group's parameter passes: its GPU check is skipped)
    monkeypatch.setattr(optim, "_adam_check_param", lambda p: None)
    with pytest.raises(L.Mi3dError, match=match):
        optim.Adam([{'params': [_param(4)]}, dict(params=[_param(3)], **kw)])


def test_unsupported_parameters_are_refused():
    with pytest.raises(L.Mi3dError, match="fp32"):
        optim.Adam([torch.nn.Parameter(torch.zeros(4, dtype=torch.float16))])
    with pytest.raises(L.Mi3dError, match="fp32"):
        optim.Adam([torch.nn.Parameter(torch.zeros(4, 6).t())])
    with pytest.raises(L.Mi3dError, match="CUDA"):
        optim.Adam([_param(4)])


def test_multi_rank_process_group_is_refused(monkeypatch):
    monkeypatch.setattr(optim.dist, "is_available", lambda: True)
    monkeypatch.setattr(optim.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(optim.dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(L.Mi3dError, match="rank"):
        optim.Adam([_param(4)])


def test_hyper_parameters_are_validated_like_torch():
    for kw in (dict(lr=-1.0), dict(eps=-1.0), dict(betas=(1.0, 0.99)), dict(betas=(0.9, -0.1)), dict(clip_grad_norm=-1.0)):
        with pytest.raises(ValueError):
            optim.Adam([_param(4)], **kw)


def test_param_group_keys_equal_torch_adam(monkeypatch):
    # the parameter check is the only one that needs a GPU; skip it to build the groups on the CPU
    monkeypatch.setattr(optim, "_adam_check_param", lambda p: None)
    ps = [_param(4), _param(3)]
    mine = optim.Adam([{'params': [ps[0]], 'lr': 1e-2}, {'params': [ps[1]]}], lr=1e-3, betas=(0.9, 0.99), eps=1e-15)
    ref = torch.optim.Adam([{'params': [ps[0]], 'lr': 1e-2}, {'params': [ps[1]]}], lr=1e-3, betas=(0.9, 0.99), eps=1e-15)
    assert mine.param_groups[0].keys() == ref.param_groups[0].keys()
    assert mine.defaults.keys() == ref.defaults.keys()
    for a, b in zip(mine.param_groups, ref.param_groups):
        assert {k: v for k, v in a.items() if k != "params"} == {k: v for k, v in b.items() if k != "params"}
    assert mine.clip_grad_norm == 0.0
