"""Helpers shared by the parity tests: run the CPU oracle (forward + autograd backward) on synthetic inputs."""
import os

import torch

from oracle import synth, univl_oracle

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name):
    """tests/golden/ref_<name>.pt; a golden kept under the 1 MB file limit by splitting lists its continuation files in
    "after_parts", whose "after" lists extend its own"""
    gold = torch.load(os.path.join(GOLDEN_DIR, "ref_%s.pt" % name), weights_only=False)
    for part in gold.pop("after_parts", []):
        gold["after"] = gold["after"] + torch.load(os.path.join(GOLDEN_DIR, part), weights_only=False)["after"]
    return gold


def run_oracle(cfg, batch, sd=None, seed=0, backward=True, dtype=torch.float32, bf16_emulation=False):
    if bf16_emulation:
        with univl_oracle.emulate_bf16():
            return run_oracle(cfg, batch, sd=sd, seed=seed, backward=backward, dtype=dtype)
    sd = sd if sd is not None else synth.make_state_dict(cfg, seed=seed)
    ties = synth.tied_keys(cfg)
    leaf = {}
    for k, v in sd.items():
        if k in ties:
            continue
        leaf[k] = v.detach().clone().to(dtype).requires_grad_(backward)
    full = dict(leaf)
    for alias, owner in ties.items():
        full[alias] = leaf[owner]
    b = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
    loss, parts = univl_oracle.univl_forward(full, cfg, b, return_parts=True)
    grads = {}
    if backward:
        loss.backward()
        grads = {k: v.grad for k, v in leaf.items() if v.grad is not None}
    return loss.detach(), parts, grads
