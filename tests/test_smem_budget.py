"""Shared-memory budget of the step kernels.  The kernels are compiled for FB_MINB resident 4-warp CTAs per SM
(fb_types.h), so that a 4096-env batch runs in one wave on an H100; a kernel whose CTA asks for more shared memory
than an SM can give FB_MINB CTAs runs in fewer and leaves a second, almost empty wave.  The CPU test checks the
requested bytes (host-emulation build, which sizes every slice exactly as the GPU launch does); the GPU test asks
the device how many CTAs fit."""
import os
import re

import pytest

import __graft_entry__ as ge
from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEP_KERNELS = {'smooth', 'solve', 'finish', 'pos', 'col', 'proj', 'vel'}
MODELS = ['walk', 'flight', 'vision']
SM90_SMEM_PER_SM = 228 * 1024          # shared memory of one sm_90 SM
SM90_SMEM_PER_CTA_RESERVED = 1024      # reserved by the system for every resident CTA


def compiled_min_blocks():
    src = open(os.path.join(ROOT, 'flybody_b200', 'csrc', 'fb_types.h')).read()
    return int(re.search(r'#define FB_MINB (\d+)', src).group(1))


@pytest.mark.parametrize('variant', MODELS)
def test_step_kernels_fit_the_compiled_blocks_per_sm(variant):
    ge.build()
    minb = compiled_min_blocks()
    sim = st.BatchedStepper(load_model(variant), 4, lib_path=ge.EMU)     # 4 envs: the sweep program is copied per CTA too
    budget = sim.step_kernel_smem()
    sim.close()
    assert set(budget) == STEP_KERNELS
    for name, (nbytes, _) in budget.items():
        assert nbytes + SM90_SMEM_PER_CTA_RESERVED <= SM90_SMEM_PER_SM // minb, (variant, name, nbytes)


@pytest.mark.gpu
@pytest.mark.parametrize('variant,n_envs', [('walk', 4096), ('flight', 4096), ('vision', 1024)])
def test_step_kernels_reach_the_compiled_blocks_per_sm(variant, n_envs):
    import torch
    props = torch.cuda.get_device_properties(0)
    ge.build()
    minb = compiled_min_blocks()
    sim = st.BatchedStepper(load_model(variant), n_envs, device=0)
    budget = sim.step_kernel_smem()
    sim.close()
    assert set(budget) == STEP_KERNELS
    for name, (nbytes, blocks) in budget.items():
        # blocks: the device's occupancy calculation (its shared memory per SM, the per-CTA reservation, registers)
        assert nbytes * minb <= props.shared_memory_per_multiprocessor, (variant, name, nbytes, props.name)
        assert blocks >= minb, (variant, name, nbytes, blocks, props.name)
