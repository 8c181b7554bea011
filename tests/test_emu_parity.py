"""CPU checks of the *kernel source* (host-emulation build, tests/_emu) against the oracle.
These are host-logic tests; the parity tests proper are tests/test_gpu_parity.py on the GPU."""
import os

import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model
from oracle import fly_oracle as fo
from conftest import walk_reset_qpos
from parity_common import (compare_stage_fields, teacher_forced_errors, summarize_tf, STAGE_TOL)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


@pytest.mark.parametrize('seed', [0, 2])
def test_stage_parity_walk(emu, seed):
    """seed 0: 55 rows (generic solver path); seed 2: 31 rows with six self-contacts (register path, both dof chains of a row)"""
    m = load_model('walk')
    compare_stage_fields(m, st.BatchedStepper(m, 2, lib_path=emu), seed=seed)


def test_stage_parity_flight(emu):
    m = load_model('flight')
    compare_stage_fields(m, st.BatchedStepper(m, 2, lib_path=emu), seed=1, vel_scale=20.0)


def test_teacher_forced_control_steps_walk(emu):
    m = load_model('walk')
    r = summarize_tf(*teacher_forced_errors(m, st.BatchedStepper(m, 1, lib_path=emu), n_steps=8, n_sub=10))
    assert r['p90_q'] < 2e-6 and r['p90_v'] < 2e-3 and r['hist_v']['<0.005'] >= 7, r
    assert r['p90_s'] < 1e-3, r          # per-substep sensor mean vs the oracle's control-step mean (8 steps: loose)


@pytest.mark.parametrize('ncap,seed', [('0', 0), ('32', 4)])
def test_solver_shared_and_global_memory_paths(emu, ncap, seed, monkeypatch):
    """The solver keeps an env's working set in its warp's shared-memory slice when nefc <= 32 and runs the
    same code on the global arrays otherwise; both placements must agree with the oracle.
    (seed 0 has nefc = 53 -> global path even with the default cap; seed 4 with pos_scale 0 has nefc = 18.)"""
    monkeypatch.setenv('FB_SOLVE_NCAP', ncap)
    m = load_model('walk')
    compare_stage_fields(m, st.BatchedStepper(m, 2, lib_path=emu), seed=seed, pos_scale=0.1 if seed == 0 else 0.0)


@pytest.mark.parametrize('chol_reg', [0, 8])
def test_hessian_block_fallback_path_matches_the_oracle(chol_reg, tmp_path):
    """The register solver factors its Hessian block in registers for up to FB_CHOL_REG = 24 columns and column by column in shared
    memory above that -- a path the steady-state walk (8 - 23 columns) rarely takes.  Built with FB_CHOL_REG = 0 (always the shared-memory
    form) and 8 (both forms within one solve) the kernel source must give the same answers against the oracle."""
    import subprocess
    lib = str(tmp_path / f'libfb_emu_chol{chol_reg}.so')
    subprocess.check_call(['g++', '-x', 'c++', '-DFB_EMU', f'-DFB_CHOL_REG={chol_reg}', '-O2', '-std=c++17', '-fPIC', '-shared', '-o', lib,
                           os.path.join(ge.CSRC, 'flybody_b200.cu'), '-lm'])
    m = load_model('walk')
    compare_stage_fields(m, st.BatchedStepper(m, 2, lib_path=lib), seed=4, pos_scale=0.0)        # 18 rows: the register solver
    r = summarize_tf(*teacher_forced_errors(m, st.BatchedStepper(m, 1, lib_path=lib), n_steps=3, n_sub=10))
    assert r['p90_q'] < 2e-6 and r['p90_v'] < 2e-3, r


def test_generic_convex_narrowphase_matches_the_oracle_on_shallow_contacts():
    """device MPR (double precision inside, fp32 inputs) vs the fp64 oracle on random sphere / capsule / ellipsoid /
    cylinder pairs brought to a 3e-4 cm overlap: same contact decision, depth within 2e-5 in >= 95 % of the cases (MPR is
    discontinuous where a support point jumps, e.g. across a cylinder rim)."""
    import ctypes as C
    from test_oracle_invariants import _convex, _rot, SPH, CAP, ELL, CYL
    ge.build()
    emu = C.CDLL(ge.EMU)
    fp = lambda a: np.ascontiguousarray(a, np.float32).ctypes.data_as(C.POINTER(C.c_float))
    emu.fb_emu_convex_pair.argtypes = [C.c_int] + [C.POINTER(C.c_float)] * 3 + [C.c_int] + [C.POINTER(C.c_float)] * 3 + [C.c_float, C.POINTER(C.c_float)]

    def dev(t1, p1, R1, s1, t2, p2, R2, s2):
        out = np.zeros(7, np.float32)
        n = emu.fb_emu_convex_pair(t1, fp(p1), fp(np.asarray(R1).reshape(9)), fp(s1), t2, fp(p2), fp(np.asarray(R2).reshape(9)), fp(s2), 0.0,
                                   out.ctypes.data_as(C.POINTER(C.c_float)))
        return n, float(out[0]), out[4:7].astype(np.float64)
    rs = np.random.RandomState(0)

    def size(t):
        if t == SPH:
            return [rs.uniform(0.01, 0.05), 0, 0]
        if t in (CAP, CYL):
            return [rs.uniform(0.005, 0.03), rs.uniform(0.01, 0.06), 0]
        return list(rs.uniform(0.005, 0.06, 3))
    tot = ok = 0
    for _ in range(200):
        t1, t2 = rs.choice([SPH, CAP, ELL, CYL], 2)
        s1, s2, R1, R2 = size(t1), size(t2), _rot(rs), _rot(rs)
        p1 = rs.normal(size=3) * 0.05
        u = rs.normal(size=3); u /= np.linalg.norm(u)
        lo, hi = 0.0, 0.3
        for _k in range(40):                      # bisect the separation to a 3e-4 overlap (oracle)
            mid = 0.5 * (lo + hi)
            n, dist, _, _ = _convex(t1, p1, R1, s1, t2, p1 + u * mid, R2, s2)
            lo, hi = (mid, hi) if (n and dist < -3e-4) else (lo, mid)
        p2 = p1 + u * lo
        n, dist, _, nrm = _convex(t1, p1, R1, s1, t2, p2, R2, s2)
        if not n:
            continue
        tot += 1
        nd, dd, nn = dev(t1, p1, R1, s1, t2, p2, R2, s2)
        ok += int(nd == 1 and abs(dd - dist) < 2e-5 and np.abs(nn - nrm).max() < 5e-2)
    assert tot > 150 and ok >= 0.95 * tot, (ok, tot)

