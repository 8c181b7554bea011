"""fp64 reference of MuJoCo's continuous-time mj_inverse at the oracle's state, for tests/test_inverse_dynamics.py.

After `Oracle.forward()` (or `step1`) the oracle holds the position / velocity stage of its state in double precision: the dense
inertia M, qfrc_bias, qfrc_passive, the dense constraint rows J with aref = -B J qvel - K imp (pos - margin) and D = 1 / R, and per
contact its row address, dimension and mu.  From these and a given qacc, `inverse` restates mj_inverse:
    jar = J qacc - aref,  efc_force = mj_constraintUpdate(jar)  (the oracle's constraint_update, fly_oracle.c, line for line),
    qfrc_constraint = J^T efc_force,  qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint.
Nothing here changes the oracle's state.
"""
import numpy as np

from oracle import fly_oracle as fo

CT_LIMIT, CT_FRICTIONLESS, CT_ELLIPTIC = 0, 1, 2      # fly_oracle.c efc types


def constraint_update(jar, D, kind, heads):
    """forces of the soft constraint model at jar (fly_oracle.c constraint_update): heads maps the first row of every elliptic contact
    to (mu, friction) -- mu of the regularised cone, friction of both tangent directions"""
    n = len(jar)
    f = np.zeros(n)
    i = 0
    while i < n:
        if kind[i] != CT_ELLIPTIC:
            f[i] = -D[i] * jar[i] if jar[i] < 0 else 0.0
            i += 1
            continue
        mu, fr = heads[i]
        U0, U1, U2 = jar[i] * mu, jar[i + 1] * fr, jar[i + 2] * fr
        N, T = U0, np.sqrt(U1 * U1 + U2 * U2)
        if mu * N + T <= 0 or (T <= 0 and N < 0):          # bottom zone
            f[i:i + 3] = -D[i:i + 3] * jar[i:i + 3]
        elif N >= mu * T or (T <= 0 and N >= 0):            # top zone
            pass
        else:                                               # middle zone
            Dm = D[i] / (mu * mu * (1 + mu * mu))
            f[i] = -Dm * (N - mu * T) * mu
            f[i + 1] = -f[i] / T * U1 * fr
            f[i + 2] = -f[i] / T * U2 * fr
        i += 3
    return f


def heads_of(o, impratio):
    """row address -> (mu, friction) of every condim-3 contact with rows at the oracle's state"""
    ncon = int(o.get(fo.NCON)[0])
    con = o.get(fo.CONTACT).reshape(-1, 16)[:ncon] if ncon else np.zeros((0, 16))
    out = {}
    for c in con:
        adr, dim, mu = int(c[12]), int(c[9]), float(c[11])
        if adr >= 0 and dim >= 3:
            out[adr] = (mu, mu * np.sqrt(impratio))     # CONTACT holds mu = friction / sqrt(impratio)
    return out


def inverse(m, o, qacc):
    """mj_inverse of the oracle's current state for accelerations qacc [nv]: dict of qfrc_inverse, qfrc_constraint, efc_force,
    qfrc_bias, qfrc_passive (fp64)"""
    nv = m.nv
    qacc = np.asarray(qacc, np.float64)
    M = o.get(fo.QM_DENSE).reshape(nv, nv)
    bias, passive = o.get(fo.QFRC_BIAS), o.get(fo.QFRC_PASSIVE)
    e = o.efc()
    jar = e['J'] @ qacc - e['aref']
    f = constraint_update(jar, e['D'], e['type'], heads_of(o, float(m.meta.get('opt_impratio', 1.0))))
    qc = e['J'].T @ f
    return dict(qfrc_inverse=M @ qacc + bias - passive - qc, qfrc_constraint=qc, efc_force=f, qfrc_bias=bias, qfrc_passive=passive,
                M=M, jar=jar)
