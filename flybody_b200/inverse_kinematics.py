"""Multi-site inverse kinematics on the device (reference `flybody/inverse_kinematics.py`), and walking datasets written from the fits.

`qpos_from_site_xpos` has the reference's arguments, defaults and results, with a `FlyModel` in place of the `physics` object.  A
target array [n_sites, 3] is one problem and gives results shaped like the reference's; [B, n_sites, 3] is B independent problems
(one env, one warp each, on the CUDA stepper) and puts a leading batch dimension on every result.  There is no CPU fallback: without the
CUDA library the call raises `StepperError`.

`write_walking_dataset` turns fitted tracks into the `.npz` layout `trajectory_loaders.HDF5WalkingTrajectoryLoader` reads, so that
`walk_imitation(ref_path=...)` trains on them directly.
"""
from collections import namedtuple

import numpy as np

from . import rewards, stepper as st
from .synthetic import mult_quat

IKResult = namedtuple('IKResult', ['qpos', 'err_norm', 'err_norm_first_term', 'steps', 'success'])

CHUNK = 4096                     # problems per device batch: memory stays bounded for any B


def _include_mask(include_inds, n_sites):
    mask = np.zeros(3 * n_sites, np.uint8)
    mask[np.arange(3 * n_sites)[include_inds]] = 1
    return mask


def qpos_from_site_xpos(model, site_names, target_xpos, joint_names, reg_strength=0.0, lr=0.01, beta=0.99, progress_threshold=0.01,
                        max_steps=20_000, include_inds=slice(None), init_qpos=None, device=0, lib_path=None):
    """Joint angles qpos whose sites `site_names` match `target_xpos`, moving only `joint_names` (hinge or free joints).

    Minimises ||s(q) - s*||^2 + reg_strength ||q_hinge||^2 by gradient descent with momentum, as the reference does: the fitted hinges'
    raw qpos are regularised, the objective is checked every 100 iterations from iteration 0, and a problem stops with success when
    lr * ||update|| / objective < progress_threshold (an objective of exactly 0 also counts as converged, where the reference divides by
    zero).  `include_inds` selects components of the flattened [n_sites, 3] targets; a NaN target component is dropped for its problem.
    `init_qpos` [nq] or [B, nq] is the start pose (default `model.qpos0`).

    Returns IKResult(qpos, err_norm, err_norm_first_term, steps, success): err_norm is the objective at the last check;
    err_norm_first_term is the site term at the returned qpos (the reference's is one update stale when it stops at max_steps without
    success); steps is the loop index at the stop, max_steps - 1 without success.  Values come from fp32 device arithmetic."""
    names = model.meta['site_names']
    site_ids = [names.index(s) for s in site_names]
    jnt_ids = [model.jnt_id(j) for j in joint_names]
    t = np.asarray(target_xpos, np.float64)
    single = t.ndim == 2
    t = t.reshape(-1, len(site_ids), 3)
    B = t.shape[0]
    q0 = model.qpos0 if init_qpos is None else np.asarray(init_qpos, np.float64)
    q0 = np.broadcast_to(q0.reshape(-1, model.nq), (B, model.nq))
    n_env = min(B, CHUNK)
    sim = st.BatchedStepper(model, n_env, device=device, lib_path=lib_path)
    try:
        sim.ik_program(site_ids, jnt_ids, _include_mask(include_inds, len(site_ids)), reg_strength, lr, beta, progress_threshold, max_steps)
        outs = []
        for a in range(0, B, n_env):
            sim.ik_solve(t[a:a + n_env], q0[a:a + n_env])
            outs.append(sim.ik_read())
    finally:
        sim.close()
    qpos, err, err1, steps, ok = (np.concatenate(c) for c in zip(*outs))
    res = IKResult(qpos.astype(np.float64), err.astype(np.float64), err1.astype(np.float64), steps.astype(np.int64), ok)
    if single:
        return IKResult(res.qpos[0], float(res.err_norm[0]), float(res.err_norm_first_term[0]), int(res.steps[0]), bool(res.success[0]))
    return res


def _root_joint(model):
    free = [j for j in range(model.njnt) if int(model.jnt_type[j]) == 0]
    if not free:
        raise ValueError('the model has no free joint to serve as the walker root')
    return free[0]


def _quat_velocity(q1, q2, dt):
    """MuJoCo mj_differentiatePos of a free joint's rotation: the body-frame angular velocity turning q1 into q2 in dt"""
    conj = q1 * np.array([1.0, -1, -1, -1])
    dq = mult_quat(conj, q2)
    axis = dq[..., 1:]
    s = np.linalg.norm(axis, axis=-1, keepdims=True)
    angle = 2 * np.arctan2(s, dq[..., :1])
    angle = np.where(angle > np.pi, angle - 2 * np.pi, angle)
    axis = np.where(s > 1e-15, axis / np.where(s > 1e-15, s, 1.0), np.array([1.0, 0, 0]))
    return axis * angle / dt


def _differentiate(qpos, root_qadr, hinge_qadr, dt):
    """forward differences of [T, nq] poses, last row repeated: root linear (world frame), root angular (body frame), hinges"""
    q = np.asarray(qpos, np.float64)
    lin = (q[1:, root_qadr:root_qadr + 3] - q[:-1, root_qadr:root_qadr + 3]) / dt
    ang = _quat_velocity(q[:-1, root_qadr + 3:root_qadr + 7], q[1:, root_qadr + 3:root_qadr + 7], dt)
    hv = (q[1:, hinge_qadr] - q[:-1, hinge_qadr]) / dt
    root_qvel = np.concatenate([lin, ang], 1)
    rep = lambda a: np.concatenate([a, a[-1:]]) if len(a) else np.zeros((1,) + a.shape[1:])
    return rep(root_qvel), rep(hv)


def write_walking_dataset(path, model, qpos_tracks, timestep, joint_names, site_names, device=0, lib_path=None):
    """Write fitted walking tracks as a dataset `walk_imitation(ref_path=path)` loads.

    qpos_tracks: one [T, nq] array or a list of them (full-model poses, e.g. `qpos_from_site_xpos` fits of consecutive frames);
    timestep: seconds between frames; joint_names: the hinges whose angles the dataset holds; site_names: the sites of root2site.
    root_qpos / qpos come from the tracks, root_qvel / qvel are forward differences (last row repeated; MuJoCo's mj_differentiatePos:
    hinge dq / dt, world-frame linear and body-frame angular root velocity), root2site and the hinges' egocentric axes come from one
    forward pass of each pose on the stepper through the observation items FB_OBS_SITES_EGO / FB_OBS_DOF_AXIS_EGO, and joint_quat
    from `rewards.joint_orientation_quat`."""
    tracks = [np.asarray(qpos_tracks, np.float64)] if np.ndim(qpos_tracks) == 2 else [np.asarray(t, np.float64) for t in qpos_tracks]
    rj = _root_joint(model)
    rq, root_body = int(model.jnt_qposadr[rj]), int(model.jnt_bodyid[rj])
    jid = [model.jnt_id(j) for j in joint_names]
    if any(int(model.jnt_type[j]) != 3 for j in jid):
        raise ValueError('joint_names must name hinge joints')
    hinge_qadr, hinge_dof = model.jnt_qposadr[jid].astype(np.int64), model.jnt_dofadr[jid].astype(np.int64)
    sid = [model.site_id(s) for s in site_names]
    ns, nj = len(sid), len(jid)
    frames = np.concatenate(tracks)
    n_env = min(len(frames), CHUNK)
    sim = st.BatchedStepper(model, n_env, device=device, lib_path=lib_path)
    try:
        dim = sim.obs_program([(st.OBS_SITES_EGO, 0, ns), (st.OBS_DOF_AXIS_EGO, ns, nj)], list(sid) + list(hinge_dof), root_body, 1)
        ego = np.zeros((len(frames), dim), np.float32)
        buf = np.zeros((n_env, dim), np.float32)
        for a in range(0, len(frames), n_env):
            chunk = frames[a:a + n_env]
            sim.reset(np.concatenate([chunk, np.repeat(chunk[-1:], n_env - len(chunk), 0)]))
            sim.task_inputs(np.zeros(n_env, np.int32), np.zeros(n_env, np.uint8))
            ego[a:a + len(chunk)] = sim.read_task_obs(buf)[:len(chunk)]
    finally:
        sim.close()
    root2site = ego[:, :3 * ns].astype(np.float64).reshape(-1, ns, 3)
    axes = ego[:, 3 * ns:].astype(np.float64).reshape(-1, nj, 3)
    d = {'timestep_seconds': np.float64(timestep), 'trajectory_lengths': np.asarray([len(t) for t in tracks], np.int64),
         'id2name/joints': np.array([j.split('/')[-1] for j in joint_names]), 'id2name/sites': np.array([s.split('/')[-1] for s in site_names])}
    off = 0
    for k, q in enumerate(tracks):
        T = len(q)
        root_qvel, qvel = _differentiate(q, rq, hinge_qadr, timestep)
        g = f'trajectories/{str(k).zfill(len(str(len(tracks))))}/'
        d[g + 'root_qpos'] = q[:, rq:rq + 7]
        d[g + 'qpos'] = q[:, hinge_qadr]
        d[g + 'root_qvel'] = root_qvel[:T]
        d[g + 'qvel'] = qvel[:T]
        d[g + 'root2site'] = root2site[off:off + T]
        d[g + 'joint_quat'] = rewards.joint_orientation_quat(axes[off:off + T], q[:, hinge_qadr])
        off += T
    np.savez(path, **d)
