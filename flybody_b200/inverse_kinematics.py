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
FREE, HINGE = 0, 3               # mjtJoint


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
    B = np.size(target_xpos) // (3 * len(site_ids))
    q0 = np.broadcast_to(np.reshape(model.qpos0 if init_qpos is None else init_qpos, (-1, model.nq)), (B, model.nq))

    def run(sim, rows, k):
        sim.ik_solve(*rows)
        return sim.ik_read()

    single, (qpos, err, err1, steps, ok) = st._batched(
        model, [('target_xpos', target_xpos, (len(site_ids), 3)), ('init_qpos', q0, (model.nq,))], run, CHUNK,
        setup=lambda sim: sim.ik_program(site_ids, jnt_ids, _include_mask(include_inds, len(site_ids)), reg_strength, lr, beta,
                                         progress_threshold, max_steps),
        device=device, lib_path=lib_path)
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


def _differentiate_pos(model, q1, q2, dt):
    """MuJoCo mj_differentiatePos for rows of poses q1, q2 [T, nq] -> [T, nv]: hinge dq / dt; free joint world-frame linear and body-frame
    angular velocity; ball joint body-frame angular velocity"""
    out = np.zeros((q1.shape[0], model.nv))
    for j in range(model.njnt):
        t, qa, da = int(model.jnt_type[j]), int(model.jnt_qposadr[j]), int(model.jnt_dofadr[j])
        if t == HINGE:
            out[:, da] = (q2[:, qa] - q1[:, qa]) / dt
            continue
        if t == FREE:
            out[:, da:da + 3] = (q2[:, qa:qa + 3] - q1[:, qa:qa + 3]) / dt
            qa, da = qa + 3, da + 3
        out[:, da:da + 3] = _quat_velocity(q1[:, qa:qa + 4], q2[:, qa:qa + 4], dt)
    return out


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
    rq, rv, root_body = int(model.jnt_qposadr[rj]), int(model.jnt_dofadr[rj]), int(model.jnt_bodyid[rj])
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
        v = _differentiate_pos(model, q[:-1], q[1:], timestep)    # forward differences, last row repeated
        v = np.concatenate([v, v[-1:]]) if len(v) else np.zeros((1, model.nv))
        g = f'trajectories/{str(k).zfill(len(str(len(tracks))))}/'
        d[g + 'root_qpos'] = q[:, rq:rq + 7]
        d[g + 'qpos'] = q[:, hinge_qadr]
        d[g + 'root_qvel'] = v[:T, rv:rv + 6]
        d[g + 'qvel'] = v[:T, hinge_dof]
        d[g + 'root2site'] = root2site[off:off + T]
        d[g + 'joint_quat'] = rewards.joint_orientation_quat(axes[off:off + T], q[:, hinge_qadr])
        off += T
    np.savez(path, **d)
