"""Compile the fly MJCF (+ task surgery) into the flat `FlyModel` arrays the stepper reads.

This plays the role of MuJoCo's model compiler for the subset of MJCF the fly uses
(SURVEY.md App. C/D).  Output: a dict of numpy arrays (see `FIELDS` in `flymodel.py`)
that is committed as `flybody_b200/assets/fly_<variant>.npz`.

Variants
  bare   : `fruitfly.xml` as is (goldens: reference `tests/test_flybare.py:12-36`)
  walk   : `walk_imitation()` model  (reference `fly_envs.py:100-155`, `tasks/base.py:367-428`,
           `tasks/walk_imitation.py:22-85`) : walker (nq 109, nv 108, nu 59) + ghost free body
  flight : `flight_imitation()` model (reference `fly_envs.py:30-97`, `tasks/base.py:271-364`)
  ball   : `walk_on_ball()` model (reference `fly_envs.py:158-191`, `tasks/walk_on_ball.py`, `tasks/arenas/ball.py`): the BallFloor
           arena's ball (ball joint: nq 4, nv 3) first, then the walker with its thorax welded to the world
"""
import json
import os
import xml.etree.ElementTree as ET

import numpy as np

from . import meshprops
from .mjcf import (ACT_TAGS, LEG_BODY_SUBSTR, _any_in, build_fly_xml, fvec, geom_frame,
                   parse_defaults, resolved, sset)
from .quat import axisangle2q, mat2q, q2mat, qmul, qnorm, qrot

_HERE = os.path.dirname(os.path.abspath(__file__))
ASSET_OUT = os.path.join(os.path.dirname(_HERE), 'assets')
_SPAWN_POS = np.array((0, 0, 0.1278))    # reference fruitfly.py:23

# enums shared with include/flybody_b200.h
GEOM_PLANE, GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX = 0, 2, 3, 4, 5, 6
GEOM_HFIELD = 1
GEOM_TYPES = {'plane': 0, 'sphere': 2, 'capsule': 3, 'ellipsoid': 4, 'cylinder': 5, 'box': 6, 'mesh': 7}
JNT_FREE, JNT_BALL, JNT_HINGE = 0, 1, 3
TRN_JOINT, TRN_TENDON, TRN_BODY = 0, 1, 2
DYN_NONE, DYN_FILTER, DYN_FILTEREXACT = 0, 2, 3
SENS_TOUCH, SENS_ACC, SENS_VEL, SENS_GYRO, SENS_FORCE = 0, 1, 2, 3, 4
SENS_TYPES = {'touch': 0, 'accelerometer': 1, 'velocimeter': 2, 'gyro': 3, 'force': 4}
MINVAL = 1e-15


# ------------------------------------------------------------------------------------------
# primitive inertia (unit density): volume, inertia diag about centre in geom frame
# ------------------------------------------------------------------------------------------

def primitive_props(gtype, size):
    if gtype == GEOM_SPHERE:
        r = size[0]
        V = 4 / 3 * np.pi * r ** 3
        return V, np.full(3, 0.4 * V * r * r)
    if gtype == GEOM_BOX:
        a, b, c = size
        V = 8 * a * b * c
        return V, V / 3 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
    if gtype == GEOM_ELLIPSOID:
        a, b, c = size
        V = 4 / 3 * np.pi * a * b * c
        return V, V / 5 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
    if gtype == GEOM_CYLINDER:
        r, h = size[0], size[1]
        V = np.pi * r * r * 2 * h
        ix = V * (3 * r * r + (2 * h) ** 2) / 12
        return V, np.array([ix, ix, V * r * r / 2])
    if gtype == GEOM_CAPSULE:
        r, h = size[0], size[1]
        vc = np.pi * r * r * 2 * h
        vs = 4 / 3 * np.pi * r ** 3
        V = vc + vs
        iz = vc * r * r / 2 + vs * 0.4 * r * r
        ix = vc * (3 * r * r + (2 * h) ** 2) / 12 + vs * (0.4 * r * r + h * h + 0.75 * r * h)
        return V, np.array([ix, ix, iz])
    return 0.0, np.zeros(3)


def rbound(gtype, size):
    if gtype == GEOM_SPHERE:
        return size[0]
    if gtype == GEOM_CAPSULE:
        return size[0] + size[1]
    if gtype == GEOM_CYLINDER:
        return float(np.hypot(size[0], size[1]))
    if gtype == GEOM_ELLIPSOID:
        return float(np.max(size))
    if gtype == GEOM_BOX:
        return float(np.linalg.norm(size))
    return 0.0


# ------------------------------------------------------------------------------------------
# ellipsoid fluid model coefficients (MuJoCo "Fluid forces -> ellipsoid model -> added mass")
# ------------------------------------------------------------------------------------------

def added_mass_kappa(dx, dy, dz):
    """kappa_x = dx dy dz * int_0^inf dl / ((dx^2+l)^(3/2) (dy^2+l)^(1/2) (dz^2+l)^(1/2))."""
    from scipy.integrate import quad
    f = lambda l: 1.0 / np.sqrt((dx * dx + l) ** 3 * (dy * dy + l) * (dz * dz + l))
    val = quad(f, 0, np.inf, epsabs=0, epsrel=1e-10, limit=400)[0]
    return dx * dy * dz * val


def geom_fluid_coefs(size, fluidcoef):
    """geom_fluid[12] = [1, blunt, slender, angular, kutta, magnus, vmass x3, vinertia x3]
    (layout: reference `ellipsoid_fluid_model.py:229-237`)."""
    dx, dy, dz = size
    kx = added_mass_kappa(dx, dy, dz)
    ky = added_mass_kappa(dy, dz, dx)
    kz = added_mass_kappa(dz, dx, dy)
    vol = 4 / 3 * np.pi * dx * dy * dz
    vmass = vol * np.array([kx / max(MINVAL, 2 - kx), ky / max(MINVAL, 2 - ky), kz / max(MINVAL, 2 - kz)])

    def vin(a, b, ka, kb):
        # virtual inertia about the axis orthogonal to semi-axes a, b
        num = (a * a - b * b) ** 2 * abs(kb - ka)
        den = abs(2 * (a * a - b * b) + (a * a + b * b) * (ka - kb))
        return vol / 5 * num / max(MINVAL, den)

    vinertia = np.array([vin(dy, dz, ky, kz), vin(dz, dx, kz, kx), vin(dx, dy, kx, ky)])
    blunt, slender, angular, kutta, magnus = fluidcoef
    return np.hstack(([1.0, blunt, slender, angular, kutta, magnus], vmass, vinertia))


# ------------------------------------------------------------------------------------------
# tree extraction
# ------------------------------------------------------------------------------------------

class Body:
    def __init__(self, name, parent, pos, quat):
        self.name, self.parent, self.pos, self.quat = name, parent, pos, quat
        self.joints, self.geoms, self.sites = [], [], []
        self.mass, self.ipos, self.iquat, self.inertia = 0.0, np.zeros(3), np.array([1.0, 0, 0, 0]), np.zeros(3)


def _extract_bodies(fx, classes, prefix, mesh_cache, inertia_mode, bodies, parent_id, root_pos,
                    root_free, free_armature=0.0):
    """Depth-first walk of fx.worldbody; appends Body objects to `bodies`."""
    mesh_defaults = classes.get('main', {}).get('mesh', {})
    mesh_files = {}
    asset = fx.root.find('asset')
    if asset is not None:
        for m in asset.iter('mesh'):
            mesh_files[m.get('name')] = m.get('file')

    def rec(el, parent, childclass, is_root):
        cc = el.get('childclass') or childclass
        pos = fvec(el.get('pos'), 3, (0, 0, 0))
        quat = qnorm(fvec(el.get('quat'), 4, (1, 0, 0, 0)))
        if is_root:
            pos = pos + root_pos
        b = Body(prefix + el.get('name'), parent, pos, quat)
        bid = len(bodies)
        bodies.append(b)
        if is_root and root_free:
            b.joints.append(dict(name=prefix.rstrip('/') + '/' if prefix else 'free', type=JNT_FREE,
                                 axis=np.array([0.0, 0, 1]), pos=np.zeros(3), range=np.zeros(2),
                                 limited=0, stiffness=0.0, damping=0.0, armature=free_armature,
                                 springref=0.0, ref=0.0, solref=np.array([0.02, 1.0]),
                                 solimp=np.array([0.9, 0.95, 0.001, 0.5, 2.0]), margin=0.0,
                                 springdamper=np.zeros(2)))
        for ch in el:
            if ch.tag == 'freejoint':
                b.joints.append(dict(name=prefix + ch.get('name', 'free'), type=JNT_FREE,
                                     axis=np.array([0.0, 0, 1]), pos=np.zeros(3), range=np.zeros(2),
                                     limited=0, stiffness=0.0, damping=0.0, armature=0.0,
                                     springref=0.0, ref=0.0, solref=np.array([0.02, 1.0]),
                                     solimp=np.array([0.9, 0.95, 0.001, 0.5, 2.0]), margin=0.0,
                                     springdamper=np.zeros(2)))
            elif ch.tag == 'joint':
                a = resolved(ch, classes, cc)
                rng = fvec(a.get('range'), 2, (0, 0))
                lim = a.get('limited')
                has_range = a.get('range') is not None
                limited = 1 if (lim == 'true' or (lim in (None, 'auto') and has_range)) else 0
                b.joints.append(dict(
                    name=prefix + ch.get('name'), type=JNT_HINGE,
                    axis=fvec(a.get('axis'), 3, (0, 0, 1)) / np.linalg.norm(fvec(a.get('axis'), 3, (0, 0, 1))),
                    pos=fvec(a.get('pos'), 3, (0, 0, 0)), range=rng, limited=limited,
                    stiffness=float(a.get('stiffness', 0)), damping=float(a.get('damping', 0)),
                    armature=float(a.get('armature', 0)), springref=float(a.get('springref', 0)),
                    ref=float(a.get('ref', 0)),
                    solref=fvec(a.get('solreflimit'), 2, (0.02, 1.0)),
                    solimp=fvec(a.get('solimplimit'), 5, (0.9, 0.95, 0.001, 0.5, 2.0)),
                    margin=float(a.get('margin', 0)),
                    springdamper=fvec(a.get('springdamper'), 2, (0, 0))))
            elif ch.tag == 'geom':
                a = resolved(ch, classes, cc)
                gtype = GEOM_TYPES[a.get('type', 'sphere')]
                gpos, gquat, gsize = geom_frame(a)
                g = dict(name=prefix + (ch.get('name') or ''), type=gtype, pos=gpos, quat=gquat, size=gsize,
                         contype=int(a.get('contype', 1)), conaffinity=int(a.get('conaffinity', 1)),
                         condim=int(a.get('condim', 3)), priority=int(a.get('priority', 0)),
                         friction=fvec(a.get('friction'), 3, (1.0, 0.005, 0.0001)),
                         solmix=float(a.get('solmix', 1.0)),
                         solref=fvec(a.get('solref'), 2, (0.02, 1.0)),
                         solimp=fvec(a.get('solimp'), 5, (0.9, 0.95, 0.001, 0.5, 2.0)),
                         margin=float(a.get('margin', 0)), gap=float(a.get('gap', 0)),
                         fluidshape=a.get('fluidshape', 'none'),
                         fluidcoef=fvec(a.get('fluidcoef'), 5, (0.5, 0.25, 1.5, 1.0, 1.0)),
                         mass=0.0, com=gpos.copy(), inertia=np.zeros((3, 3)))
                density = float(a.get('density', 1000.0))
                mass_attr = a.get('mass')
                if gtype == GEOM_TYPES['mesh']:
                    mp = mesh_cache[a['mesh']][inertia_mode]
                    V, c, I = mp['volume'], np.array(mp['com']), np.array(mp['inertia'])
                    R = q2mat(gquat)
                    mass = float(mass_attr) if mass_attr is not None else density * V
                    sc = mass / V
                    g['mass'] = mass
                    g['com'] = gpos + R @ c
                    g['inertia'] = sc * (R @ I @ R.T)
                else:
                    V, Id = primitive_props(gtype, gsize)
                    mass = float(mass_attr) if mass_attr is not None else density * V
                    if V > 0 and mass > 0:
                        R = q2mat(gquat)
                        g['mass'] = mass
                        g['inertia'] = (mass / V) * (R @ np.diag(Id) @ R.T)
                b.geoms.append(g)
            elif ch.tag == 'site':
                a = resolved(ch, classes, cc)
                spos, squat, ssize = geom_frame(a)
                stype = GEOM_TYPES[a.get('type', 'sphere')]
                b.sites.append(dict(name=prefix + ch.get('name'), pos=spos, quat=squat, size=ssize, type=stype))
        for ch in el:
            if ch.tag == 'body':
                rec(ch, bid, cc, False)
        return bid

    roots = []
    for el in fx.worldbody:
        if el.tag == 'body':
            roots.append(rec(el, parent_id, None, True))
    return roots


def _body_inertial(b):
    """Compose geom masses into body mass / ipos / iquat / principal inertia."""
    M = sum(g['mass'] for g in b.geoms)
    b.mass = M
    if M <= 0:
        b.ipos, b.iquat, b.inertia = np.zeros(3), np.array([1.0, 0, 0, 0]), np.zeros(3)
        return
    com = sum(g['mass'] * g['com'] for g in b.geoms) / M
    I = np.zeros((3, 3))
    for g in b.geoms:
        if g['mass'] <= 0:
            continue
        d = g['com'] - com
        I += g['inertia'] + g['mass'] * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
    w, V = np.linalg.eigh(0.5 * (I + I.T))
    order = np.argsort(-w)
    w, V = w[order], V[:, order]
    if np.linalg.det(V) < 0:
        V[:, 2] *= -1
    b.ipos, b.iquat, b.inertia = com, mat2q(V), w


def _fuse_subtree(bodies, root):
    """Fuse all bodies of a joint-less subtree (ghost) into bodies[root]; returns kept body."""
    # world placement relative to root frame
    n = len(bodies)
    rel_pos = {root: np.zeros(3)}
    rel_quat = {root: np.array([1.0, 0, 0, 0])}
    members = [root]
    for i in range(root + 1, n):
        p = bodies[i].parent
        if p in rel_pos:
            rel_pos[i] = rel_pos[p] + qrot(rel_quat[p], bodies[i].pos)
            rel_quat[i] = qmul(rel_quat[p], bodies[i].quat)
            members.append(i)
    rb = bodies[root]
    for i in members[1:]:
        R = q2mat(rel_quat[i])
        for g in bodies[i].geoms:
            g2 = dict(g)
            g2['com'] = rel_pos[i] + R @ g['com']
            g2['pos'] = rel_pos[i] + R @ g['pos']
            g2['quat'] = qmul(rel_quat[i], g['quat'])
            g2['inertia'] = R @ g['inertia'] @ R.T
            rb.geoms.append(g2)
        for s in bodies[i].sites:
            s2 = dict(s)
            s2['pos'] = rel_pos[i] + R @ s['pos']
            s2['quat'] = qmul(rel_quat[i], s['quat'])
            rb.sites.append(s2)
    for i in sorted(members[1:], reverse=True):
        del bodies[i]
    return rb


# ------------------------------------------------------------------------------------------
# main entry
# ------------------------------------------------------------------------------------------

def _reference_assets(assets_dir):
    """`assets_dir`, else the directory flymodel.reference_assets_dir() finds the reference's fruitfly.xml in"""
    if assets_dir:
        return assets_dir
    from ..flymodel import reference_assets_dir
    found = reference_assets_dir()
    if found is None:
        raise FileNotFoundError("the reference's fruitfly.xml was not found: install flybody or set FLYBODY_ASSETS to its fruitfly/assets directory")
    return found


def load_mesh_cache(assets_dir=None, rebuild=False):
    path = os.path.join(ASSET_OUT, 'mesh_props.json')
    if os.path.exists(path) and not rebuild:
        with open(path) as f:
            return json.load(f)
    assets_dir = _reference_assets(assets_dir)
    root = ET.parse(os.path.join(assets_dir, 'fruitfly.xml')).getroot()
    scale = fvec(root.find('default').find('mesh').get('scale'))
    files = {m.get('name'): m.get('file') for m in root.find('asset').iter('mesh')}
    os.makedirs(ASSET_OUT, exist_ok=True)
    return meshprops.build_cache(assets_dir, files, scale, path)


def compile_variant(variant='walk', assets_dir=None, inertia_mode='legacy2', mesh_cache=None,
                    joint_filter=None, claw_friction=1.0, terminal=None, force_actuators=False, use_wings=None, use_legs=None,
                    use_mouth=False, use_antennae=False, adhesion_filter=0.007, dyntype_filterexact=False):
    """`variant` picks the task's model surgery (reference tasks/base.py `Walking` / `Flying`); `force_actuators`, `use_wings`,
    `use_legs` and `joint_filter` are the `FruitFly` constructor switches the env factories expose (reference fly_envs.py:100-246:
    force_actuators, disable_wings, disable_legs, joint_filter); None keeps the task's default."""
    assets_dir = _reference_assets(assets_dir)
    xml_path = os.path.join(assets_dir, 'fruitfly.xml')
    mesh_cache = mesh_cache or load_mesh_cache(assets_dir)

    floor = None
    hfield = None
    ghost = False
    if variant == 'bare':
        fx = _bare_xml(xml_path)
        timestep = float(fx.root.find('option').get('timestep'))
        spawn = np.zeros(3)
        prefix = ''
    elif variant == 'walker':
        # the `FruitFly` entity on its own, as the reference's tests/test_flywalker.py builds it (`mjcf.Physics.from_mjcf_model(
        # fly.mjcf_model)`): the walker's MJCF surgery, no task, no arena, no ghost; the free joint is removed (fruitfly.py:187),
        # so the thorax is welded to the world
        fx = build_fly_xml(xml_path, name='walker', use_legs=True if use_legs is None else use_legs,
                           use_wings=True if use_wings is None else use_wings, use_mouth=use_mouth, use_antennae=use_antennae,
                           joint_filter=0.01 if joint_filter is None else joint_filter, adhesion_filter=adhesion_filter,
                           force_actuators=force_actuators, dyntype_filterexact=dyntype_filterexact)
        timestep = float(fx.root.find('option').get('timestep'))
        spawn, prefix = np.zeros(3), ''
    elif variant == 'ball':
        # walk_on_ball (reference fly_envs.py:158-191, tasks/walk_on_ball.py:18-43): the Walking surgery without the ghost, the walker's
        # free joint removed (its thorax welded to the world at the spawn pose), one exclude between the thorax and each of its child
        # bodies, and the BallFloor arena (tasks/arenas/ball.py) instead of the floor plane
        fx = build_fly_xml(xml_path, name='walker', use_legs=True if use_legs is None else use_legs,
                           use_wings=False if use_wings is None else use_wings, use_mouth=False, use_antennae=False,
                           joint_filter=0.01 if joint_filter is None else joint_filter, adhesion_filter=adhesion_filter,
                           force_actuators=force_actuators, dyntype_filterexact=dyntype_filterexact)
        timestep = 2e-4                                  # reference tasks/constants.py:11
        spawn, prefix = _SPAWN_POS, 'walker/'
        _add_wing_leg_excludes(fx)                        # base.py:404-411
        _add_thorax_excludes(fx)                          # walk_on_ball.py:30-38
        if claw_friction is not None:                     # walk_on_ball.py:40-44
            fx.class_child('adhesion-collision', 'geom').set('friction', repr(float(claw_friction)))
    elif variant in ('walk', 'template'):
        # template: template_task (reference fly_envs.py:249-300, tasks/template_task.py:35-43), the same Walking surgery
        # without the ghost (add_ghost=False), with the factory's adhesion filter
        jf = 0.01 if joint_filter is None else joint_filter
        fx = build_fly_xml(xml_path, name='walker', use_legs=True if use_legs is None else use_legs,
                           use_wings=False if use_wings is None else use_wings, use_mouth=False,
                           use_antennae=False, joint_filter=jf, adhesion_filter=adhesion_filter, force_actuators=force_actuators,
                           dyntype_filterexact=dyntype_filterexact)
        timestep = 2e-4                                  # reference tasks/constants.py:11
        spawn, prefix, ghost = _SPAWN_POS, 'walker/', variant == 'walk'
        # Walking.__init__: floor params (base.py:398-401)
        floor = dict(friction=np.array([0.5, 0.005, 0.0001]), solref=np.array([0.001, 1.0]),
                     solimp=np.array([0.95, 0.99, 0.01, 0.5, 2.0]), contype=1, conaffinity=1)
        _add_wing_leg_excludes(fx)                        # base.py:404-411
        if claw_friction is not None:                     # walk_imitation.py:70-73
            fx.class_child('adhesion-collision', 'geom').set('friction', repr(float(claw_friction)))
    elif variant == 'flight':
        jf = 0.0 if joint_filter is None else joint_filter
        fx = build_fly_xml(xml_path, name='walker', use_legs=False if use_legs is None else use_legs,
                           use_wings=True if use_wings is None else use_wings, use_mouth=False,
                           use_antennae=False, joint_filter=jf, adhesion_filter=0.007, force_actuators=force_actuators,
                           dyntype_filterexact=dyntype_filterexact, body_pitch_angle=47.5, stroke_plane_angle=0.0)
        timestep = 5e-5                                  # reference tasks/constants.py:17
        spawn, prefix, ghost = _SPAWN_POS, 'walker/', True
        # Flying.__init__ (base.py:308-346): floor contacts off, wing gains, fluid model, wing joint params
        floor = dict(friction=np.array([1.0, 0.005, 0.0001]), solref=np.array([0.02, 1.0]),
                     solimp=np.array([0.9, 0.95, 0.001, 0.5, 2.0]), contype=0, conaffinity=0)
        for i, dc in enumerate(['yaw', 'roll', 'pitch']):
            fx.class_child(dc, 'general').set('gainprm', repr(float([18, 18, 18][i])))
        for g in fx.all('geom'):
            if 'fluid' in (g.get('name') or ''):
                g.set('fluidshape', 'ellipsoid')
                sset(g, 'fluidcoef', [1.0, 0.5, 1.5, 1.7, 1.0])
        wj = fx.class_child('wing', 'joint')
        wj.set('stiffness', repr(0.01))
        wj.set('damping', repr(0.007769230))
        _add_wing_leg_excludes(fx)
    elif variant == 'vision':
        # vision_guided_flight (reference fly_envs.py:194-246, tasks/vision_flight.py:20-79): the flight model without a ghost,
        # ground contacts ON (floor_contacts=True -> the arena's geoms keep MuJoCo's defaults), and the arena of
        # tasks/arenas/hills.py:143-251 ('outdoor_natural'): heightfield `terrain` at z = -0.01 over [-20, 20]^2, 401 x 401
        # points, elevation scale 1, base 0.05, next to the ground plane at z = 0
        fx = build_fly_xml(xml_path, name='walker', use_legs=False if use_legs is None else use_legs,
                           use_wings=True if use_wings is None else use_wings, use_mouth=False,
                           use_antennae=False, joint_filter=0.0 if joint_filter is None else joint_filter, adhesion_filter=0.007,
                           force_actuators=force_actuators, body_pitch_angle=47.5, stroke_plane_angle=0.0)
        timestep = 5e-5
        spawn, prefix, ghost = _SPAWN_POS, 'walker/', False
        floor = dict(friction=np.array([1.0, 0.005, 0.0001]), solref=np.array([0.02, 1.0]),
                     solimp=np.array([0.9, 0.95, 0.001, 0.5, 2.0]), contype=1, conaffinity=1)
        hfield = dict(size=np.array([20.0, 20.0, 1.0, 0.05]), nrow=401, ncol=401, pos=np.array([0.0, 0.0, -0.01]))
        for i, dc in enumerate(['yaw', 'roll', 'pitch']):
            fx.class_child(dc, 'general').set('gainprm', repr(float([18, 18, 18][i])))
        for g in fx.all('geom'):
            if 'fluid' in (g.get('name') or ''):
                g.set('fluidshape', 'ellipsoid')
                sset(g, 'fluidcoef', [1.0, 0.5, 1.5, 1.7, 1.0])
        wj = fx.class_child('wing', 'joint')
        wj.set('stiffness', repr(0.01))
        wj.set('damping', repr(0.007769230))
        _add_wing_leg_excludes(fx)
    else:
        raise ValueError(variant)

    classes = parse_defaults(fx.root)
    bodies = [Body('world', -1, np.zeros(3), np.array([1.0, 0, 0, 0]))]
    if variant == 'ball':             # the arena is built before the walker is attached: its body, joint, qpos and dofs come first
        bodies.append(_ball_body())
    _extract_bodies(fx, classes, prefix, mesh_cache, inertia_mode, bodies, 0, spawn,
                    root_free=(variant not in ('bare', 'walker', 'ball')))
    n_walker_bodies = len(bodies)

    # excludes -> body-name pairs
    excludes = set()
    for e in fx.all('exclude'):
        excludes.add(frozenset((prefix + e.get('body1'), prefix + e.get('body2'))))

    ghost_body = None
    if ghost:
        # ghost = FruitFly(name='ghost', use_wings=False, use_legs=False) + make_ghost_fly
        # (base.py:142-154, task_utils.py:124-160): no joints, wings removed, only mesh geoms,
        # contacts off; one free joint with armature 1.  Fused here into one rigid body.
        gx = build_fly_xml(xml_path, name='ghost', use_legs=False, use_wings=False)
        for j in gx.all('joint'):
            gx.remove(j)
        for b in gx.all('body'):
            if b.get('name', '').startswith('wing'):
                gx.remove(b)
        gcls = parse_defaults(gx.root)
        g0 = len(bodies)
        _extract_bodies(gx, gcls, 'ghost/', mesh_cache, inertia_mode, bodies, 0, spawn, root_free=True,
                        free_armature=1.0)
        ghost_body = _fuse_subtree(bodies, g0)
        ghost_body.geoms = [g for g in ghost_body.geoms if g['type'] == GEOM_TYPES['mesh']]
        for g in ghost_body.geoms:
            g['contype'] = g['conaffinity'] = 0
        ghost_body.sites = [s for s in ghost_body.sites if s['name'] in ('ghost/thorax',)]

    for b in bodies[1:]:
        _body_inertial(b)

    actuators = fx.all('actuator')
    tendons = fx.all('tendon')
    sensors = fx.all('sensor')
    model = _flatten(bodies, classes, fx, prefix, actuators, tendons, sensors, excludes, floor, timestep,
                     variant, hfield=hfield)
    model['ctrl_indices'] = {k: v for k, v in fx.ctrl_indices.items()}
    model['observable_joints'] = [prefix + n for n in fx.observable_joints]
    return model


def _bare_xml(xml_path):
    from .mjcf import FlyXML
    fx = FlyXML(xml_path)
    fx.name = ''
    fx.ctrl_indices = {}
    fx.observable_joints = [j.get('name') for j in fx.all('joint') if j.tag == 'joint']
    return fx


def _ball_body(pos=(-0.05, 0, -0.419), radius=0.454, density=0.0025):
    """BallFloor's ball as walk_on_ball builds it (reference fly_envs.py:174-177, tasks/arenas/ball.py:60-67): a sphere on a ball
    joint, with Walking's ground-geom contact parameters (base.py:398-401)"""
    b = Body('ball', 0, np.array(pos, float), np.array([1.0, 0, 0, 0]))
    b.joints.append(dict(name='ball', type=JNT_BALL, axis=np.array([0.0, 0, 1]), pos=np.zeros(3), range=np.zeros(2), limited=0,
                         stiffness=0.0, damping=0.0, armature=0.0, springref=0.0, ref=0.0, solref=np.array([0.02, 1.0]),
                         solimp=np.array([0.9, 0.95, 0.001, 0.5, 2.0]), margin=0.0, springdamper=np.zeros(2)))
    size = np.array([radius, 0.0, 0.0])
    V, Id = primitive_props(GEOM_SPHERE, size)
    b.geoms.append(dict(name='', type=GEOM_SPHERE, pos=np.zeros(3), quat=np.array([1.0, 0, 0, 0]), size=size, contype=1,
                        conaffinity=1, condim=3, priority=0, friction=np.array([0.5, 0.005, 0.0001]), solmix=1.0,
                        solref=np.array([0.001, 1.0]), solimp=np.array([0.95, 0.99, 0.01, 0.5, 2.0]), margin=0.0, gap=0.0,
                        fluidshape='none', fluidcoef=np.array([0.5, 0.25, 1.5, 1.0, 1.0]), mass=density * V, com=np.zeros(3),
                        inertia=density * np.diag(Id)))
    return b


def _add_thorax_excludes(fx):
    contact = fx.root.find('contact')
    thorax = next(b for b in fx.all('body') if b.get('name') == 'thorax')
    for child in thorax:
        if child.tag == 'body':
            ET.SubElement(contact, 'exclude', name=f"thorax_{child.get('name')}", body1='thorax', body2=child.get('name'))
    fx._reindex()


def _add_wing_leg_excludes(fx):
    contact = fx.root.find('contact')
    for body in fx.all('body'):
        if _any_in(LEG_BODY_SUBSTR, body.get('name')):
            for wing in ('wing_left', 'wing_right'):
                ET.SubElement(contact, 'exclude', name=f"{body.get('name')}_{wing}",
                              body1=body.get('name'), body2=wing)
    fx._reindex()


def _flatten(bodies, classes, fx, prefix, actuators, tendons, sensors, excludes, floor, timestep, variant, hfield=None):
    opt = fx.root.find('option')
    m = {}
    nbody = len(bodies)
    # ---- bodies / joints / dofs
    body_parent = np.array([b.parent for b in bodies], dtype=np.int32)
    body_parent[0] = 0
    jnt, qpos0, qspring = [], [], []
    body_jntadr = np.full(nbody, -1, np.int32)
    body_jntnum = np.zeros(nbody, np.int32)
    body_dofadr = np.full(nbody, -1, np.int32)
    body_dofnum = np.zeros(nbody, np.int32)
    jnt_qposadr, jnt_dofadr, jnt_bodyid = [], [], []
    dof_bodyid, dof_jntid, dof_armature, dof_damping = [], [], [], []
    nq = nv = 0
    for bi, b in enumerate(bodies):
        if b.joints:
            body_jntadr[bi] = len(jnt)
            body_jntnum[bi] = len(b.joints)
            body_dofadr[bi] = nv
        for j in b.joints:
            jid = len(jnt)
            jnt.append(j)
            jnt_qposadr.append(nq)
            jnt_dofadr.append(nv)
            jnt_bodyid.append(bi)
            if j['type'] == JNT_FREE:
                qpos0 += list(b.pos) + list(b.quat)
                qspring += list(b.pos) + list(b.quat)
                nq += 7
                nd = 6
            elif j['type'] == JNT_BALL:
                qpos0 += [1.0, 0.0, 0.0, 0.0]
                qspring += [1.0, 0.0, 0.0, 0.0]
                nq += 4
                nd = 3
            else:
                qpos0.append(j['ref'])
                qspring.append(j['springref'])
                nq += 1
                nd = 1
            for _ in range(nd):
                dof_bodyid.append(bi)
                dof_jntid.append(jid)
                dof_armature.append(j['armature'])
                dof_damping.append(j['damping'])
            nv += nd
        body_dofnum[bi] = nv - body_dofadr[bi] if b.joints else 0
    njnt = len(jnt)
    dof_bodyid = np.array(dof_bodyid, np.int32)
    # last dof on or above each body
    body_lastdof = np.full(nbody, -1, np.int32)
    for bi in range(1, nbody):
        if body_dofnum[bi] > 0:
            body_lastdof[bi] = body_dofadr[bi] + body_dofnum[bi] - 1
        else:
            body_lastdof[bi] = body_lastdof[body_parent[bi]]
    dof_parent = np.full(nv, -1, np.int32)
    for d in range(nv):
        bi = dof_bodyid[d]
        if d > body_dofadr[bi]:
            dof_parent[d] = d - 1
        else:
            dof_parent[d] = body_lastdof[body_parent[bi]]
    dof_Madr = np.zeros(nv, np.int32)
    nM = 0
    for d in range(nv):
        dof_Madr[d] = nM
        k = d
        while k >= 0:
            nM += 1
            k = dof_parent[k]
    body_weld = np.zeros(nbody, np.int32)
    body_root = np.zeros(nbody, np.int32)
    for bi in range(1, nbody):
        body_weld[bi] = bi if body_jntnum[bi] > 0 else body_weld[body_parent[bi]]
        body_root[bi] = bi if body_parent[bi] == 0 else body_root[body_parent[bi]]

    m.update(nq=nq, nv=nv, nbody=nbody, njnt=njnt, nM=nM)
    m['body_parentid'] = body_parent
    m['body_rootid'] = body_root
    m['body_weldid'] = body_weld
    m['body_jntadr'], m['body_jntnum'] = body_jntadr, body_jntnum
    m['body_dofadr'], m['body_dofnum'] = body_dofadr, body_dofnum
    m['body_lastdof'] = body_lastdof
    m['body_pos'] = np.array([b.pos for b in bodies])
    m['body_quat'] = np.array([b.quat for b in bodies])
    m['body_ipos'] = np.array([b.ipos for b in bodies])
    m['body_iquat'] = np.array([b.iquat for b in bodies])
    m['body_mass'] = np.array([b.mass for b in bodies])
    m['body_inertia'] = np.array([b.inertia for b in bodies])
    sub = m['body_mass'].copy()
    for bi in range(nbody - 1, 0, -1):
        sub[body_parent[bi]] += sub[bi]
    m['body_subtreemass'] = sub
    m['jnt_type'] = np.array([j['type'] for j in jnt], np.int32)
    m['jnt_qposadr'] = np.array(jnt_qposadr, np.int32)
    m['jnt_dofadr'] = np.array(jnt_dofadr, np.int32)
    m['jnt_bodyid'] = np.array(jnt_bodyid, np.int32)
    m['jnt_pos'] = np.array([j['pos'] for j in jnt])
    m['jnt_axis'] = np.array([j['axis'] for j in jnt])
    m['jnt_stiffness'] = np.array([j['stiffness'] for j in jnt])
    m['jnt_range'] = np.array([j['range'] for j in jnt])
    m['jnt_limited'] = np.array([j['limited'] for j in jnt], np.int32)
    m['jnt_solref'] = np.array([j['solref'] for j in jnt])
    m['jnt_solimp'] = np.array([j['solimp'] for j in jnt])
    m['jnt_margin'] = np.array([j['margin'] for j in jnt])
    m['_jnt_springdamper'] = [j['springdamper'] for j in jnt]
    m['qpos0'] = np.array(qpos0)
    m['qpos_spring'] = np.array(qspring)
    m['dof_bodyid'] = dof_bodyid
    m['dof_jntid'] = np.array(dof_jntid, np.int32)
    m['dof_parentid'] = dof_parent
    m['dof_Madr'] = dof_Madr
    m['dof_armature'] = np.array(dof_armature)
    m['dof_damping'] = np.array(dof_damping)
    m['body_names'] = [b.name for b in bodies]
    m['jnt_names'] = [j['name'] for j in jnt]

    # ---- geoms: only collision geoms (+ floor) go to the stepper; fluid geoms separately
    geoms, fluid_geoms, ngeom_all = [], [], 0
    if floor is not None:
        geoms.append(dict(name='floor', type=GEOM_PLANE, body=0, pos=np.zeros(3), quat=np.array([1.0, 0, 0, 0]),
                          size=np.array([8.0, 8.0, 0.25]), contype=floor['contype'], conaffinity=floor['conaffinity'],
                          condim=3, priority=0, friction=floor['friction'], solmix=1.0, solref=floor['solref'],
                          solimp=floor['solimp'], margin=0.0, gap=0.0))
        ngeom_all += 1
    if hfield is not None:
        # the terrain: a world geom of MuJoCo type hfield (1).  It sits in the geom arrays for the contact parameters; its pairs
        # are kept out of the generic pair list (hf_pair_geom below) because the heightfield narrowphase is its own kernel
        geoms.append(dict(name='terrain', type=GEOM_HFIELD, body=0, pos=hfield['pos'], quat=np.array([1.0, 0, 0, 0]),
                          size=hfield['size'][:3], contype=floor['contype'], conaffinity=floor['conaffinity'],
                          condim=3, priority=0, friction=floor['friction'], solmix=1.0, solref=floor['solref'],
                          solimp=floor['solimp'], margin=0.0, gap=0.0))
        ngeom_all += 1
    for bi, b in enumerate(bodies):
        for g in b.geoms:
            ngeom_all += 1
            if g['type'] == GEOM_TYPES['mesh']:
                continue
            if g.get('fluidshape') == 'ellipsoid':
                fluid_geoms.append(dict(g, body=bi))
            if g['contype'] or g['conaffinity']:
                geoms.append(dict(g, body=bi))
    ngeom = len(geoms)
    m['ngeom'] = ngeom
    m['ngeom_all'] = ngeom_all
    m['geom_type'] = np.array([g['type'] for g in geoms], np.int32)
    m['geom_bodyid'] = np.array([g['body'] for g in geoms], np.int32)
    m['geom_size'] = np.array([g['size'] for g in geoms]).reshape(ngeom, 3)
    m['geom_pos'] = np.array([g['pos'] for g in geoms]).reshape(ngeom, 3)
    m['geom_quat'] = np.array([g['quat'] for g in geoms]).reshape(ngeom, 4)
    m['geom_rbound'] = np.array([rbound(g['type'], g['size']) for g in geoms])
    m['geom_condim'] = np.array([g['condim'] for g in geoms], np.int32)
    m['geom_priority'] = np.array([g['priority'] for g in geoms], np.int32)
    m['geom_friction'] = np.array([g['friction'] for g in geoms]).reshape(ngeom, 3)
    m['geom_solmix'] = np.array([g['solmix'] for g in geoms])
    m['geom_solref'] = np.array([g['solref'] for g in geoms]).reshape(ngeom, 2)
    m['geom_solimp'] = np.array([g['solimp'] for g in geoms]).reshape(ngeom, 5)
    m['geom_margin'] = np.array([g['margin'] for g in geoms])
    m['geom_gap'] = np.array([g['gap'] for g in geoms])
    m['geom_names'] = [g['name'] for g in geoms]
    nfl = len(fluid_geoms)
    m['nfluid'] = nfl
    m['fluid_bodyid'] = np.array([g['body'] for g in fluid_geoms], np.int32)
    m['fluid_pos'] = np.array([g['pos'] for g in fluid_geoms]).reshape(nfl, 3)
    m['fluid_quat'] = np.array([g['quat'] for g in fluid_geoms]).reshape(nfl, 4)
    m['fluid_size'] = np.array([g['size'] for g in fluid_geoms]).reshape(nfl, 3)
    m['fluid_coef'] = np.array([geom_fluid_coefs(g['size'], g['fluidcoef']) for g in fluid_geoms]).reshape(nfl, 12)
    # bodies that use the ellipsoid model skip the inertia-box model (engine_passive.c)
    body_fluid_ell = np.zeros(nbody, np.int32)
    for g in fluid_geoms:
        body_fluid_ell[g['body']] = 1
    m['body_fluid_ellipsoid'] = body_fluid_ell

    # ---- collision pair list (filters: SURVEY.md App. A.7)
    pairs, hf_pairs = [], []
    for a in range(ngeom):
        for b_ in range(a + 1, ngeom):
            ga, gb = geoms[a], geoms[b_]
            if not ((ga['contype'] & gb['conaffinity']) or (gb['contype'] & ga['conaffinity'])):
                continue
            if GEOM_HFIELD in (ga['type'], gb['type']):
                if ga['body'] != gb['body'] and GEOM_PLANE not in (ga['type'], gb['type']):
                    hf_pairs.append(b_ if ga['type'] == GEOM_HFIELD else a)
                continue
            b1, b2 = ga['body'], gb['body']
            if b1 == b2:
                continue
            w1, w2 = body_weld[b1], body_weld[b2]
            if w1 == w2:
                continue
            wp1, wp2 = body_weld[body_parent[w1]], body_weld[body_parent[w2]]
            if w1 != 0 and w2 != 0 and (w1 == wp2 or w2 == wp1):
                continue
            if frozenset((bodies[b1].name, bodies[b2].name)) in excludes:
                continue
            # order so that type1 <= type2 (collision function table is upper-triangular)
            if ga['type'] > gb['type']:
                pairs.append((b_, a))
            else:
                pairs.append((a, b_))
    m['npair'] = len(pairs)
    if hfield is not None:
        m['hf_geom'] = [g['type'] for g in geoms].index(GEOM_HFIELD)
        m['hf_pair_geom'] = np.array(hf_pairs, np.int32)
        m['hf_size'] = np.asarray(hfield['size'], np.float64)
        m['hf_nrow'], m['hf_ncol'] = int(hfield['nrow']), int(hfield['ncol'])
    m['pair_geom1'] = np.array([p[0] for p in pairs], np.int32)
    m['pair_geom2'] = np.array([p[1] for p in pairs], np.int32)

    # ---- sites
    sites = []
    for bi, b in enumerate(bodies):
        for s in b.sites:
            sites.append(dict(s, body=bi))
    ns = len(sites)
    m['nsite'] = ns
    m['site_bodyid'] = np.array([s['body'] for s in sites], np.int32)
    m['site_pos'] = np.array([s['pos'] for s in sites]).reshape(ns, 3)
    m['site_quat'] = np.array([s['quat'] for s in sites]).reshape(ns, 4)
    m['site_type'] = np.array([s['type'] for s in sites], np.int32)
    m['site_size'] = np.array([s['size'] for s in sites]).reshape(ns, 3)
    m['site_names'] = [s['name'] for s in sites]

    # ---- tendons (fixed)
    jname2id = {n: i for i, n in enumerate(m['jnt_names'])}
    t_adr, t_num, w_dof, w_coef, t_names = [], [], [], [], []
    for t in tendons:
        t_adr.append(len(w_dof))
        terms = [c for c in t if c.tag == 'joint']
        t_num.append(len(terms))
        for c in terms:
            jid = jname2id[prefix + c.get('joint')]
            w_dof.append(m['jnt_dofadr'][jid])
            w_coef.append(float(c.get('coef', 1)))
        t_names.append(prefix + t.get('name'))
    m['ntendon'] = len(tendons)
    m['nwrap'] = len(w_dof)
    m['tendon_adr'] = np.array(t_adr, np.int32)
    m['tendon_num'] = np.array(t_num, np.int32)
    m['wrap_dofid'] = np.array(w_dof, np.int32)
    m['wrap_qposadr'] = np.array([m['jnt_qposadr'][m['dof_jntid'][d]] for d in w_dof], np.int32)
    m['wrap_coef'] = np.array(w_coef)
    m['tendon_names'] = t_names

    # ---- actuators
    tname2id = {n: i for i, n in enumerate(t_names)}
    bname2id = {n: i for i, n in enumerate(m['body_names'])}
    nu = len(actuators)
    A = dict(trntype=[], trnid=[], dyntype=[], dynprm=[], gainprm=[], biasprm=[], biastype=[], ctrllimited=[],
             ctrlrange=[], forcelimited=[], forcerange=[], actadr=[], names=[])
    na = 0
    for a_el in actuators:
        a = resolved(a_el, classes, None)
        if a_el.tag == 'adhesion':
            trntype, trnid = TRN_BODY, bname2id[prefix + a['body']]
            biastype = 0
        elif a.get('joint') is not None:
            trntype, trnid = TRN_JOINT, jname2id[prefix + a['joint']]
            biastype = {'none': 0, 'affine': 1}[a.get('biastype', 'none')]
        else:
            trntype, trnid = TRN_TENDON, tname2id[prefix + a['tendon']]
            biastype = {'none': 0, 'affine': 1}[a.get('biastype', 'none')]
        dyn = {'none': DYN_NONE, 'filter': DYN_FILTER, 'filterexact': DYN_FILTEREXACT}[a.get('dyntype', 'none')]
        A['trntype'].append(trntype)
        A['trnid'].append(trnid)
        A['dyntype'].append(dyn)
        A['dynprm'].append(fvec(a.get('dynprm'), 3, (1, 0, 0)))
        A['gainprm'].append(fvec(a.get('gainprm'), 3, (1, 0, 0)))
        A['biasprm'].append(fvec(a.get('biasprm'), 3, (0, 0, 0)) if biastype else np.zeros(3))
        A['biastype'].append(biastype)
        cr = a.get('ctrlrange')
        cl = a.get('ctrllimited')
        A['ctrllimited'].append(1 if (cl == 'true' or (cl in (None, 'auto') and cr is not None)) else 0)
        A['ctrlrange'].append(fvec(cr, 2, (0, 0)))
        fr = a.get('forcerange')
        fl = a.get('forcelimited')
        A['forcelimited'].append(1 if (fl == 'true' or (fl in (None, 'auto') and fr is not None)) else 0)
        A['forcerange'].append(fvec(fr, 2, (0, 0)))
        if dyn != DYN_NONE:
            A['actadr'].append(na)
            na += 1
        else:
            A['actadr'].append(-1)
        A['names'].append(prefix + a_el.get('name'))
    m['nu'], m['na'] = nu, na
    m['actuator_trntype'] = np.array(A['trntype'], np.int32)
    m['actuator_trnid'] = np.array(A['trnid'], np.int32)
    m['actuator_dyntype'] = np.array(A['dyntype'], np.int32)
    m['actuator_dynprm'] = np.array(A['dynprm']).reshape(nu, 3)
    m['actuator_gainprm'] = np.array(A['gainprm']).reshape(nu, 3)
    m['actuator_biasprm'] = np.array(A['biasprm']).reshape(nu, 3)
    m['actuator_biastype'] = np.array(A['biastype'], np.int32)
    m['actuator_ctrllimited'] = np.array(A['ctrllimited'], np.int32)
    m['actuator_ctrlrange'] = np.array(A['ctrlrange']).reshape(nu, 2)
    m['actuator_forcelimited'] = np.array(A['forcelimited'], np.int32)
    m['actuator_forcerange'] = np.array(A['forcerange']).reshape(nu, 2)
    m['actuator_actadr'] = np.array(A['actadr'], np.int32)
    m['actuator_names'] = A['names']

    # ---- sensors
    sname2id = {n: i for i, n in enumerate(m['site_names'])}
    s_type, s_obj, s_adr, s_dim, s_names = [], [], [], [], []
    nsd = 0
    for s in sensors:
        tp = SENS_TYPES[s.tag]
        dim = 1 if tp == SENS_TOUCH else 3
        s_type.append(tp)
        s_obj.append(sname2id[prefix + s.get('site')])
        s_adr.append(nsd)
        s_dim.append(dim)
        s_names.append(prefix + s.get('name'))
        nsd += dim
    m['nsensor'], m['nsensordata'] = len(sensors), nsd
    m['sensor_type'] = np.array(s_type, np.int32)
    m['sensor_objid'] = np.array(s_obj, np.int32)
    m['sensor_adr'] = np.array(s_adr, np.int32)
    m['sensor_dim'] = np.array(s_dim, np.int32)
    m['sensor_names'] = s_names

    # ---- options
    m['opt_timestep'] = float(timestep)
    m['opt_gravity'] = fvec(opt.get('gravity'), 3, (0, 0, -9.81))
    m['opt_density'] = float(opt.get('density', 0))
    m['opt_viscosity'] = float(opt.get('viscosity', 0))
    m['opt_wind'] = np.zeros(3)
    m['opt_impratio'] = 1.0
    m['opt_tolerance'] = 1e-8
    m['opt_iterations'] = 100
    m['opt_ls_iterations'] = 50
    m['opt_ls_tolerance'] = 0.01
    m['opt_noslip_iterations'] = int(opt.get('noslip_iterations', 0))
    m['opt_noslip_tolerance'] = 1e-6
    m['opt_cone_elliptic'] = 1 if opt.get('cone', 'pyramidal') == 'elliptic' else 0

    _set0(m)
    return m


# ------------------------------------------------------------------------------------------
# quantities evaluated at qpos0 (MuJoCo `mj_setConst`): invweight0, meaninertia, springdamper
# ------------------------------------------------------------------------------------------

def kinematics0(m, qpos=None):
    """Body world frames at qpos (default qpos0).  Returns xpos, xquat, anchors, axes (per dof)."""
    nbody, nv = m['nbody'], m['nv']
    qpos = m['qpos0'] if qpos is None else qpos
    xpos = np.zeros((nbody, 3))
    xquat = np.zeros((nbody, 4))
    xquat[0] = [1, 0, 0, 0]
    dof_axis = np.zeros((nv, 3))      # rotation axis (world) or translation direction
    dof_anchor = np.zeros((nv, 3))
    dof_istrans = np.zeros(nv, bool)
    for b in range(1, nbody):
        p = m['body_parentid'][b]
        pos = xpos[p] + qrot(xquat[p], m['body_pos'][b])
        quat = qmul(xquat[p], m['body_quat'][b])
        for k in range(m['body_jntnum'][b]):
            j = m['body_jntadr'][b] + k
            qa, da = m['jnt_qposadr'][j], m['jnt_dofadr'][j]
            if m['jnt_type'][j] == JNT_FREE:
                pos = qpos[qa:qa + 3].copy()
                quat = qnorm(qpos[qa + 3:qa + 7])
                R = q2mat(quat)
                for i in range(3):
                    dof_axis[da + i] = np.eye(3)[i]
                    dof_istrans[da + i] = True
                    dof_axis[da + 3 + i] = R[:, i]
                    dof_anchor[da + 3 + i] = pos
            elif m['jnt_type'][j] == JNT_BALL:
                # rotation about the anchor (MuJoCo mj_kinematics); the dof axes are the body frame's columns (mj_comPos)
                anchor = pos + qrot(quat, m['jnt_pos'][j])
                quat = qmul(quat, qnorm(qpos[qa:qa + 4]))
                pos = anchor - qrot(quat, m['jnt_pos'][j])
                R = q2mat(quat)
                for i in range(3):
                    dof_axis[da + i] = R[:, i]
                    dof_anchor[da + i] = anchor
            else:
                anchor = pos + qrot(quat, m['jnt_pos'][j])
                axis = qrot(quat, m['jnt_axis'][j])
                ang = qpos[qa] - m['qpos0'][qa]
                quat = qmul(quat, axisangle2q(m['jnt_axis'][j], ang))
                pos = anchor - qrot(quat, m['jnt_pos'][j])
                dof_axis[da] = axis
                dof_anchor[da] = anchor
        xpos[b], xquat[b] = pos, qnorm(quat)
    return xpos, xquat, dof_axis, dof_anchor, dof_istrans


def body_jacobian(m, b, point, kin):
    _, _, ax, an, tr = kin
    nv = m['nv']
    Jp, Jr = np.zeros((3, nv)), np.zeros((3, nv))
    d = m['body_lastdof'][b]
    while d >= 0:
        if tr[d]:
            Jp[:, d] = ax[d]
        else:
            Jr[:, d] = ax[d]
            Jp[:, d] = np.cross(ax[d], point - an[d])
        d = m['dof_parentid'][d]
    return Jp, Jr


def dense_mass_matrix(m, qpos=None):
    kin = kinematics0(m, qpos)
    xpos, xquat = kin[0], kin[1]
    nv = m['nv']
    M = np.zeros((nv, nv))
    for b in range(1, m['nbody']):
        mass = m['body_mass'][b]
        if mass <= 0:
            continue
        c = xpos[b] + qrot(xquat[b], m['body_ipos'][b])
        Ri = q2mat(qmul(xquat[b], m['body_iquat'][b]))
        Iw = Ri @ np.diag(m['body_inertia'][b]) @ Ri.T
        Jp, Jr = body_jacobian(m, b, c, kin)
        M += mass * Jp.T @ Jp + Jr.T @ Iw @ Jr
    M += np.diag(m['dof_armature'])
    return M, kin


def _set0(m):
    nv, nbody = m['nv'], m['nbody']
    if nv == 0:
        m['dof_invweight0'] = np.zeros(0)
        m['body_invweight0'] = np.zeros((nbody, 2))
        m['stat_meaninertia'] = 1.0
        return
    M, kin = dense_mass_matrix(m)
    Minv = np.linalg.inv(M)
    m['stat_meaninertia'] = float(np.mean(np.diag(M)))
    xpos, xquat = kin[0], kin[1]
    biw = np.zeros((nbody, 2))
    for b in range(1, nbody):
        if m['body_lastdof'][b] < 0:
            continue
        c = xpos[b] + qrot(xquat[b], m['body_ipos'][b])
        Jp, Jr = body_jacobian(m, b, c, kin)
        Ap = Jp @ Minv @ Jp.T
        Ar = Jr @ Minv @ Jr.T
        biw[b] = [np.trace(Ap) / 3, np.trace(Ar) / 3]
    m['body_invweight0'] = biw
    diw = np.zeros(nv)
    for j in range(m['njnt']):
        da = m['jnt_dofadr'][j]
        if m['jnt_type'][j] == JNT_FREE:
            d = np.diag(Minv)[da:da + 6]
            diw[da:da + 3] = d[:3].mean()
            diw[da + 3:da + 6] = d[3:].mean()
        elif m['jnt_type'][j] == JNT_BALL:
            diw[da:da + 3] = np.diag(Minv)[da:da + 3].mean()
        else:
            diw[da] = Minv[da, da]
    m['dof_invweight0'] = diw
    # springdamper (halteres, fruitfly.xml:90): mass-spring-damper with given (timeconst, dampratio)
    # using the dof's effective inertia at qpos0 (MuJoCo mj_setConst).  [3P-memory]
    # joint dict list is not available here; springdamper was stored by the caller in jnt arrays
    sd = m.get('_jnt_springdamper')
    if sd is not None:
        for j in range(m['njnt']):
            tc, dr = sd[j]
            if tc > 0 and dr > 0:
                da = m['jnt_dofadr'][j]
                inertia = 1.0 / max(MINVAL, diw[da])
                m['jnt_stiffness'][j] = inertia / max(MINVAL, tc * tc * dr * dr)
                m['dof_damping'][da] = 2 * inertia / max(MINVAL, tc)


def save_model(m, path):
    arrays, meta = {}, {}
    for k, v in m.items():
        if k.startswith('_'):
            continue
        if isinstance(v, np.ndarray):
            arrays[k] = v
        else:
            meta[k] = v
    arrays['__meta__'] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(path, **arrays)


def main():
    import sys
    mode = sys.argv[1] if len(sys.argv) > 1 else 'legacy2'
    os.makedirs(ASSET_OUT, exist_ok=True)
    for variant in (sys.argv[2:] or ('bare', 'walk', 'flight', 'vision')):
        m = compile_variant(variant, inertia_mode=mode)
        save_model(m, os.path.join(ASSET_OUT, f'fly_{variant}.npz'))
        print(variant, {k: m[k] for k in ('nq', 'nv', 'nu', 'na', 'nbody', 'njnt', 'ngeom', 'ngeom_all', 'npair',
                                          'nsite', 'ntendon', 'nsensor', 'nsensordata', 'nM')},
              'mass', m['body_subtreemass'][1])


if __name__ == '__main__':
    main()
