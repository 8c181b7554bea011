"""`FlyModel`: the flat model the stepper reads, and its ctypes mirror of `FbModel`
(`include/flybody_b200.h`).  The field table below is the single source of truth: the C struct
text in the header is generated from it (`c_struct_text`) and a test keeps them in sync.

Arrays are the subset of `mjModel` the fly's `mj_step` pipeline touches (SURVEY.md App. D.1).
"""
import ctypes as C
import json
import os

import numpy as np

ASSETS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'assets')

# (name, kind) kind: 'i' int32 scalar, 'd' double scalar, 'd3' double[3], 'pi' const int32*, 'pd' const double*
FIELDS = [
    # sizes
    ('nq', 'i'), ('nv', 'i'), ('nu', 'i'), ('na', 'i'), ('nbody', 'i'), ('njnt', 'i'), ('ngeom', 'i'),
    ('npair', 'i'), ('nsite', 'i'), ('ntendon', 'i'), ('nwrap', 'i'), ('nsensor', 'i'),
    ('nsensordata', 'i'), ('nM', 'i'), ('nfluid', 'i'),
    # options
    ('opt_iterations', 'i'), ('opt_ls_iterations', 'i'), ('opt_noslip_iterations', 'i'),
    ('opt_cone_elliptic', 'i'),
    ('opt_timestep', 'd'), ('opt_gravity', 'd3'), ('opt_density', 'd'), ('opt_viscosity', 'd'),
    ('opt_wind', 'd3'), ('opt_impratio', 'd'), ('opt_tolerance', 'd'), ('opt_ls_tolerance', 'd'),
    ('opt_noslip_tolerance', 'd'), ('stat_meaninertia', 'd'),
    # bodies
    ('body_parentid', 'pi'), ('body_rootid', 'pi'), ('body_jntadr', 'pi'), ('body_jntnum', 'pi'),
    ('body_dofadr', 'pi'), ('body_dofnum', 'pi'), ('body_lastdof', 'pi'), ('body_fluid_ellipsoid', 'pi'),
    ('body_pos', 'pd'), ('body_quat', 'pd'), ('body_ipos', 'pd'), ('body_iquat', 'pd'),
    ('body_mass', 'pd'), ('body_inertia', 'pd'), ('body_invweight0', 'pd'), ('body_subtreemass', 'pd'),
    # joints / dofs
    ('jnt_type', 'pi'), ('jnt_qposadr', 'pi'), ('jnt_dofadr', 'pi'), ('jnt_bodyid', 'pi'),
    ('jnt_limited', 'pi'),
    ('jnt_pos', 'pd'), ('jnt_axis', 'pd'), ('jnt_stiffness', 'pd'), ('jnt_range', 'pd'),
    ('jnt_solref', 'pd'), ('jnt_solimp', 'pd'), ('jnt_margin', 'pd'), ('qpos0', 'pd'), ('qpos_spring', 'pd'),
    ('dof_bodyid', 'pi'), ('dof_jntid', 'pi'), ('dof_parentid', 'pi'), ('dof_Madr', 'pi'),
    ('dof_armature', 'pd'), ('dof_damping', 'pd'), ('dof_invweight0', 'pd'),
    # collision geoms
    ('geom_type', 'pi'), ('geom_bodyid', 'pi'), ('geom_condim', 'pi'), ('geom_priority', 'pi'),
    ('geom_size', 'pd'), ('geom_pos', 'pd'), ('geom_quat', 'pd'), ('geom_rbound', 'pd'),
    ('geom_friction', 'pd'), ('geom_solmix', 'pd'), ('geom_solref', 'pd'), ('geom_solimp', 'pd'),
    ('geom_margin', 'pd'), ('geom_gap', 'pd'),
    ('pair_geom1', 'pi'), ('pair_geom2', 'pi'),
    # ellipsoid-fluid geoms
    ('fluid_bodyid', 'pi'), ('fluid_pos', 'pd'), ('fluid_quat', 'pd'), ('fluid_size', 'pd'),
    ('fluid_coef', 'pd'),
    # sites
    ('site_bodyid', 'pi'), ('site_type', 'pi'), ('site_pos', 'pd'), ('site_quat', 'pd'), ('site_size', 'pd'),
    # tendons
    ('tendon_adr', 'pi'), ('tendon_num', 'pi'), ('wrap_dofid', 'pi'), ('wrap_qposadr', 'pi'),
    ('wrap_coef', 'pd'),
    # actuators
    ('actuator_trntype', 'pi'), ('actuator_trnid', 'pi'), ('actuator_dyntype', 'pi'),
    ('actuator_biastype', 'pi'), ('actuator_ctrllimited', 'pi'), ('actuator_forcelimited', 'pi'),
    ('actuator_actadr', 'pi'),
    ('actuator_dynprm', 'pd'), ('actuator_gainprm', 'pd'), ('actuator_biasprm', 'pd'),
    ('actuator_ctrlrange', 'pd'), ('actuator_forcerange', 'pd'),
    # sensors
    ('sensor_type', 'pi'), ('sensor_objid', 'pi'), ('sensor_adr', 'pi'), ('sensor_dim', 'pi'),
]

_CT = {'i': C.c_int32, 'd': C.c_double, 'd3': C.c_double * 3,
       'pi': C.POINTER(C.c_int32), 'pd': C.POINTER(C.c_double)}
_CDECL = {'i': 'int32_t %s;', 'd': 'double %s;', 'd3': 'double %s[3];',
          'pi': 'const int32_t* %s;', 'pd': 'const double* %s;'}


class FbModel(C.Structure):
    _fields_ = [(n, _CT[k]) for n, k in FIELDS]


def c_struct_text():
    lines = ['typedef struct FbModel {']
    lines += ['  ' + _CDECL[k] % n for n, k in FIELDS]
    lines.append('} FbModel;')
    return '\n'.join(lines)


class FlyModel:
    """Host-side model: numpy arrays + names + a live ctypes `FbModel` view."""

    def __init__(self, arrays, meta):
        self.meta = meta
        self.a = {}
        for k, v in arrays.items():
            self.a[k] = v
        for k, v in meta.items():
            if k not in self.a:
                self.a[k] = v
        self._keep = []
        self.c = self._build_c()

    def __getattr__(self, k):
        a = self.__dict__.get('a')
        if a is not None and k in a:
            return a[k]
        raise AttributeError(k)

    def _build_c(self):
        s = FbModel()
        for n, k in FIELDS:
            v = self.a[n]
            if k == 'i':
                setattr(s, n, int(v))
            elif k == 'd':
                setattr(s, n, float(v))
            elif k == 'd3':
                setattr(s, n, (C.c_double * 3)(*[float(x) for x in np.asarray(v).ravel()]))
            elif k == 'pi':
                arr = np.ascontiguousarray(np.asarray(v, dtype=np.int32).ravel())
                if arr.size == 0:
                    arr = np.zeros(1, np.int32)
                self._keep.append(arr)
                setattr(s, n, arr.ctypes.data_as(C.POINTER(C.c_int32)))
            else:
                arr = np.ascontiguousarray(np.asarray(v, dtype=np.float64).ravel())
                if arr.size == 0:
                    arr = np.zeros(1, np.float64)
                self._keep.append(arr)
                setattr(s, n, arr.ctypes.data_as(C.POINTER(C.c_double)))
        return s

    def rebuild(self):
        """Re-create the ctypes view after editing arrays in `self.a`."""
        self._keep = []
        self.c = self._build_c()
        return self

    def copy(self):
        import copy as _copy
        return FlyModel({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self.a.items()
                         if isinstance(v, np.ndarray)}, _copy.deepcopy(self.meta))

    # name lookups ------------------------------------------------------------------------
    def body_id(self, name):
        return self.meta['body_names'].index(name)

    def jnt_id(self, name):
        return self.meta['jnt_names'].index(name)

    def site_id(self, name):
        return self.meta['site_names'].index(name)

    def jnt_qposadr_of(self, name):
        return int(self.a['jnt_qposadr'][self.jnt_id(name)])

    def jnt_dofadr_of(self, name):
        return int(self.a['jnt_dofadr'][self.jnt_id(name)])


def load_model(variant='walk', path=None):
    if path is None and variant == 'template':
        return template_from_walk(load_model('walk'))
    if path is None and variant == 'ball':
        return ball_from_template(load_model('template'))
    path = path or os.path.join(ASSETS, f'fly_{variant}.npz')
    d = np.load(path)
    meta = json.loads(bytes(d['__meta__']).decode())
    arrays = {k: d[k] for k in d.files if k != '__meta__'}
    return FlyModel(arrays, meta)


_TRAILING = (('body_', 'nbody', 'body_names'), ('jnt_', 'njnt', 'jnt_names'), ('site_', 'nsite', 'site_names'))


def template_from_walk(walk):
    """The model of `template_task` (reference tasks/template_task.py:35: the Walking task with add_ghost=False) cut from the walk model:
    the compiler appends the ghost after the walker (its body, free joint, 7 qpos, 6 dofs and site come last, its geoms do not collide),
    so the walker's arrays are the leading parts of the walk model's.  Recomputed: the sizes, the world's subtree mass and the mean
    inertia at qpos0 (mj_setConst; the ghost's armature dominated it).  The invweights and the stiffness / damping the compiler derives
    from them are kept: the ghost is a tree of its own, so they differ from a compile without it by rounding only
    (`compile_variant('template')` compiles it, and tests/test_template_task.py holds the two together where the reference's XML is
    reachable)."""
    a, meta = dict(walk.a), json.loads(json.dumps(walk.meta))
    cut = {}
    for prefix, size, names in _TRAILING:
        keep = [n for n in meta[names] if not n.startswith('ghost/')]
        assert meta[names][:len(keep)] == keep, f'the ghost is not at the end of {names}'
        cut[prefix] = len(keep)
        meta[names], meta[size] = keep, len(keep)
    nv = int((a['dof_bodyid'] < cut['body_']).sum())
    assert np.all(a['dof_bodyid'][:nv] < cut['body_']), 'the ghost dofs are not at the end'
    last = cut['jnt_'] - 1                 # free (type 0): 7 qpos; hinge: 1
    nq = int(a['jnt_qposadr'][last] + (7 if a['jnt_type'][last] == 0 else 1))
    cut['dof_'] = nv
    out = {}
    for k, v in a.items():
        if not isinstance(v, np.ndarray) or k in meta:
            continue
        n = nq if k in ('qpos0', 'qpos_spring') else next((cut[p] for p in cut if k.startswith(p)), None)
        out[k] = v[:n].copy() if n is not None else v.copy()
    for k in ('geom_bodyid', 'site_bodyid', 'fluid_bodyid'):
        assert not len(out[k]) or out[k].max() < meta['nbody'], k
    chain = np.zeros(nv, np.int64)
    for d in range(nv):
        p = out['dof_parentid'][d]
        chain[d] = 1 + (chain[p] if p >= 0 else 0)
    meta['nv'], meta['nq'], meta['nM'] = nv, nq, int(chain.sum())
    assert np.array_equal(out['dof_Madr'], np.concatenate([[0], np.cumsum(chain)[:-1]]))
    children = out['body_parentid'][1:] == 0
    out['body_subtreemass'][0] = out['body_mass'][0] + out['body_subtreemass'][1:][children].sum()
    meta.pop('ngeom_all', None)           # (the count of every geom of the compiled MJCF, visual ones included, is not recoverable here)
    from .compiler.compile_model import dense_mass_matrix
    M, _ = dense_mass_matrix({**out, **meta})
    meta['stat_meaninertia'] = float(np.mean(np.diag(M)))
    return FlyModel(out, meta)


def ball_from_template(template):
    """The model of `walk_on_ball` (reference fly_envs.py:158-191, tasks/walk_on_ball.py) built from the template model: the same Walking
    surgery without the ghost, with the walker's free joint removed (its thorax becomes a jointless root at the spawn pose) and BallFloor's
    ball (`compiler.compile_model._ball_body`: a sphere on a ball joint, 4 qpos, 3 dofs) as the first body, joint, qpos and dofs, its
    geom in place of the floor plane.  The collision pairs are the template's with the ball in the floor's place: the floor's pairs become
    the ball's, and the thorax excludes of walk_on_ball.py:30-38 remove the thorax-child pairs that the template's parent-child filter
    removed.  The world's subtree mass, the invweights, the mean inertia and the halteres' springdamper stiffness and damping are
    recomputed at qpos0 (mj_setConst: welding the thorax changes the halteres' effective inertia).  `compile_variant('ball')` compiles it
    from the reference's XML, and tests/test_walk_on_ball.py holds the two together where that file is reachable."""
    from .compiler import compile_model as cm
    t, meta = template.a, json.loads(json.dumps(template.meta))
    jn = meta['jnt_names']
    assert jn[0] == 'walker/' and t['jnt_type'][0] == cm.JNT_FREE and t['jnt_qposadr'][1] == 7 and t['jnt_dofadr'][1] == 6, \
        'the template model does not start with the walker\'s free joint'
    assert t['geom_type'][0] == cm.GEOM_PLANE and t['geom_bodyid'][0] == 0, 'the template model has no floor plane first'
    assert t['body_parentid'][1] == 0 and t['body_jntadr'][1] == 0 and t['body_jntnum'][1] == 1
    ball = cm._ball_body()
    cm._body_inertial(ball)
    bj, bg = ball.joints[0], ball.geoms[0]
    nb, nv = int(meta['nbody']) + 1, int(meta['nv']) - 3
    a = {}

    def ins(k, row):                       # insert the ball's row at body index 1
        return np.insert(np.asarray(t[k]), 1, row, axis=0)
    bshift = lambda v: np.where(np.asarray(v) > 0, np.asarray(v) + 1, np.asarray(v))      # body ids after the inserted ball
    a['body_parentid'] = ins('body_parentid', 0)
    a['body_parentid'][2:] = bshift(t['body_parentid'][1:])
    a['body_rootid'] = ins('body_rootid', 1)
    a['body_rootid'][2:] = bshift(t['body_rootid'][1:])
    a['body_weldid'] = np.zeros(nb, np.int32)
    a['body_jntadr'] = ins('body_jntadr', 0)
    a['body_jntadr'][2] = -1
    a['body_jntnum'] = ins('body_jntnum', 1)
    a['body_jntnum'][2] = 0
    a['body_dofadr'] = ins('body_dofadr', 0)
    a['body_dofadr'][2:] = np.where(t['body_dofadr'][1:] >= 6, t['body_dofadr'][1:] - 3, -1)
    a['body_dofnum'] = ins('body_dofnum', 3)
    a['body_dofnum'][2] = 0
    for k, row in (('body_pos', ball.pos), ('body_quat', ball.quat), ('body_ipos', ball.ipos), ('body_iquat', ball.iquat),
                   ('body_mass', ball.mass), ('body_inertia', ball.inertia), ('body_fluid_ellipsoid', 0), ('body_invweight0', (0.0, 0.0)),
                   ('body_subtreemass', ball.mass)):
        a[k] = ins(k, row)
    for b in range(1, nb):
        a['body_weldid'][b] = b if a['body_jntnum'][b] > 0 else a['body_weldid'][a['body_parentid'][b]]
    lastdof = np.full(nb, -1, np.int32)
    for b in range(1, nb):
        lastdof[b] = a['body_dofadr'][b] + a['body_dofnum'][b] - 1 if a['body_dofnum'][b] > 0 else lastdof[a['body_parentid'][b]]
    a['body_lastdof'] = lastdof
    a['body_subtreemass'][0] = a['body_mass'][0] + a['body_subtreemass'][1:][a['body_parentid'][1:] == 0].sum()
    # joints: the walker's free joint (joint 0) becomes the ball joint; qpos 7 -> 4, dofs 6 -> 3
    for k in [k for k in t if k.startswith('jnt_') and isinstance(t[k], np.ndarray)]:
        a[k] = np.array(t[k], copy=True)
    a['jnt_type'][0], a['jnt_bodyid'][0] = cm.JNT_BALL, 1
    a['jnt_bodyid'][1:] = t['jnt_bodyid'][1:] + 1
    a['jnt_qposadr'][1:] -= 3
    a['jnt_dofadr'][1:] -= 3
    for k, v in (('jnt_pos', bj['pos']), ('jnt_axis', bj['axis']), ('jnt_stiffness', bj['stiffness']), ('jnt_range', bj['range']),
                 ('jnt_limited', bj['limited']), ('jnt_solref', bj['solref']), ('jnt_solimp', bj['solimp']), ('jnt_margin', bj['margin'])):
        a[k][0] = v
    a['qpos0'] = np.concatenate([[1.0, 0, 0, 0], t['qpos0'][7:]])
    a['qpos_spring'] = np.concatenate([[1.0, 0, 0, 0], t['qpos_spring'][7:]])
    a['dof_bodyid'] = np.concatenate([[1, 1, 1], t['dof_bodyid'][6:] + 1]).astype(np.int32)
    a['dof_jntid'] = np.concatenate([[0, 0, 0], t['dof_jntid'][6:]]).astype(np.int32)
    a['dof_armature'] = np.concatenate([[bj['armature']] * 3, t['dof_armature'][6:]])
    a['dof_damping'] = np.concatenate([[bj['damping']] * 3, t['dof_damping'][6:]])
    par = np.full(nv, -1, np.int32)
    for d in range(nv):
        b = a['dof_bodyid'][d]
        par[d] = d - 1 if d > a['body_dofadr'][b] else lastdof[a['body_parentid'][b]]
    a['dof_parentid'] = par
    chain = np.zeros(nv, np.int64)
    for d in range(nv):
        chain[d] = 1 + (chain[par[d]] if par[d] >= 0 else 0)
    a['dof_Madr'] = np.concatenate([[0], np.cumsum(chain)[:-1]]).astype(np.int32)
    # geoms: the ball's sphere in the floor's slot (both come first: the world's, then body 1's)
    for k in [k for k in t if k.startswith('geom_') and isinstance(t[k], np.ndarray)]:
        a[k] = np.array(t[k], copy=True)
    a['geom_bodyid'][1:] += 1
    for k, v in (('geom_type', bg['type']), ('geom_bodyid', 1), ('geom_size', bg['size']), ('geom_pos', bg['pos']), ('geom_quat', bg['quat']),
                 ('geom_rbound', cm.rbound(bg['type'], bg['size'])), ('geom_condim', bg['condim']), ('geom_priority', bg['priority']),
                 ('geom_friction', bg['friction']), ('geom_solmix', bg['solmix']), ('geom_solref', bg['solref']), ('geom_solimp', bg['solimp']),
                 ('geom_margin', bg['margin']), ('geom_gap', bg['gap'])):
        a[k][0] = v
    meta['geom_names'][0] = bg['name']
    for k in ('site_bodyid', 'fluid_bodyid'):
        a[k] = t[k] + 1
    a['wrap_dofid'], a['wrap_qposadr'] = t['wrap_dofid'] - 3, t['wrap_qposadr'] - 3
    a['actuator_trnid'] = np.where(t['actuator_trntype'] == cm.TRN_BODY, t['actuator_trnid'] + 1, t['actuator_trnid'])
    for k, v in t.items():
        if isinstance(v, np.ndarray) and k not in a:
            a[k] = np.array(v, copy=True)
    meta['jnt_names'][0] = bj['name']
    meta['body_names'].insert(1, ball.name)
    meta.update(nbody=nb, nq=int(meta['nq']) - 3, nv=nv, nM=int(chain.sum()))
    # mj_setConst at qpos0: the invweights, the mean inertia and the springdamper joints (class `haltere`, fruitfly.xml:89-91), whose
    # (timeconst, dampratio) are recovered from the template's values
    m = {**a, **meta}
    sd = [np.zeros(2)] * len(jn)
    for j, name in enumerate(jn):
        if 'haltere' in name:
            da = t['jnt_dofadr'][j]
            inertia = 1.0 / t['dof_invweight0'][da]
            tc = 2 * inertia / t['dof_damping'][da]
            sd[j] = np.array([tc, np.sqrt(inertia / (t['jnt_stiffness'][j] * tc * tc))])
    m['_jnt_springdamper'] = sd
    cm._set0(m)
    for k in ('body_invweight0', 'dof_invweight0', 'jnt_stiffness', 'dof_damping'):
        a[k] = m[k]
    meta['stat_meaninertia'] = m['stat_meaninertia']
    return FlyModel(a, meta)


def from_compiled(m):
    arrays = {k: v for k, v in m.items() if isinstance(v, np.ndarray)}
    meta = {k: v for k, v in m.items() if not isinstance(v, np.ndarray) and not k.startswith('_')}
    return FlyModel(arrays, meta)


# ------------------------------------------------------------------------------------------------ model variants on demand
def reference_assets_dir():
    """Directory holding the reference's `fruitfly.xml` + meshes: $FLYBODY_ASSETS or an installed `flybody` package.  None if
    neither is present (only the shipped, pre-compiled variants are available)."""
    cand = [os.environ.get('FLYBODY_ASSETS')]
    try:
        import importlib.util
        spec = importlib.util.find_spec('flybody')
        if spec is not None and spec.submodule_search_locations:
            cand.append(os.path.join(list(spec.submodule_search_locations)[0], 'fruitfly', 'assets'))
    except Exception:
        pass
    for c in cand:
        if c and os.path.exists(os.path.join(c, 'fruitfly.xml')):
            return c
    return None


def variant_name(variant, force_actuators=False, use_wings=None, use_legs=None, joint_filter=None, adhesion_filter=None):
    name = f'fly_{variant}'
    if force_actuators:
        name += '_force'
    if use_wings is not None:
        name += '_wings' if use_wings else '_nowings'
    if use_legs is not None:
        name += '_legs' if use_legs else '_nolegs'
    if joint_filter is not None:
        name += f'_jf{joint_filter:g}'
    if adhesion_filter is not None:
        name += f'_af{adhesion_filter:g}'
    return name


def model_for(variant, force_actuators=False, use_wings=None, use_legs=None, joint_filter=None, cache_dir=None, adhesion_filter=None):
    """The compiled model of a task (`variant` = walk / flight / vision / template) with the `FruitFly` switches the reference's env
    factories expose (reference fly_envs.py:100-300: force_actuators, disable_wings, disable_legs, joint_filter, adhesion_filter;
    None = the task's default).
    The default models ship pre-compiled (`assets/fly_*.npz`); any other combination is compiled from the reference's
    `fruitfly.xml` on first use (`flybody_b200.compiler`, ~2 s) and cached."""
    if not force_actuators and use_wings is None and use_legs is None and joint_filter is None and adhesion_filter is None:
        return load_model(variant)
    if variant == 'ball':               # walk_on_ball's model is cut from the template model with the same switches
        return ball_from_template(model_for('template', force_actuators, use_wings, use_legs, joint_filter, cache_dir, adhesion_filter))
    name = variant_name(variant, force_actuators, use_wings, use_legs, joint_filter, adhesion_filter)
    cache_dir = cache_dir or os.environ.get('FLYBODY_B200_CACHE') or os.path.join(os.path.expanduser('~'), '.cache', 'flybody_b200')
    for d in (ASSETS, cache_dir):
        p = os.path.join(d, name + '.npz')
        if os.path.exists(p):
            return load_model(path=p)
    src = reference_assets_dir()
    if src is None:
        raise NotImplementedError(
            f'model variant {name} is not among the pre-compiled ones ({sorted(f for f in os.listdir(ASSETS) if f.endswith(".npz"))}) and the '
            "reference's fruitfly.xml was not found to compile it: install flybody or set FLYBODY_ASSETS to its fruitfly/assets directory")
    from .compiler import compile_model as cm
    m = cm.compile_variant(variant, assets_dir=src, mesh_cache=cm.load_mesh_cache(src), force_actuators=force_actuators, use_wings=use_wings,
                           use_legs=use_legs, joint_filter=joint_filter, **({} if adhesion_filter is None else dict(adhesion_filter=adhesion_filter)))
    os.makedirs(cache_dir, exist_ok=True)
    p = os.path.join(cache_dir, name + '.npz')
    cm.save_model(m, p)
    return load_model(path=p)
