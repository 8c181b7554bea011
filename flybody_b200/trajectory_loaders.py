"""Reference-trajectory loaders for the imitation tasks (reference `flybody/tasks/trajectory_loaders.py`).

Same classes, constructor arguments and return values as the reference: `HDF5WalkingTrajectoryLoader.get_trajectory`
returns the dict {qpos, qvel, root2site, joint_quat} of one walking snippet (`trajectory_loaders.py:185-264`),
`HDF5FlightTrajectoryLoader.get_trajectory` the (com_qpos, com_qvel) pair of one flight trajectory (`:67-141`); the
`Inference*` loaders serve the built-in synthetic trajectories (`:144-183`, `:267-302`).

Dataset layout (both files, `trajectory_loaders.py:35-37,94-100,235-262`):
    timestep_seconds                      scalar
    trajectories/<zero-padded idx>/...    walking: root_qpos [T,7] qpos [T,nj] root_qvel [T,6] qvel [T,nj]
                                                   root2site [T,ns,3] joint_quat [T,nj,4];  flight: com_qpos [T,7] com_qvel [T,6]
    trajectory_lengths [n_traj], id2name/joints, id2name/sites      (walking only)

h5py is not part of this image, so two storage backends are accepted behind the same classes: a real `.hdf5` file
when `h5py` is importable, and an `.npz` archive whose keys are the HDF5 paths above (`convert_hdf5_to_npz` writes one
wherever h5py exists).  There is no silent fallback between them: an `.hdf5` path without h5py raises ImportError.
"""
import numpy as np

from flybody_b200.synthetic import constant_speed_trajectory, _FLY_CONTROL_TIMESTEP, _WALK_CONTROL_TIMESTEP


class _Store:
    """Read-only view of a dataset file: `keys(prefix)`, `get(path)`."""

    def __init__(self, path):
        self._path = str(path)
        if self._path.endswith('.npz'):
            self._npz = np.load(self._path, allow_pickle=False)
            self._h5 = None
        else:
            try:
                import h5py
            except ImportError as exc:       # no CPU stand-in for a missing reader: say what to do
                raise ImportError(f'{self._path}: reading HDF5 needs h5py (absent here); convert the dataset with '
                                  'flybody_b200.trajectory_loaders.convert_hdf5_to_npz where h5py exists') from exc
            self._h5 = h5py.File(self._path, 'r')
            self._npz = None

    def children(self, group):
        if self._h5 is not None:
            return sorted(self._h5[group].keys())
        pre = group.rstrip('/') + '/'
        return sorted({k[len(pre):].split('/')[0] for k in self._npz.files if k.startswith(pre)})

    def get(self, path):
        if self._h5 is not None:
            return self._h5[path][()]
        return self._npz[path]


def convert_hdf5_to_npz(h5_path, npz_path):
    """Flatten an HDF5 trajectory dataset into the `.npz` layout `_Store` reads (needs h5py)."""
    import h5py
    out = {}
    with h5py.File(h5_path, 'r') as f:
        def visit(name, obj):
            if isinstance(obj, h5py.Dataset):
                v = obj[()]
                out[name] = np.asarray(v).astype('U') if getattr(v, 'dtype', None) is not None and v.dtype.kind in 'SO' else v
        f.visititems(visit)
    np.savez_compressed(npz_path, **out)


class HDF5TrajectoryLoader:
    """Base class (`trajectory_loaders.py:13-64`)."""

    def __init__(self, path, traj_indices=None, random_state=None):
        self._random_state = np.random.RandomState(None) if random_state is None else random_state
        self._store = _Store(path)
        self._keys = self._store.children('trajectories')
        self._n_traj = len(self._keys)
        self._timestep = float(np.asarray(self._store.get('timestep_seconds')))
        self._traj_indices = np.arange(self._n_traj) if traj_indices is None else traj_indices
        self._n_zeros = len(str(self._n_traj))

    @property
    def timestep(self):
        return self._timestep

    @property
    def num_trajectories(self):
        return self._n_traj

    @property
    def traj_indices(self):
        return self._traj_indices

    def _key(self, idx):
        return str(int(idx)).zfill(self._n_zeros)


class HDF5FlightTrajectoryLoader(HDF5TrajectoryLoader):
    """`trajectory_loaders.py:67-141`: CoM trajectories, optionally cut at a random start step."""

    def __init__(self, path, traj_indices=None, randomize_start_step=True, random_state=None):
        super().__init__(path, traj_indices, random_state=random_state)
        self._randomize_start_step = randomize_start_step
        self._com_qpos, self._com_qvel = [], []
        for idx in range(self._n_traj):
            g = f'trajectories/{self._key(idx)}/'
            self._com_qpos.append(np.asarray(self._store.get(g + 'com_qpos')))
            self._com_qvel.append(np.asarray(self._store.get(g + 'com_qvel')))
            assert self._com_qpos[-1].shape[0] == self._com_qvel[-1].shape[0]

    START_MARGIN = 50                                          # a random start leaves at least this many rows

    def trajectory_len(self, traj_idx):
        return len(self._com_qpos[traj_idx])

    @property
    def randomize_start_step(self):
        return self._randomize_start_step

    def full_trajectory(self, traj_idx):
        """(com_qpos [T,7], com_qvel [T,6]) of one whole trajectory as stored: no start cut, no shift to the origin (read-only)."""
        q, v = self._com_qpos[traj_idx].view(), self._com_qvel[traj_idx].view()
        q.flags.writeable = v.flags.writeable = False
        return q, v

    def get_trajectory(self, traj_idx=None, start_step=None, end_step=None):
        if traj_idx is None:
            traj_idx = self._random_state.choice(self._traj_indices)
        traj_len = len(self._com_qpos[traj_idx])
        if self._randomize_start_step:
            start_step, end_step = self._random_state.randint(traj_len - self.START_MARGIN), traj_len
        else:
            start_step = 0 if start_step is None else start_step
            end_step = traj_len if end_step is None else end_step
        com_qpos = self._com_qpos[traj_idx][start_step:end_step].copy()
        com_qvel = self._com_qvel[traj_idx][start_step:end_step]
        com_qpos[:, :2] -= com_qpos[0, :2]                    # every episode starts above the origin
        return com_qpos, com_qvel


class HDF5WalkingTrajectoryLoader(HDF5TrajectoryLoader):
    """`trajectory_loaders.py:185-264`: full-body walking snippets."""

    def __init__(self, path, traj_indices=None, random_state=None):
        super().__init__(path, traj_indices, random_state=random_state)
        self._traj_lens = np.asarray(self._store.get('trajectory_lengths'))

    def trajectory_len(self, traj_idx):
        return int(self._traj_lens[traj_idx])

    _FIELDS = ('root_qpos', 'qpos', 'root_qvel', 'qvel', 'root2site', 'joint_quat')

    def full_trajectory(self, traj_idx):
        """{root_qpos, qpos, root_qvel, qvel, root2site, joint_quat} of one whole trajectory as stored: no shift of the root x, y to
        the origin, no draw from the loader's RandomState (read-only)."""
        g = f'trajectories/{self._key(traj_idx)}/'
        out = {}
        for k in self._FIELDS:
            out[k] = np.array(self._store.get(g + k))
            out[k].flags.writeable = False
        return out

    def get_trajectory(self, traj_idx=None, start_step=None, end_step=None):
        if traj_idx is None:
            traj_idx = self._random_state.choice(self._traj_indices)
        start_step = 0 if start_step is None else start_step
        end_step = int(self._traj_lens[traj_idx]) if end_step is None else end_step
        g = f'trajectories/{self._key(traj_idx)}/'
        get = lambda k: np.asarray(self._store.get(g + k))[start_step:end_step]
        qpos = np.concatenate((get('root_qpos'), get('qpos')), axis=1)
        qvel = np.concatenate((get('root_qvel'), get('qvel')), axis=1)
        qpos[:, :2] -= qpos[0, :2]
        return {'qpos': qpos, 'qvel': qvel, 'root2site': get('root2site'), 'joint_quat': get('joint_quat')}

    @staticmethod
    def _names(arr):
        return [s.decode('utf-8') if isinstance(s, bytes) else str(s) for s in np.asarray(arr).tolist()]

    def get_site_names(self):
        return self._names(self._store.get('id2name/sites'))

    def get_joint_names(self):
        return self._names(self._store.get('id2name/joints'))


class InferenceWalkingTrajectoryLoader:
    """`trajectory_loaders.py:267-302`: a 300-step straight walk at 2 cm/s unless `set_next_trajectory` is called."""

    def __init__(self):
        qpos, qvel = constant_speed_trajectory(n_steps=300, speed=2, init_pos=(0, 0, 0.1278), control_timestep=_WALK_CONTROL_TIMESTEP)
        self.set_next_trajectory(qpos, qvel)

    def set_next_trajectory(self, qpos, qvel):
        self._snippet = {'qpos': np.asarray(qpos, np.float64), 'qvel': np.asarray(qvel, np.float64)}

    def get_trajectory(self, traj_idx=None):
        return self._snippet

    def get_joint_names(self):
        return []

    def get_site_names(self):
        return []


class InferenceFlightTrajectoryLoader:
    """`trajectory_loaders.py:144-183`: a 200-step straight flight at 20 cm/s, 1 cm above the floor, pitched -47.5 deg."""

    def __init__(self):
        qpos, qvel = constant_speed_trajectory(n_steps=200, speed=20, init_pos=(0, 0, 1), body_rot_angle_y=-47.5,
                                               control_timestep=_FLY_CONTROL_TIMESTEP)
        self.set_next_trajectory(qpos, qvel)

    def set_next_trajectory(self, com_qpos, com_qvel):
        self._com_qpos = np.array(com_qpos, np.float64)
        self._com_qpos[:, :2] -= self._com_qpos[0, :2]
        self._com_qvel = np.asarray(com_qvel, np.float64)

    def get_trajectory(self, traj_idx=None):
        return self._com_qpos, self._com_qvel
