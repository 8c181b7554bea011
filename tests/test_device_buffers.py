"""Device buffers of a stepper handle on the host-emulation build, where device memory is process heap: a re-programmed eye camera
frees the images it replaces, renders as a handle programmed once, and the env's device view follows the new buffer."""
import ctypes

import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import vision_env


class _Mallinfo2(ctypes.Structure):
    _fields_ = [(f, ctypes.c_size_t) for f in ('arena', 'ordblks', 'smblks', 'hblks', 'hblkhd', 'usmblks', 'fsmblks', 'uordblks', 'fordblks',
                                              'keepcost')]


def _heap_in_use():
    """bytes of the process heap in use (glibc mallinfo2: allocated small blocks + mmapped blocks)"""
    libc = ctypes.CDLL(None)
    libc.mallinfo2.restype = _Mallinfo2
    m = libc.mallinfo2()
    return m.uordblks + m.hblkhd


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def _env(emu, n_envs, size):
    return vision_env.BatchedVisionFlightEnv(n_envs, lib_path=emu, seed=5, eye_camera_size=size, terrain_bank=2)


def _reprogram(env, size):
    """the env's eye program again, with images of size x size"""
    m = env.model
    env._eye_program(size, 150.0, m.meta['hf_nrow'], m.meta['hf_ncol'], env._half, float(m.geom_pos[m.meta['hf_geom']][2]))


def test_eye_program_frees_the_images_it_replaces(emu):
    env = _env(emu, 64, 64)
    image = 64 * 2 * 64 * 64 * 3                                        # one program's images: 1.5 MiB
    _reprogram(env, 64)
    before = _heap_in_use()
    for _ in range(20):
        _reprogram(env, 64)
    grown = _heap_in_use() - before
    env.close()
    assert grown < image, f'20 eye programs kept {grown / image:.1f} image buffers'


def test_reprogrammed_eyes_render_as_a_fresh_handle(emu):
    env, fresh = _env(emu, 4, 32), _env(emu, 4, 24)
    env.reset()
    fresh.reset()
    _reprogram(env, 24)
    img = env._sim.render_eyes()
    assert img.shape == (4, 2, 24, 24, 3)
    np.testing.assert_array_equal(img, fresh._sim.render_eyes())
    env.close()
    fresh.close()


def test_eyes_device_reads_the_live_buffer_after_a_reprogram(emu, monkeypatch):
    def host_view(ptr, shape, typestr, device):      # emulation build: the library's "device" buffer is host memory
        return np.ctypeslib.as_array((ctypes.c_uint8 * int(np.prod(shape))).from_address(ptr)).reshape(shape)
    monkeypatch.setattr(vision_env, '_device_tensor', host_view)
    env = _env(emu, 4, 32)
    env.reset()
    env.eyes_device()
    _reprogram(env, 32)
    img = env._sim.render_eyes()
    view = env.eyes_device()
    assert view.ctypes.data == env._sim.eyes_ptr()[0]
    np.testing.assert_array_equal(view, img)
    env.close()
