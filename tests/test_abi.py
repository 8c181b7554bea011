"""The C ABI (no GPU needed): every function include/flybody_b200.h declares is bound and exported by both builds, and the
bindings, struct layouts and enum values that flybody_b200.abi reads from the header agree with what the C compiler makes of it."""
import ctypes
import os
import re
import subprocess

import pytest

import __graft_entry__ as ge
from flybody_b200 import abi, stepper
from flybody_b200.flymodel import FbModel
from oracle import fly_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROGRAMS = {'FbObsProgram': stepper.FbObsProgram, 'FbTaskProgram': stepper.FbTaskProgram, 'FbEyeProgram': stepper.FbEyeProgram,
            'FbIkProgram': stepper.FbIkProgram, 'FbModel': FbModel}


def declared_symbols():
    hdr = open(os.path.join(ROOT, 'include', 'flybody_b200.h')).read()
    return set(re.findall(r'\b(fb_[a-z_]+)\s*\(', hdr))


def exported_symbols(so):
    out = subprocess.run(['nm', '-D', '--defined-only', so], check=True, capture_output=True, text=True).stdout
    return {ln.split()[-1] for ln in out.splitlines() if ln.split()[-1].startswith('fb_')}


def run_cxx(tmp_path, source):
    """compile C++ that includes the header with g++ and run it -> its stdout"""
    src, exe = tmp_path / 'abi_probe.cpp', tmp_path / 'abi_probe'
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include <type_traits>\n#include "flybody_b200.h"\n' + source)
    subprocess.check_call(['g++', '-std=c++17', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)])
    return subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout


def test_build_binds_and_exports_every_declared_function():
    ge.build()
    lib = stepper.load_library()
    bound = {name for name in abi.read().functions if getattr(lib, name).argtypes is not None}
    assert len(bound) >= 20
    assert bound == declared_symbols() == exported_symbols(stepper.LIB_PATH) & exported_symbols(ge.EMU)
    assert b'sm_90a' in ctypes.c_char_p(ctypes.cast(lib.fb_version, ctypes.CFUNCTYPE(ctypes.c_char_p))()).value


def test_struct_layouts_match_the_compiler(tmp_path):
    """sizeof and every field's offset and size of the program structs and FbModel, from g++ against the ctypes classes"""
    probe = ''.join(f'  printf("{s} sizeof 0 %zu\\n", sizeof({s}));\n' + ''.join(
        f'  printf("{s} {f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s}*)0)->{f}));\n' for f, _ in cls._fields_)
        for s, cls in PROGRAMS.items())
    want = run_cxx(tmp_path, f'int main() {{\n{probe}  return 0;\n}}\n').splitlines()
    have = []
    for s, cls in PROGRAMS.items():
        have.append(f'{s} sizeof 0 {ctypes.sizeof(cls)}')
        have += [f'{s} {f} {getattr(cls, f).offset} {getattr(cls, f).size}' for f, _ in cls._fields_]
    assert have == want


def _kind(t):
    """size and kind of a bound ctypes type (f floating point, p pointer, i integer), or void"""
    if t is None:
        return 'void'
    kind = 'f' if t in (ctypes.c_float, ctypes.c_double) else 'p' if t in (ctypes.c_void_p, ctypes.c_char_p) else 'i'
    return f'{ctypes.sizeof(t)}{kind}'


def test_bound_signatures_match_the_compiler(tmp_path):
    """the size and kind (floating point, pointer, integer) of every bound return type and parameter, from the compiler's
    decltype(&fb_x) against the restype and argtypes load_library sets"""
    lib = stepper.load_library()
    funcs = abi.read().functions
    probe = '''template <class T> void put() {
  if constexpr (std::is_void_v<T>) printf(" void");
  else printf(" %zu%c", sizeof(T), std::is_floating_point_v<T> ? 'f' : std::is_pointer_v<T> ? 'p' : 'i');
}
template <class F> struct Sig;
template <class R, class... A> struct Sig<R (*)(A...)> {
  static void put_all(const char* name) { printf("%s", name); put<R>(); printf(" :"); (put<A>(), ...); printf("\\n"); }
};
int main() {
''' + ''.join(f'  Sig<decltype(&{f})>::put_all("{f}");\n' for f in funcs) + '  return 0;\n}\n'
    want = run_cxx(tmp_path, probe).splitlines()
    have = [' '.join([f, _kind(getattr(lib, f).restype), ':'] + [_kind(t) for t in getattr(lib, f).argtypes]) for f in funcs]
    assert have == want
    assert len(want) == len(declared_symbols())


def test_enum_values_are_pinned():
    """the ids the Python side has always used; changing one in the header changes every caller's meaning"""
    fields = ('QPOS QVEL ACT CTRL QACC QACC_WARMSTART SENSORDATA SENSOR_MEAN XPOS XMAT SITE_XPOS SITE_XMAT SUBTREE_COM NCON NEFC TIME '
              'QFRC_SMOOTH QM_DENSE QFRC_CONSTRAINT SOLVER_NITER QFRC_PASSIVE QFRC_BIAS QFRC_ACTUATOR CONTACT EFC_FORCE FLAGS '
              'QFRC_APPLIED XFRC_APPLIED').split()
    obs = ('SENSOR_MEAN SENSOR_NOW ACT QPOS QVEL SITES_EGO ROOT_ZAXIS REF_DISP REF_QUAT SCALARS ROOT_POSE SUBTREE_COM DOF_AXIS_EGO '
           'WORLD_CONTACT TASK_TARGET').split()
    for i, name in enumerate(fields):
        assert getattr(stepper, name) == getattr(fly_oracle, name) == i, name
    for i, name in enumerate(obs):
        assert getattr(stepper, 'OBS_' + name) == i, name
    for i, name in enumerate(('WALK', 'FLIGHT', 'VISION', 'TEMPLATE', 'BALL')):
        assert getattr(stepper, 'TASK_' + name) == i, name
    assert stepper.PARAMS == ('body_mass', 'body_inertia', 'dof_armature', 'dof_damping', 'jnt_stiffness', 'geom_friction',
                              'actuator_gainprm', 'actuator_biasprm', 'gravity', 'wind', 'density', 'viscosity')
    assert sorted(abi.read().enums['FbParam'].values()) == list(range(len(stepper.PARAMS) + 1))     # + FB_NPARAMS
    assert (stepper.MAXCON, stepper.MAXEFC) == (64, 160)


@pytest.mark.parametrize('old, new, line', [
    ('int fb_sync(FbHandle h);', 'int fb_sync(FbHandle h);\nint fb_new(FbHandle h, size_t n);', 'int fb_new(FbHandle h, size_t n);'),
    ('long long fb_launch_count(FbHandle h);', 'unsigned fb_launch_count(FbHandle h);', 'unsigned fb_launch_count(FbHandle h);'),
    ('int fb_sync(FbHandle h);', 'int fb_sync();', 'int fb_sync();'),
    ('float fovy_deg;', 'short fovy_deg;', 'short fovy_deg;'),
    ('int32_t n_cam;', 'int32_t** n_cam;', 'int32_t** n_cam;'),
    ('FB_OBS_SENSOR_NOW = 1,', 'FB_OBS_SENSOR_NOW,', 'FB_OBS_SENSOR_NOW,'),
    ('#define FB_MAXEFC 160', '#define FB_MAXEFC (160)', '#define FB_MAXEFC (160)'),
    ('int fb_sync(FbHandle h);', 'int fb_sync(FbHandle h);\n// a comment', '// a comment'),
])
def test_reader_refuses_what_it_does_not_know(old, new, line):
    """a construct or type outside the reader's subset of C is an error naming its line, never a guess"""
    hdr = open(abi.HEADER).read()
    assert old in hdr
    bad = hdr.replace(old, new, 1)
    lineno = bad[:bad.index(line)].count('\n') + 1
    with pytest.raises(stepper.StepperError, match=rf'^h\.h:{lineno}: .*{re.escape(line)}'):
        abi.parse(bad, 'h.h')


def test_product_path_has_no_cpu_fallback(tmp_path):
    with pytest.raises(stepper.StepperError):
        stepper.load_library(str(tmp_path / 'missing.so'))
    with pytest.raises(stepper.StepperError):
        abi.read(str(tmp_path / 'missing.h'))
    # the product package never references the oracle or the emulation build
    pkg = os.path.join(ROOT, 'flybody_b200')
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.h')) and 'compiler' not in dp:
                src = open(os.path.join(dp, f)).read()
                assert 'fly_oracle' not in src and 'libflyoracle' not in src, f
                if f.endswith('.py'):
                    assert 'libfb_emu' not in src, f
