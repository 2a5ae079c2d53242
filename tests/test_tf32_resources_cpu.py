"""Single-pass TF32 mode (no GPU): the dedicated kernels in the built library and the mode setting.

conv_tf32_kernel, wgrad_tf32_kernel and wgrad2_tf32_kernel are the single-product twins of conv_tc_kernel, wgrad_tc_kernel
and wgrad2_tc_kernel: every template instantiation of the parity kernels exists once more, fits the 128 registers a
512-thread CTA gets per thread without a stack frame, and reallocates registers between its warpgroups exactly as its
parity twin does (setmaxnreg in the conv engine, none in the two wgrad kernels).  bts_b200.set_precision and
BTS_B200_PRECISION accept "fp32" and "tf32" only."""
import functools
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bts_b200", "libbts_b200.so")

# mangled-name prefix of each single-pass kernel -> (its parity twin, instantiations)
KERNELS = {
    "16conv_tf32_kernel": ("14conv_tc_kernel", 24),       # PRE 0-3 x source mode 0-2 x vector loads
    "17wgrad_tf32_kernel": ("15wgrad_tc_kernel", 16),     # PRE 0-3 x up-sample x vector loads
    "18wgrad2_tf32_kernel": ("16wgrad2_tc_kernel", 24),   # PRE 0-3 x (landing ring: up-sample; loads: up-sample x vector)
}


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe:
        return exe
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.isfile(os.path.join(home, "bin", "cuobjdump")):
            return os.path.join(home, "bin", "cuobjdump")
    return None


@functools.lru_cache(maxsize=None)
def _dump(flag):
    """cuobjdump output of the built library (one run per flag: the SASS of every kernel takes a while)"""
    if not os.path.isfile(LIB):
        pytest.skip("libbts_b200.so is not built")
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    return subprocess.run([exe, flag, LIB], capture_output=True, text=True, check=True).stdout


def _family(name):
    for k, (twin, _) in KERNELS.items():
        if k in name:
            return k
        if twin in name:
            return twin
    return None


def _resources():
    """{kernel family: {mangled name: (REG, STACK)}}"""
    res = {}
    name = None
    for line in _dump("-res-usage").splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name and _family(name):
            res.setdefault(_family(name), {})[name] = (int(m.group(1)), int(m.group(2)))
        name = None
    return res


def _reallocations():
    """{kernel family: {mangled name: set of USETMAXREG forms in its SASS}}"""
    out = {}
    fam = name = None
    for line in _dump("-sass").splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            fam = _family(name)
            if fam:
                out.setdefault(fam, {})[name] = set()
            continue
        if fam:
            m = re.search(r"USETMAXREG\.(\w+)", line)
            if m:
                out[fam][name].add(m.group(1))
    return out


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_every_parity_instantiation_has_a_single_pass_twin(kernel):
    res = _resources()
    twin, n = KERNELS[kernel]
    assert len(res.get(kernel, {})) == n, "expected %d %s instantiations, found %d" % (n, kernel, len(res.get(kernel, {})))
    assert len(res.get(twin, {})) == n
    # the same template arguments: the names differ in the kernel's identifier only
    strip = lambda names, k: sorted(s.split(k, 1)[1] for s in names)
    assert strip(res[kernel], kernel) == strip(res[twin], twin)


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_single_pass_kernels_fit_registers_without_spills(kernel):
    res = _resources().get(kernel, {})
    assert res, "no %s in the library" % kernel
    bad = {k: v for k, v in res.items() if v[0] > 128 or v[1] != 0}
    assert not bad, "%s instantiations over 128 registers or with a stack frame (REG, STACK): %s" % (kernel, bad)


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_single_pass_kernels_reallocate_registers_like_their_twins(kernel):
    re_ = _reallocations()
    twin = KERNELS[kernel][0]
    mine = {n.split(kernel, 1)[1]: ops for n, ops in re_.get(kernel, {}).items()}
    theirs = {n.split(twin, 1)[1]: ops for n, ops in re_.get(twin, {}).items()}
    assert mine and mine == theirs
    if kernel == "16conv_tf32_kernel":
        assert all({"TRY_ALLOC", "DEALLOC"} <= ops for ops in mine.values()), mine


def test_set_precision_returns_the_previous_mode_and_rejects_unknown_ones():
    import bts_b200
    from bts_b200 import conv
    start = bts_b200.get_precision()
    try:
        assert bts_b200.set_precision("tf32") == start
        assert conv._engine_precision(None) == 1 and conv._engine_precision(0) == 0
        assert bts_b200.set_precision("fp32") == "tf32"
        assert conv._engine_precision(None) == 0 and conv._engine_precision(1) == 1
        for bad in ("TF32", "fp16", "bf16", "", None, 1, 0):
            with pytest.raises(ValueError):
                bts_b200.set_precision(bad)
        assert bts_b200.get_precision() == "fp32"
    finally:
        bts_b200.set_precision(start)


def _import_with(value):
    env = dict(os.environ)
    env.pop("BTS_B200_PRECISION", None)
    if value is not None:
        env["BTS_B200_PRECISION"] = value
    code = "import sys; sys.path.insert(0, %r); import bts_b200; print(bts_b200.get_precision())" % ROOT
    return subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)


@pytest.mark.parametrize("value,mode", [(None, "fp32"), ("fp32", "fp32"), ("tf32", "tf32")])
def test_environment_sets_the_initial_mode(value, mode):
    r = _import_with(value)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip().splitlines()[-1] == mode


def test_an_invalid_environment_value_fails_the_import():
    r = _import_with("bogus")
    assert r.returncode != 0
    assert "BTS_B200_PRECISION" in r.stderr and "bogus" in r.stderr
