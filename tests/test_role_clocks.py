"""The role clocks of the composite kernels (-DF3DGS_ROLE_CLOCKS, composite_common.cuh) and the tool that reads them
(tools/time_composite_roles.py).

CPU: the tool names the counters in the order of `enum RoleClock`, and a variant build lands beside, not in, the package.
GPU: the instrumented library builds into a directory of its own, runs a small scene forward + backward, and every wait
it reports is a share of its role's loop between 0 and 100 %.
"""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "tools", "time_composite_roles.py")
HEADER = os.path.join(ROOT, "feature-3dgs_b200", "csrc", "composite_common.cuh")


def _tool_constant(name):
    """A module-level tuple of the tool, without importing it (it imports torch and rewires sys.path)."""
    import ast

    for node in ast.parse(open(TOOL).read()).body:
        if isinstance(node, ast.Assign) and node.targets[0].id == name:
            return ast.literal_eval(node.value)
    raise KeyError(name)


def test_tool_names_the_counters_in_enum_order():
    src = open(HEADER).read()
    body = re.search(r"enum RoleClock \{(.*?)\};", src, re.S).group(1)
    names = re.findall(r"\bkClk([A-Za-z]+)", re.sub(r"//.*", "", body))
    snake = ["_".join(w.lower() for w in re.findall(r"[A-Z][a-z]*", n)) for n in names]
    assert tuple(snake) == _tool_constant("CLOCKS")
    used = {k for _, loop, waits in _tool_constant("ROWS") for k in (loop, *[w[1] for w in waits])}
    assert used == set(snake)


def test_variant_build_paths_are_outside_the_package(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
    try:
        import build as native_build
    finally:
        sys.path.pop(0)
    assert native_build._paths(native_build.PKG) == (native_build.OBJ, native_build.LIB, native_build.EXT)
    for p in native_build._paths(str(tmp_path)):
        assert p.startswith(str(tmp_path)) and not p.startswith(native_build.PKG)


@pytest.mark.gpu
def test_role_clock_build_reports_shares_of_each_loop(tmp_path):
    r = subprocess.run([sys.executable, TOOL, "--config", "small128", "--views", "2", "--build-dir", str(tmp_path)],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stdout)
    kernels = re.split(r"^composite_", r.stdout, flags=re.M)[1:]
    assert [k.split()[0] for k in kernels] == ["fwd", "bwd"]
    roles = {"fwd": ["producer", "alpha warps", "feature warps"], "bwd": ["producer", "alpha warps"]}
    for k in kernels:
        rows = re.findall(r"^  (\S.*?)\s+loop\s+([\d.]+) Mcycles \| (.*)$", k, flags=re.M)
        assert [row[0] for row in rows] == roles[k.split()[0]]
        for _, loop, cells in rows:
            assert float(loop) > 0
            shares = [float(x) for x in re.findall(r"([\d.]+) %", cells)]
            assert shares and all(0.0 <= x <= 100.0 for x in shares), cells
    assert os.path.exists(os.path.join(str(tmp_path), "libf3dgs_b200.so"))  # the variant, beside the normal build
