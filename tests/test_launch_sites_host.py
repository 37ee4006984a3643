"""CPU: every kernel launch, launch count and dynamic shared-memory opt-in in csrc/ goes through the one helper in
common.cuh / common.cu, so each launch is checked right after it is made and counted exactly once."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sam_road_b200", "csrc")


def _code(name):
    """The source of csrc/<name> without comments."""
    src = open(os.path.join(CSRC, name)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _sources():
    names = sorted(n for n in os.listdir(CSRC) if n.endswith((".cu", ".cuh", ".h")))
    assert "common.cuh" in names and "common.cu" in names and len(names) > 10
    return {n: _code(n) for n in names}


def _body(code, signature):
    """The text of the function whose definition starts with `signature`, up to its closing brace."""
    start = code.index(signature)
    depth, i = 0, code.index("{", start)
    while True:
        depth += {"{": 1, "}": -1}.get(code[i], 0)
        if depth == 0:
            return code[start:i + 1]
        i += 1


def _sites(sources, token):
    return {n: code.count(token) for n, code in sources.items() if token in code}


def test_kernels_launch_only_through_srb_launch():
    sources = _sources()
    assert _sites(sources, "<<<") == {"common.cuh": 1}
    assert "<<<" in _body(sources["common.cuh"], "int launch(")


def test_dynamic_smem_opt_in_only_through_allow_dynamic_smem():
    sources = _sources()
    assert _sites(sources, "cudaFuncSetAttribute") == {"common.cu": 1}
    assert "cudaFuncSetAttribute" in _body(sources["common.cu"], "int allow_dynamic_smem(const void* kernel")


def test_launch_count_and_srb_try_live_in_common():
    sources = _sources()
    assert set(_sites(sources, "note_launch(")) == {"common.cu"}
    assert _sites(sources, "#define SRB_TRY") == {"common.cuh": 1}
