"""CPU check of the host side's ownership rules (kimera_semantics_b200/csrc/ksg_api.cu): every device / pinned allocation, stream and
event is made and released by the one owner type (`Resources`), so that an integrator, or a call's temporaries, cannot leak what
they made; the development knobs are read from the environment in one place; CUDA errors are reported through the handle."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
API = os.path.join(ROOT, "kimera_semantics_b200", "csrc", "ksg_api.cu")

RESOURCE_CALLS = re.compile(r"\b(cudaMalloc|cudaMallocHost|cudaFree|cudaFreeHost|cudaStreamCreate\w*|cudaStreamDestroy|"
                            r"cudaEventCreate\w*|cudaEventDestroy)\s*\(")


def source():
    text = open(API).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def block(text, header):
    """(start, end) of the brace-delimited body that follows the first match of `header`."""
    m = re.search(header, text)
    assert m, header
    i = text.index("{", m.end() - 1)
    depth = 0
    for j in range(i, len(text)):
        depth += {"{": 1, "}": -1}.get(text[j], 0)
        if depth == 0:
            return m.start(), j + 1
    raise AssertionError(f"unbalanced braces after {header}")


def outside(text, header):
    a, b = block(text, header)
    return text[:a] + text[b:], text[a:b]


def test_resources_are_made_and_released_only_by_the_owner():
    rest, owner = outside(source(), r"\bclass Resources\s*\{")
    assert RESOURCE_CALLS.search(owner), "the owner type makes the allocations"
    stray = sorted({m.group(1) for m in RESOURCE_CALLS.finditer(rest)})
    assert not stray, f"made or released outside Resources: {stray}"


def test_environment_is_read_only_by_read_knobs():
    rest, knobs = outside(source(), r"\bKnobs\s+read_knobs\s*\(\s*\)\s*\{")
    assert "getenv" in knobs
    assert "getenv" not in rest


def test_no_local_fail_lambdas():
    assert not re.search(r"\bauto\s+fail\s*=", source())
