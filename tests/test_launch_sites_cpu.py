"""Launch sites of the CUDA sources (open_vins_b200/csrc), read statically.

Every kernel is launched through ovb_launch (ovb_internal.cuh), which counts the launch, brackets it with profile events
while profiling and sets the programmatic-dependent-launch (PDL) attribute otherwise. So:
  - no `<<< >>>` launch and no cudaLaunchKernelEx outside ovb_internal.cuh;
  - no hand-kept launch count (`n_launch +=`, `n_launch++` and the like);
  - every __global__ body reaches griddepcontrol.wait, through OVB_PDL_ENTER() or its own asm, directly or in a function
    it calls: a kernel launched with the PDL attribute that never waits races with the kernel before it.
"""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open_vins_b200", "csrc")
SOURCES = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh")))
WAIT = re.compile(r"OVB_PDL_ENTER\(\)|griddepcontrol\.wait")


def _code(name):
    """the file without comments (string literals stay: the asm of griddepcontrol.wait is one)"""
    with open(os.path.join(CSRC, name)) as f:
        s = f.read()
    return re.sub(r'"(?:\\.|[^"\\\n])*"|//[^\n]*|/\*.*?\*/', lambda m: m.group(0) if m.group(0).startswith('"') else " ", s, flags=re.S)


def _functions(code):
    """(name, is_global, body) of every function definition"""
    out = []
    for m in re.finditer(r"\b([A-Za-z_]\w*)\s*\(", code):
        name = m.group(1)
        if name in ("if", "for", "while", "switch", "return", "sizeof", "defined", "__launch_bounds__", "decltype", "static_assert"):
            continue
        # the parameter list, then an optional qualifier, then the body's brace
        depth, i = 0, m.end() - 1
        while i < len(code):
            depth += {"(": 1, ")": -1}.get(code[i], 0)
            i += 1
            if depth == 0:
                break
        tail = re.match(r"\s*(?:const\s*)?(?:noexcept\s*)?\{", code[i:])
        if not tail:
            continue
        start = i + tail.end() - 1
        depth, j = 0, start
        while j < len(code):
            depth += {"{": 1, "}": -1}.get(code[j], 0)
            j += 1
            if depth == 0:
                break
        head = code[max(0, code.rfind(";", 0, m.start()), code.rfind("}", 0, m.start())):m.start()]
        out.append((name, "__global__" in head, code[start:j]))
    return out


@pytest.fixture(scope="module")
def code():
    return {f: _code(f) for f in SOURCES}


def test_sources_found(code):
    assert "ovb_internal.cuh" in code and "ovb_api.cu" in code


def test_no_triple_chevron_launch(code):
    bad = [(f, c[m.start():m.start() + 60]) for f, c in code.items() for m in re.finditer(r"<<<", c)]
    assert not bad, bad


def test_cudaLaunchKernelEx_only_in_ovb_launch(code):
    sites = {f: len(re.findall(r"\bcudaLaunchKernelEx\b", c)) for f, c in code.items()}
    assert sites.pop("ovb_internal.cuh") == 1
    assert not any(sites.values()), sites


def test_no_hand_kept_launch_count(code):
    pat = re.compile(r"\bn_launch\s*(?:\+=|-=|\+\+)|\+\+\s*ctx->n_launch\b")
    sites = [(f, c[m.start():m.start() + 40]) for f, c in code.items() for m in pat.finditer(c)]
    assert [f for f, _ in sites] == ["ovb_internal.cuh"], sites  # the one count is ovb_launch's own


def test_every_kernel_waits_on_its_predecessor(code):
    funcs = [fn for c in code.values() for fn in _functions(c)]
    bodies = {}
    for name, _, body in funcs:
        bodies.setdefault(name, []).append(body)
    memo = {}

    def waits(body, seen):
        calls = set(re.findall(r"\b([A-Za-z_]\w*)\s*(?:<[^;{}()]*>)?\s*\(", body))
        return bool(WAIT.search(body)) or any(reaches(c, seen) for c in calls - seen)

    def reaches(name, seen):
        """some definition of `name` (an overload or template) reaches the wait"""
        if name not in memo:
            memo[name] = name in bodies and any(waits(b, seen | {name}) for b in bodies[name])
        return memo[name]

    kernels = [(name, body) for name, g, body in funcs if g]
    assert len(kernels) >= 40, [k for k, _ in kernels]  # the parser found the kernels
    missing = sorted({name for name, body in kernels if not waits(body, frozenset({name}))})
    assert not missing, missing
