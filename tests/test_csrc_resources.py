"""CPU-side source check of csrc/: device memory, streams and events are held by the owners in common.cuh (Scratch, Stream, Event).

An owner frees what it holds on every path out of a function, error returns included, and a table built in a local owner reaches a
cache only once it is complete.  A raw allocation or create call elsewhere needs a hand-written release on each of those paths,
which is how leaks and cache entries for tables that were never built come about, so such calls are refused outside common.cuh.
The one exception is zk_dev_alloc / zk_dev_free: by the API's contract, that memory belongs to the caller."""
import re

from test_csrc_streams import sources

RAW = re.compile(r"\b(cudaMalloc\w*|cudaHostAlloc|cudaFree\w*|cudaStreamCreate\w*|cudaStreamDestroy|cudaEventCreate\w*|cudaEventDestroy)\s*\(")
OWNERS = "common.cuh"
CALLER_OWNED = ("api.cu", ("zk_dev_alloc", "zk_dev_free"))   # file, functions whose memory the caller frees


def function_span(src: str, name: str) -> tuple:
    """[start, end) of the definition of function `name` in src: from its name to its closing brace"""
    m = re.search(r"\b" + name + r"\s*\([^;{]*\)\s*\{", src)
    assert m, f"no definition of {name}"
    depth = 0
    for i in range(m.end() - 1, len(src)):
        depth += {"{": 1, "}": -1}.get(src[i], 0)
        if depth == 0:
            return m.start(), i + 1
    raise AssertionError(f"unbalanced braces in {name}")


def raw_calls():
    """(file, line, call) of every raw allocation, free, create or destroy outside the owners and the caller-owned memory"""
    for name, src in sources():
        if name == OWNERS:
            continue
        spans = [function_span(src, f) for f in CALLER_OWNED[1]] if name == CALLER_OWNED[0] else []
        for m in RAW.finditer(src):
            if not any(a <= m.start() < b for a, b in spans):
                yield name, src.count("\n", 0, m.start()) + 1, m.group(1)


def test_function_span():
    src = "int f(int a) { if (a) { return 1; } return 0; }\nint g(void) { return 2; }"
    a, b = function_span(src, "f")
    assert src[a:b] == "f(int a) { if (a) { return 1; } return 0; }"


def test_the_scan_sees_the_owners_and_the_caller_owned_memory():
    found = {name: [m.group(1) for m in RAW.finditer(src)] for name, src in sources()}
    assert {"cudaMalloc", "cudaFree", "cudaEventDestroy", "cudaStreamDestroy"} <= set(found[OWNERS])
    api = dict(sources())[CALLER_OWNED[0]]
    for f in CALLER_OWNED[1]:
        a, b = function_span(api, f)
        assert RAW.search(api[a:b]), f"{f} no longer allocates or frees: drop it from CALLER_OWNED"


def test_device_memory_streams_and_events_live_in_owners():
    bad = list(raw_calls())
    assert not bad, ("hold device memory in a DevScratch / PinnedScratch, streams in a Stream and events in an Event (common.cuh): "
                     + repr(bad))
