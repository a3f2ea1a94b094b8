"""CPU-side source check of csrc/: every device operation is queued on a stream the context chose.

A caller who hands the context a stream (zk_ctx_set_stream) orders its own work against the library's through that stream alone.
A kernel launched without a stream, or a synchronous cudaMemcpy / cudaMemset, runs on the legacy default stream instead, which a
non-blocking stream (the context's own, or torch's) does not wait for.  Such a call is correct only while something else happens
to synchronise first, so it is refused here."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "proof_systems_b200", "csrc")
LEGACY_STREAMS = {"0", "nullptr", "NULL", "cudaStreamLegacy", "cudaStreamPerThread"}


def sources():
    """(file name, text with comments blanked out) of csrc/*.cu and *.cuh"""
    files = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
    assert len(files) > 10
    out = []
    for f in files:
        src = open(f).read()
        src = re.sub(r"/\*.*?\*/", lambda m: re.sub(r"[^\n]", " ", m.group(0)), src, flags=re.S)
        src = re.sub(r"//[^\n]*", "", src)
        out.append((os.path.basename(f), src))
    return out


def split_top_level(config: str) -> list:
    """the launch parameters of <<<config>>>, split at commas outside parentheses and brackets"""
    parts, depth, cur = [], 0, ""
    for ch in config:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append(cur.strip())
            cur = ""
        else:
            cur += ch
    parts.append(cur.strip())
    return parts


def launches():
    for name, src in sources():
        for m in re.finditer(r"<<<(.*?)>>>", src, flags=re.S):
            yield name, src.count("\n", 0, m.start()) + 1, split_top_level(m.group(1))


def test_split_top_level():
    assert split_top_level("dim3(c, G), ft, (ft / 4) * sizeof(x), st") == ["dim3(c, G)", "ft", "(ft / 4) * sizeof(x)", "st"]
    assert split_top_level("blocks, 128") == ["blocks", "128"]


def test_every_kernel_launch_names_its_stream():
    found = list(launches())
    assert len(found) > 50                       # the scan sees the library's launches
    bad = [(name, line, args) for name, line, args in found if len(args) != 4 or args[3] in LEGACY_STREAMS]
    assert not bad, "launches without an explicit stream (grid, block, shared memory, stream): " + repr(bad)


def test_no_copy_set_or_sync_on_the_legacy_stream():
    bad = []
    for name, src in sources():
        for m in re.finditer(r"\b(cudaMemcpy|cudaMemset|cudaDeviceSynchronize)\s*\(", src):
            bad.append((name, src.count("\n", 0, m.start()) + 1, m.group(1)))
    assert not bad, "use the *Async form on the context's stream (then cudaStreamSynchronize if the host reads the result): " + repr(bad)
