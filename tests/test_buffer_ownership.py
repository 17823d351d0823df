"""Every device and pinned host allocation of the library has one owner: DeviceBuffer / PinnedBuffer (csrc/buffers.h)
allocate and free it.  A raw cudaMalloc or cudaFree elsewhere is a lifetime written by hand again, with a capacity
to keep in step and a destroy list to extend, and a leak when either is forgotten."""
import os
import re

import helpers

CSRC = os.path.join(helpers.ROOT, "jsmpeg_b200", "csrc")
RAW = re.compile(r"\bcuda(?:Malloc|MallocHost|HostAlloc|Free|FreeHost)\b")


def raw_calls(path):
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    return sorted(set(RAW.findall(text)))


def test_raw_allocations_live_only_in_the_buffer_type():
    found = {f: raw_calls(os.path.join(CSRC, f)) for f in sorted(os.listdir(CSRC))}
    found = {f: calls for f, calls in found.items() if calls}
    assert found.pop("buffers.h") == ["cudaFree", "cudaFreeHost", "cudaHostAlloc", "cudaMalloc"]
    # the per-device multi-symbol table (parse.cu) is kept for the life of the process by design
    assert found == {"parse.cu": ["cudaMalloc"]}
