"""Every CUDA allocation, event and library-created stream of the engine has one owner (csrc/owner.cuh).  Raw
allocate / free / create / destroy calls are allowed only inside that header, in table_mem / table_free (table
placement: cudaMalloc or shareable VMM memory that peers map) and for h->stream, which ctr_set_stream can replace
with a caller's stream.  Anything else would need a hand-kept free list again."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "go-ctr_b200", "csrc")

RAW = re.compile(r"\bcuda(Malloc|MallocHost|HostAlloc|Free|FreeHost|EventDestroy|StreamDestroy|EventCreate\w*|StreamCreate\w*)\(")
STREAM_CALL = re.compile(RAW.pattern + r"&?h->stream\b")
FUNC = re.compile(r"^[A-Za-z].*?\b([A-Za-z_]\w*)\s*\([^;]*\)\s*(const\s*)?\{")
TABLE_FUNCS = {"table_mem", "table_free"}


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, f.read().splitlines()


def test_raw_cuda_resource_calls_only_in_their_owners():
    stray = []
    for name, lines in _sources():
        if name == "owner.cuh":
            continue
        func = None
        for no, line in enumerate(lines, 1):
            m = FUNC.match(line)
            if m:
                func = m.group(1)
            if not RAW.search(line):
                continue
            if func in TABLE_FUNCS:
                continue
            if all(STREAM_CALL.match(line, m.start()) for m in RAW.finditer(line)):
                continue
            stray.append("%s:%d (%s): %s" % (name, no, func, line.strip()))
    assert not stray, "raw CUDA resource calls outside owner.cuh:\n" + "\n".join(stray)


def test_no_goto_cleanup():
    gotos = ["%s:%d" % (name, no) for name, lines in _sources() for no, line in enumerate(lines, 1)
             if re.search(r"\bgoto\b", line.split("//")[0])]
    assert not gotos, gotos
