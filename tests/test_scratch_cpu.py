"""Device scratch of the native library, checked on its sources: temporaries inside a C entry
point are gsp::Scratch owners and CUB temporary storage goes through gsp::cub_temp
(csrc/common.cuh), so every return path frees what the entry point allocated."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pygsp_b200",
                    "csrc")


def _sources():
    for root, _, files in os.walk(CSRC):
        for name in sorted(files):
            path = os.path.join(root, name)
            with open(path, encoding="utf-8", errors="replace") as fh:
                yield os.path.relpath(path, CSRC), fh.read()


def test_only_scratch_calls_the_stream_ordered_allocator():
    pattern = re.compile(r"\bcuda(Malloc|Free)Async\b")
    offenders = [name for name, text in _sources()
                 if name != "common.cuh" and pattern.search(text)]
    assert offenders == []


def test_no_cub_size_query_by_hand():
    pattern = re.compile(r"cub::[\w:]+\s*\(\s*nullptr\s*,")
    offenders = [(name, m.group(0)) for name, text in _sources() for m in pattern.finditer(text)]
    assert offenders == []
