"""The one status-to-kind table every asynchronous call's finish kernel uses (async_kind_of, through pco_b200_debug_async_kind), without a
GPU: each PCO_B200_ASYNC_* code gets the kind its comment in include/pco_b200.h states, and each chunk status the kind status_to_error
gives it."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = {"OK": 0, "CORRUPTION": 1, "INSUFFICIENT_DATA": 2, "INVALID_ARGUMENT": 3, "IO": 4, "UNSUPPORTED": 7}


def _read(*path):
    with open(os.path.join(ROOT, *path)) as f:
        return f.read()


@pytest.fixture(scope="module")
def kind_of():
    from pcodec_b200 import _lib

    L = _lib.bind("_async_kind_ready", pco_b200_debug_async_kind=[C.c_uint])
    L.pco_b200_debug_async_kind.restype = C.c_uint
    return lambda st: L.pco_b200_debug_async_kind(C.c_uint(st))


def _documented_codes():
    """{name: (code, kind)} of every PCO_B200_ASYNC_* code, the kind the last one named in parentheses in its comment."""
    codes = {}
    for name, code, comment in re.findall(r"(PCO_B200_ASYNC_\w+)\s*=\s*(0x[0-9a-fA-F]+)[^/]*/\*(.*?)\*/", _read("include", "pco_b200.h"), flags=re.S):
        kinds = re.findall(r"\((?:PCO_B200_)?(" + "|".join(KINDS) + r")\)", comment)
        assert kinds, f"{name}: no kind in its comment"
        codes[name] = (int(code, 16), KINDS[kinds[-1]])
    return codes


def test_every_async_code_has_the_kind_its_comment_states(kind_of):
    codes = _documented_codes()
    values = sorted(c for c, _ in codes.values())
    assert values == list(range(0x101, 0x120)), "the codes are 0x101 .. 0x11f, each once"
    wrong = {name: (kind_of(code), kind) for name, (code, kind) in codes.items() if kind_of(code) != kind}
    assert not wrong, wrong


def test_chunk_statuses_have_the_kinds_status_to_error_gives(kind_of):
    statuses = {name: int(v) for name, v in re.findall(r"\b(ST_[A-Z_]+) = (\d+)", _read("pcodec_b200", "csrc", "codec_common.cuh"))}
    assert {"ST_OK", "ST_CORRUPTION", "ST_UNSUPPORTED", "ST_TERMINATOR"} <= set(statuses)
    body = re.search(r"inline PcoB200Error status_to_error\(.*?\n}\n", _read("pcodec_b200", "csrc", "host_common.hpp"), flags=re.S).group(0)
    cases = {name: KINDS[kind] for name, kind in re.findall(r"case (ST_\w+):\s*return (?:fail\()?PCO_B200_(\w+)", body)}
    default = KINDS[re.search(r"default: return fail\(PCO_B200_(\w+)", body).group(1)]
    assert cases["ST_OK"] == 0 and cases["ST_UNSUPPORTED"] == 7
    for name, st in statuses.items():
        assert kind_of(st) == cases.get(name, default), name
    for st in (4, 5, 6, 8, 99, 103, 0x100, 0x120, 0xFFFFFFFF):  # no status: the catch-all kind
        assert kind_of(st) == default, st
