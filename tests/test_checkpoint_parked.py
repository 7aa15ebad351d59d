"""Checkpoints whose maps hold parked entries (format version 2, checkpoint.h, DESIGN.md §13): an independent Python writer of the
version-2 framing and of the parked lists of the engine section, and the reader's checks of those lists before any CUDA call."""
import struct

import numpy as np
import pytest

import test_checkpoint as tc

MARKER = b"LAMAPARK"
BASE = 1321122 - 4   # the window of tc.pf_payload: 8 x 8 patches from (BASE, BASE)
SLOTS = 2 * (4096 + 128)


def v2_file(lists, refcount=(3, 2), P=3):
    """tc.pf_payload's PFSlam2D with parked lists {(particle, kind): [(px, py, entry), ...]} between its directories and its slots"""
    b = tc.pf_payload(P=P, refcount=refcount)
    lens = [len(lists.get((p, k), [])) for p in range(P) for k in range(2)]
    parked = struct.pack(f"<{len(lens)}I", *lens)
    for p in range(P):
        for k in range(2):
            for e in lists.get((p, k), []):
                parked += struct.pack("<3i", *e)
    return tc.frame(MARKER + b[:-SLOTS] + parked + b[-SLOTS:], version=2)


FAR = BASE + 20
GOOD = {(1, 0): [(FAR, BASE, 1), (FAR + 1, BASE, 1 | tc.OWN)]}   # particle 1's occupancy map parks two patches of slot 1


def test_valid_parked_file_is_read(api, tmp_path):
    p = tmp_path / "ok.ckpt"
    p.write_bytes(v2_file(GOOD, refcount=(3, 3)))
    tc._expect_valid(api, p)


@pytest.mark.parametrize("name,lists,refcount,msg", [
    ("unsorted", {(1, 0): [(FAR + 1, BASE, 1), (FAR, BASE, 1)]}, (3, 3), "not strictly sorted"),
    ("duplicate", {(1, 0): [(FAR, BASE, 1), (FAR, BASE, 1)]}, (3, 3), "not strictly sorted"),
    ("inside the window", {(1, 0): [(BASE + 2, BASE + 3, 1)]}, (3, 2), "inside the saved window"),
    ("slot past K", {(1, 0): [(FAR, BASE, 2)]}, (3, 1), "past the saved slots"),
    ("unknown flag", {(1, 0): [(FAR, BASE, 1 | (1 << 27))]}, (3, 2), "unknown flag bits"),
    ("absent entry", {(1, 0): [(FAR, BASE, -1)]}, (3, 1), "unknown flag bits"),
    ("reference count", {(1, 0): [(FAR, BASE, 1)]}, (3, 1), "reference count differs"),
])
def test_malformed_parked_lists_are_refused(api, tmp_path, name, lists, refcount, msg):
    p = tmp_path / "bad.ckpt"
    p.write_bytes(v2_file(lists, refcount=refcount))
    tc._expect_bad(api, p, msg=msg)


def test_version_2_needs_its_marker_and_version_1_reads_no_lists(api, tmp_path):
    # a version-1 body framed as version 2 is refused, naming the version
    p = tmp_path / "v1as2.ckpt"
    p.write_bytes(tc.frame(tc.pf_payload(), version=2))
    tc._expect_bad(api, p, msg="version 2")
    # a version-2 body framed as version 1 does not parse either
    b = v2_file(GOOD, refcount=(3, 3))
    p.write_bytes(tc.frame(b[tc.HDR:], version=1))
    tc._expect_bad(api, p)
    # and a truncated parked section is refused
    body = b[tc.HDR:]
    p.write_bytes(tc.frame(body[:len(body) - SLOTS - 4] + body[len(body) - SLOTS:], version=2))
    tc._expect_bad(api, p)


def test_sharded_load_refuses_parked_state(api, tmp_path):
    import ctypes as C
    p = tmp_path / "ok.ckpt"
    p.write_bytes(v2_file(GOOD, refcount=(3, 3)))
    L = api.lib()
    paths = (C.c_char_p * 1)(str(p).encode())
    h = C.c_void_p()
    rc = L.lama_pf_load_state_sharded(paths, 1, 0, 1, None, C.byref(h))
    assert rc == tc.ERR_ARG and not h.value, (rc, L.lama_last_error())
    assert b"parked" in L.lama_last_error()
