"""CPU tests of the direct glass reader (xapiand_b200/csrc/xgm_glass.cu): `xgm_glass_export_flat` parses
iamglass + postlist.glass itself and must produce, byte for byte, the file `ref_runner export` writes by walking
the same database through the reference's public iterators (allterms / postlist / doclength / valuestream).
tests/golden/glass_300 is a small database the reference wrote, stored with the digest of the reference's export of
it, so that the comparison also runs where the compiled reference is not available."""
import filecmp
import hashlib
import json
import os
import shutil
import subprocess
import tempfile
import ctypes

import pytest

from oracle import oracle as O
from xapiand_b200 import xgm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
needs_reference = pytest.mark.skipif(not O.have_reference(), reason="compiled reference (oracle/_ref) not built")


@needs_reference
@pytest.mark.parametrize("ndocs,vocab,kw", [(3000, 500, {}), (20000, 3000, dict(mvalues=True, sparse=(7, 5))),
                                            (40000, 200, dict(values=True)), (1, 5, {})])
def test_direct_reader_equals_the_reference_iterators(ndocs, vocab, kw):
    tmp = tempfile.mkdtemp(prefix="xgm_glass_")
    try:
        db = os.path.join(tmp, "db")
        O.ref_build(db, ndocs, vocab, seed=5, **kw)
        subprocess.check_call([O.REF_RUNNER, "export", "--db", db, "--out", os.path.join(tmp, "ref.flat")],
                              stdout=subprocess.DEVNULL)
        st = xgm.lib().xgm_glass_export_flat(db.encode(), os.path.join(tmp, "mine.flat").encode())
        assert st == 0, xgm.lib().xgm_last_error()
        assert filecmp.cmp(os.path.join(tmp, "ref.flat"), os.path.join(tmp, "mine.flat"), shallow=False)
        rev, dc, last = ctypes.c_uint64(), ctypes.c_uint32(), ctypes.c_uint32()
        assert xgm.lib().xgm_glass_revision(db.encode(), ctypes.byref(rev), ctypes.byref(dc), ctypes.byref(last)) == 0
        assert (dc.value, last.value) == (ndocs, ndocs) and rev.value >= 1
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def test_direct_reader_equals_the_stored_reference_export(tmp_path):
    with open(os.path.join(GOLDEN, "glass_300.json")) as f:
        fx = json.load(f)
    db = os.path.join(GOLDEN, "glass_300")
    mine = tmp_path / "mine.flat"
    st = xgm.lib().xgm_glass_export_flat(db.encode(), str(mine).encode())
    assert st == 0, xgm.lib().xgm_last_error()
    data = mine.read_bytes()
    assert len(data) == fx["ref_export_bytes"]
    assert hashlib.sha256(data).hexdigest() == fx["ref_export_sha256"]
    rev, dc, last = ctypes.c_uint64(), ctypes.c_uint32(), ctypes.c_uint32()
    assert xgm.lib().xgm_glass_revision(db.encode(), ctypes.byref(rev), ctypes.byref(dc), ctypes.byref(last)) == 0
    assert (dc.value, last.value) == (fx["ndocs"], fx["ndocs"]) and rev.value >= 1


def test_reader_rejects_what_is_not_a_glass_database(tmp_path):
    assert xgm.lib().xgm_glass_export_flat(str(tmp_path).encode(), str(tmp_path / "x").encode()) == xgm.E_IO
    (tmp_path / "iamglass").write_bytes(b"not a version file" * 4)
    assert xgm.lib().xgm_glass_export_flat(str(tmp_path).encode(), str(tmp_path / "x").encode()) == xgm.E_IO
