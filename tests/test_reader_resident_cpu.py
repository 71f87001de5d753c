"""CPU checks of device-resident reading: the new entries are declared, exported and bound; their kernels compile for sm_90a without
spills; the device queue's word order (numpy.random.Philox.random_raw: counter bumped before each 4-word block) restated in numpy;
the host queue's state_dict round trip; the refusal of empty and short files."""
import os
import re
import sys

import numpy as np
import pytest

import reader_train_oracle as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "hand3d_b200", "build", "nvcc.log")
NEW = ("h3d_reader_next_serials", "h3d_decode_records_gather")


def test_new_entries_declared_exported_and_bound():
    from hand3d_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "hand3d_b200.h")).read()
    lib = _lib.load()
    assert lib.h3d_version() >= 102
    for n in NEW:
        assert re.search(r"H3D_API\s+int\s+%s\s*\(" % n, hdr), n
        assert hasattr(lib, n) and n in _lib.SIGNATURES, n
    for name, value in (("CAPACITY", 100), ("STATE_COUNT", 0), ("STATE_NEXT", 1), ("STATE_SLOTS", 2), ("STATE_WORDS", 102),
                        ("MAX_GATHER", 4096)):
        m = re.search(r"#define H3D_READER_%s (\d+)" % ("QUEUE_" + name if name == "CAPACITY" else name), hdr)
        assert m and int(m.group(1)) == value == getattr(_lib, "READER_" + ("QUEUE_" + name if name == "CAPACITY" else name)), name


def test_resident_reader_kernels_compile_for_sm90a_without_spills():
    if not os.path.exists(LOG):
        pytest.skip("no build log: run python -m hand3d_b200.build first")
    found = {}
    for sec in open(LOG).read().split("Compiling entry function")[1:]:
        name = sec.split("'")[1]
        for k in ("decode_records_kernelILb1E", "decode_records_kernelILb0E", "next_serials_kernel"):
            if k in name:
                assert "for 'sm_90a'" in sec, name
                found[k] = int(re.search(r"(\d+) bytes spill stores", sec).group(1))
    assert sorted(found) == ["decode_records_kernelILb0E", "decode_records_kernelILb1E", "next_serials_kernel"], found
    assert all(v == 0 for v in found.values()), found


@pytest.mark.parametrize("seed", [0, 1, 2 ** 64 - 1, 20171003])
def test_device_word_order_is_numpy_random_raw(seed):
    """Word n = word (n mod 4) of Philox4x64-10 at counter (n // 4 + 1, 0, 0, 0), as next_serials_kernel draws it."""
    n = np.arange(1001, dtype=np.uint64)
    ctr = np.zeros((n.size, 4), np.uint64)
    ctr[:, 0] = n // np.uint64(4) + np.uint64(1)
    words = A.philox4x64_10(ctr, np.broadcast_to(np.array([seed, A.STREAM_SHUFFLE], np.uint64), (n.size, 2)))
    got = words[np.arange(n.size), (n % np.uint64(4)).astype(np.int64)]
    np.testing.assert_array_equal(got, np.random.Philox(key=np.array([seed, A.STREAM_SHUFFLE], np.uint64)).random_raw(n.size))


@pytest.mark.parametrize("first", [0, 1, 2, 3, 4, 37, 250])
def test_host_queue_state_round_trip(first):
    from hand3d_b200.data.BinaryDbReader import _ShuffleQueue
    q = _ShuffleQueue(99)
    q.take(first)
    st = q.state_dict()
    assert st["count"] == first and st["shuffle"] and len(st["slots"]) == 100
    want = q.take(123)
    r = _ShuffleQueue(99)
    r.load_state_dict(st)
    assert r.take(123) == want
    np.testing.assert_array_equal(want, A.shuffle_serials(99, first + 123)[first:])


def test_in_order_reader_state_and_mode_checks(tmp_path):
    sys.path.insert(0, ROOT)
    from examples._synthetic_db import fake_rhd
    from hand3d_b200.data.BinaryDbReader import BinaryDbReader
    p = tmp_path / "rhd.bin"
    p.write_bytes(fake_rhd(3))
    rd = BinaryDbReader(mode="training", shuffle=False, path_to_db=str(p), seed=1)
    assert rd.device_bytes == 0 and rd.state_dict() == {"shuffle": False, "count": 0, "next": 0, "slots": None}
    rd.load_state_dict({"shuffle": False, "count": 7, "next": 7, "slots": None})
    assert rd._next_serial == 7
    sh = BinaryDbReader(mode="training", shuffle=True, path_to_db=str(p), seed=1)
    with pytest.raises(ValueError, match="cannot resume"):
        sh.load_state_dict(rd.state_dict())


@pytest.mark.parametrize("size", [0, 1, 410519])
def test_resident_reader_refuses_empty_and_short_files(tmp_path, size):
    from hand3d_b200.data.BinaryDbReader import BinaryDbReader, BinaryDbReaderSTB
    p = tmp_path / "short.bin"
    p.write_bytes(b"\0" * size)
    with pytest.raises(ValueError, match="less than one 410520-byte record"):
        BinaryDbReader(mode="training", path_to_db=str(p), device_resident=True)
    with pytest.raises(ValueError, match="less than one 922104-byte record"):
        BinaryDbReaderSTB(mode="evaluation", shuffle=False, path_to_db=str(p), device_resident=True)
