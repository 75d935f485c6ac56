"""Host halves of the GPU TFRecord input (tf_repos_b200/tfrecord_device.py): ctr_tfrecord_frame against
tfrecord.read_records(verify_crc=True), and the pass-2 group planner against din_main.index_stream.  No GPU."""
import os
import struct

import numpy as np
import pytest

from tf_repos_b200 import ops
from tf_repos_b200 import tfrecord as tfr
from tf_repos_b200.din_main import index_stream
from tf_repos_b200.tfrecord_device import group_slots, plan_groups


def _file(tmp_path, sizes, seed=0):
    rng = np.random.RandomState(seed)
    recs = [rng.bytes(s) for s in sizes]
    p = os.path.join(tmp_path, "x.tfrecord")
    tfr.write_records(p, recs)
    return p, recs, np.frombuffer(open(p, "rb").read(), dtype=np.uint8)


def _frame_all(buf, chunk):
    """frame buf in chunks of `chunk` bytes the way TFRecordIndex.build does -> record data slices"""
    out, pos = [], 0
    while pos < len(buf):
        want = min(chunk, len(buf) - pos)
        final = pos + want >= len(buf)
        rec_off, consumed, cls, at, need = ops.tfrecord_frame(buf[pos:pos + want], final, want // 16 + 1)
        assert cls == 0, (cls, at)
        if len(rec_off):
            assert consumed == rec_off[-1] + 16 + struct.unpack_from("<Q", buf[pos:].tobytes(), rec_off[-1])[0]
        for o in rec_off:
            ln = struct.unpack_from("<Q", buf.tobytes(), pos + o)[0]
            out.append(buf[pos + o + 12:pos + o + 12 + ln].tobytes())
        if consumed == 0:
            assert not final and need > want
            chunk = max(2 * chunk, need)
        pos += consumed
    return out


def test_frame_matches_read_records_for_every_chunking(tmp_path):
    sizes = [0, 1, 2, 5, 11, 12, 13, 100, 1000, 4999, 5000, 0, 3, 2048]
    p, recs, buf = _file(tmp_path, sizes)
    assert list(tfr.read_records(p, verify_crc=True)) == recs
    for chunk in (16, 17, 29, 64, 100, 1000, 4096, 5016, 5017, len(buf), len(buf) + 7):
        assert _frame_all(buf, chunk) == recs, chunk


def test_frame_sizes_0_to_5000(tmp_path):
    sizes = list(range(0, 5001, 37)) + [5000]
    p, recs, buf = _file(tmp_path, sizes, seed=1)
    rec_off, consumed, cls, _, _ = ops.tfrecord_frame(buf, True, len(buf) // 16 + 1)
    assert cls == 0 and consumed == len(buf) and len(rec_off) == len(recs)
    assert _frame_all(buf, 777) == recs


def test_frame_cut_mid_header_and_mid_record_leaves_the_tail(tmp_path):
    p, recs, buf = _file(tmp_path, [40, 50, 60])
    first = 16 + 40
    for cut in (first + 5, first + 12, first + 30):                 # mid-header, header only, mid-record
        rec_off, consumed, cls, _, need = ops.tfrecord_frame(buf[:cut], False, 10)
        assert cls == 0 and list(rec_off) == [0] and consumed == first
    rec_off, consumed, cls, _, need = ops.tfrecord_frame(buf[:first + 20], False, 10)
    assert need == 16 + 50
    rec_off, consumed, _, _, _ = ops.tfrecord_frame(buf, True, 2)   # max_records
    assert len(rec_off) == 2 and consumed == first + 66


def test_frame_errors_match_read_records(tmp_path):
    p, recs, buf = _file(tmp_path, [40, 50, 60])
    at = 16 + 40
    for byte in (at, at + 3, at + 8, at + 11):                      # flipped length or header-CRC byte
        bad = buf.copy()
        bad[byte] ^= 0x10
        open(p, "wb").write(bad.tobytes())
        with pytest.raises(ValueError, match=f"corrupted record length at byte {at}$"):
            list(tfr.read_records(p, verify_crc=True))
        _, consumed, cls, off, _ = ops.tfrecord_frame(bad, True, 10)
        assert (cls, off, consumed) == (2, at, at)
    for cut, cls_want, what in ((len(buf) - 1, 3, "truncated record"), (at + 16 + 50 + 7, 1, "truncated record header")):
        open(p, "wb").write(buf[:cut].tobytes())
        with pytest.raises(ValueError, match=f"{what} at byte (\\d+)$") as e:
            list(tfr.read_records(p, verify_crc=True))
        _, consumed, cls, off, _ = ops.tfrecord_frame(buf[:cut], True, 10)
        assert cls == cls_want and str(e.value).endswith(f"at byte {off}")
        assert ops.tfrecord_frame(buf[:cut], False, 10)[2] == 0      # not final: the tail waits for more bytes


def _batches_of(groups, n, epochs, B):
    out = []
    for b0, b1 in groups:
        idx, counts = group_slots(n, epochs, B, b0, b1)
        idx = idx.reshape(-1, B)
        for row, c in zip(idx, counts):
            assert (row[c:] == row[0]).all()                        # padding slots = the batch's first sample
            out.append(row[:c].tolist())
    return out


def test_group_planner_concatenates_to_index_stream():
    rng = np.random.RandomState(3)
    for _ in range(200):
        n, epochs, B = int(rng.randint(1, 40)), int(rng.randint(1, 4)), int(rng.randint(1, 50))
        cost = rng.randint(16, 300, n).astype(np.int64)
        budget = int(rng.randint(1, 4000))
        groups = plan_groups(cost, epochs, B, budget)
        assert _batches_of(groups, n, epochs, B) == list(index_stream(n, epochs, B))
        assert [g[0] for g in groups[1:]] == [g[1] for g in groups[:-1]] and groups[0][0] == 0
        stream = np.tile(cost, epochs)
        for b0, b1 in groups:
            got = stream[b0 * B:b1 * B].sum()
            assert got <= budget or b1 == b0 + 1                     # within budget, or a single oversized batch
    assert plan_groups(np.zeros(0, np.int64), 2, 4, 100) == []
    assert plan_groups(np.ones(5, np.int64), 0, 4, 100) == []
