"""CPU: the host half of the parallel JPEG entropy decode: which restart intervals it takes, how it cuts them into
subsequences, and the subsequence records pack_cls_batch / pack_batch reserve for it in the decode's scratch."""
import numpy as np
import pytest

import jpeg_oracle as O
from multimae_b200 import data as D
from multimae_b200 import jpeg as J
from multimae_b200 import kernels as K


def test_parallel_threshold():
    assert J.PARALLEL_MIN_BYTES == 32 * J.SUB_BYTES and J.SUB_BYTES % J.SLOT_BYTES == 0
    assert not J.parallel_interval(0) and not J.parallel_interval(J.PARALLEL_MIN_BYTES - 1)
    assert J.parallel_interval(J.PARALLEL_MIN_BYTES) and J.parallel_interval((1 << 28) - 1)
    assert not J.parallel_interval(1 << 28)


def _unstuffed_index(seg):
    """Index of every byte of `seg` in the stream with the zero of each FF 00 pair removed (-1 for those zeros)."""
    out, u, skip = [], 0, False
    for b in seg:
        if skip:
            out.append(-1)
            skip = False
            continue
        out.append(u)
        u += 1
        skip = b == 0xFF
    return out


@pytest.mark.parametrize("seed", range(4))
def test_subsequences_never_start_inside_a_stuffed_pair(seed):
    data = O.encode(O.image(seed, 300 + 40 * seed, 200), quality=95, subsampling=seed % 3)
    src = J.parse(data)
    seg = data[src.scan[0]:src.scan[1]]
    index = _unstuffed_index(seg)
    subs = J.subsequences(seg)
    assert len(subs) == -(-len(seg) // J.SUB_BYTES)
    moved = 0
    for j, (r, u) in enumerate(subs):
        assert r in (j * J.SUB_BYTES, j * J.SUB_BYTES + 1)
        moved += r != j * J.SUB_BYTES
        assert index[r] == u and u >= 0
    # a start moved on is one the naive cut would have put on a stuffed zero
    assert moved == sum(index[j * J.SUB_BYTES] < 0 for j in range(1, len(subs)))


def test_stuffed_pair_at_every_cut():
    seg = bytearray([1] * (6 * J.SUB_BYTES + 5))
    for r in range(J.SUB_BYTES, len(seg), J.SUB_BYTES):
        seg[r - 1:r + 1] = b"\xff\x00"
    seg = bytes(seg)
    subs = J.subsequences(seg)
    assert [r for r, _ in subs[1:]] == [j * J.SUB_BYTES + 1 for j in range(1, len(subs))]
    assert [u for _, u in subs] == [r - seg[:r].count(0xFF) for r, _ in subs]


def test_subsequence_slots_hold_every_interval():
    for kw in (dict(), dict(restart_marker_blocks=1), dict(restart_marker_blocks=5), dict(restart_marker_rows=2)):
        src = J.parse(O.encode(O.image(3, 640, 200), quality=90, **kw))
        nbytes = src.scan[1] - src.scan[0]
        slots = J.subsequence_slots(nbytes, len(src.intervals))
        used = set()
        for k, (a, b) in enumerate(src.intervals):
            first = a // J.SLOT_BYTES + k
            rec = set(range(first, first + -(-(b - a) // J.SLOT_BYTES)))
            assert not rec & used and all(r < slots for r in rec), (kw, k)
            used |= rec


def _cls_batch():
    datas = [O.encode(O.image(k, 300 + 50 * k, 200), quality=90, subsampling=k % 3,
                      **({"restart_marker_rows": 3} if k == 1 else {})) for k in range(3)]
    srcs = [J.parse(d) for d in datas]
    samples = [D.ClsSample(None, D.FILTER_BICUBIC, False, [], jpeg=(s, (3, 4, 25, 30))) for s in srcs]
    samples.insert(1, D.ClsSample(O.image(9, 20, 30), D.FILTER_BICUBIC, True, []))
    return srcs, D.pack_cls_batch(samples, 32, (0.5,) * 3, (0.5,) * 3, (128,) * 3)


def test_pack_reserves_subsequence_records():
    srcs, p = _cls_batch()
    off, n, coef_blocks, plane_bytes = p.jpeg
    buf = p.buffer.numpy()
    jd = buf[off * 16:off * 16 + n * D.JPEG_FIELDS * 4].view(np.int32).reshape(n, D.JPEG_FIELDS)
    running = 0
    for s, d in zip(srcs, jd):
        assert d[24] == running
        running += J.subsequence_slots(s.scan[1] - s.scan[0], len(s.intervals))
    assert K.jpeg_subsequence_slots(p.buffer, off, n) == running
    a = lambda x: (x + 255) // 256 * 256  # noqa: E731
    assert K.jpeg_scratch_bytes(coef_blocks, plane_bytes, running) == \
        a(coef_blocks * 128) + a(plane_bytes) + running * J.SUB_RECORD_BYTES
    assert K.jpeg_scratch_bytes(coef_blocks, plane_bytes) == a(coef_blocks * 128) + a(plane_bytes)


def test_pretrain_pack_reserves_subsequence_records():
    srcs = [J.parse(O.encode(O.image(k, 200, 150 + 10 * k), quality=85, subsampling=k % 3)) for k in range(3)]
    crops = [D.Crops({"rgb": (s, (0, 0, 100, 120))}, False, 100, 120) for s in srcs]
    p = D.pack_batch(crops, 32, (0.5,) * 3, (0.5,) * 3)
    off, n = p.jpeg[:2]
    jd = p.buffer.numpy()[off * 16:off * 16 + n * D.JPEG_FIELDS * 4].view(np.int32).reshape(n, D.JPEG_FIELDS)
    want = np.cumsum([0] + [J.subsequence_slots(s.scan[1] - s.scan[0], len(s.intervals)) for s in srcs])
    assert list(jd[:, 24]) == list(want[:-1])
    assert K.jpeg_subsequence_slots(p.buffer, off, n) == want[-1]
