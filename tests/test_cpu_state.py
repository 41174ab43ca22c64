"""rb_state_info on crafted session blobs (include/rebvo_b200.h, session checkpoints; layout in DESIGN.md §5): it accepts a
well-formed header and refuses a bad magic, another version, inconsistent sizes and offsets, and a checksum that does not
match the bytes.  Host code: runs without a GPU."""
import ctypes as C
import struct

import pytest

HEADER = struct.Struct("<8sIIQQiiffffiiddqiiQQQQ")   # StateHeader, 128 bytes
M64 = (1 << 64) - 1


def checksum(data):
    """FNV-1a over 64-bit little-endian words, then the bytes of a shorter tail."""
    h = 0xcbf29ce484222325
    n8 = len(data) // 8 * 8
    for (w,) in struct.iter_unpack("<Q", data[:n8]):
        h = ((h ^ w) * 0x100000001b3) & M64
    for b in data[n8:]:
        h = ((h ^ b) * 0x100000001b3) & M64
    return h


def blob(kn=3, dev_bytes=1024, host_bytes=16, **over):
    f = dict(magic=b"RBB2STAT", version=1, header_bytes=128, total=0, checksum=0, w=752, h=480, ppx=367.2, ppy=248.4,
             zfx=458.6, zfy=457.3, kl_capacity=40000, mode=0, sigma0=3.56, ksigma=1.2599, n_pushed=20, kn=kn, det_r=2,
             imu_count=0, imu_checksum=0, off_dev=128, off_host=128 + dev_bytes)
    payload = bytes((7 * i + 3) & 0xff for i in range(dev_bytes + host_bytes))
    f["total"] = 128 + len(payload)
    fix_sum = over.pop("fix_checksum", True)
    f.update(over)
    head = HEADER.pack(*f.values())
    data = head + payload
    if fix_sum:
        f["checksum"] = checksum(data[32:])
        data = HEADER.pack(*f.values()) + payload
    return data


def info(data):
    from rebvo_b200 import capi
    out = capi.StateInfo()
    r = capi.lib().rb_state_info(data, C.c_size_t(len(data)), C.byref(out))
    return r, out


def test_header_size():
    assert HEADER.size == 128


def test_accepts_a_well_formed_blob(built):
    from rebvo_b200 import capi
    data = blob()
    r, out = info(data)
    assert r == 0
    assert (out.version, out.mode, out.bytes, out.kn, out.n_pushed, out.kl_capacity) == (1, 0, len(data), 3, 20, 40000)
    assert (out.cam.w, out.cam.h) == (752, 480) and out.Sigma0 == 3.56 and out.KSigma == 1.2599
    d = capi.state_info(data)
    assert d["w"] == 752 and d["kn"] == 3 and d["bytes"] == len(data) and d["mode"] == capi.STATE_VISION


@pytest.mark.parametrize("what,over", [
    ("magic", dict(magic=b"RBB2STAX")),
    ("version", dict(version=2)),
    ("header size", dict(header_bytes=120)),
    ("total size", dict(total=5000)),
    ("device offset", dict(off_dev=136)),
    ("host offset past the end", dict(off_host=128 + 4096)),
    ("device section shorter than its keylines", dict(kn=9)),
    ("keylines above capacity", dict(kl_capacity=2)),
    ("keylines before any frame", dict(n_pushed=0)),
    ("mode", dict(mode=3)),
])
def test_rejects_inconsistent_headers(built, what, over):
    r, _ = info(blob(**over))
    assert r == -2, what


def test_rejects_bad_checksum_and_truncation(built):
    data = bytearray(blob())
    assert info(bytes(data))[0] == 0
    data[500] ^= 1
    assert info(bytes(data))[0] == -2, "flipped payload byte"
    assert info(blob(fix_checksum=False, checksum=1))[0] == -2, "wrong checksum"
    good = blob()
    assert info(good[:-8])[0] == -2, "truncated"
    assert info(good[:100])[0] == -2, "shorter than the header"
    from rebvo_b200 import capi
    with pytest.raises(capi.RbError):
        capi.state_info(good[:-1])
