"""Checkpoints on the CPU oracle (oracle/checkpoint_oracle.c): a saved volume resumes bit for bit, save -> load -> save is
identical, and every malformed or mismatched buffer is refused before anything is written."""
import numpy as np
import pytest

from dynslam_b200 import abi, formats
from tests import checkpointlib as K
from tests import hostlib as H
from tests.parity import Cfg

# small minAge: the queue pops and blocks are freed inside the sequence
CFG = Cfg(scale=0.2, numBlocks=16384, numBuckets=0x4000, excessSize=0x2000)
DECAY = (3, 2)
K_CUT, M_MORE = 5, 4


@pytest.fixture(scope="module")
def run():
    frames = K.street_frames(K_CUT + M_MORE)
    h, w = frames[0][0].shape
    a = K.host_volume(CFG, w, h)
    for f in frames[:K_CUT]:
        K.oracle_frame(a, *f, DECAY)
    buf = K.oracle_save(a)
    hdr = formats.checkpoint_header(buf)
    b = K.host_volume(CFG, w, h, fill=0xA5)
    assert K.oracle_load(b, buf) == (abi.OK, 0)
    saved_again = K.oracle_save(b)
    for f in frames[K_CUT:]:
        K.oracle_frame(a, *f, DECAY)
        K.oracle_frame(b, *f, DECAY)
    return dict(a=a, b=b, buf=buf, hdr=hdr, saved_again=saved_again, w=w, h=h)


def test_resume_is_bit_exact(run):
    hdr = run["hdr"]
    assert hdr["totalDecayed"] > 0 and hdr["noSnapshots"] == DECAY[1] and hdr["frameIdx"] == K_CUT   # the queue popped, blocks freed
    assert H.oracle().oracle_decayed_block_count(run["a"].engine) > hdr["totalDecayed"]           # and decays after the cut too
    K.assert_same(K.volume_state(run["a"]), K.volume_state(run["b"]))
    assert K.oracle_save(run["a"]).tobytes() == K.oracle_save(run["b"]).tobytes()                  # the queues too


def test_save_load_save_is_identical(run):
    assert run["saved_again"].tobytes() == run["buf"].tobytes()


def test_layout(run):
    buf, hdr = run["buf"], run["hdr"]
    assert hdr["totalBytes"] == buf.size and hdr["version"] == abi.CHECKPOINT_VERSION
    off, ln = hdr["sections"]["BLOCK_DATA"]
    assert off % 4096 == 0 and ln == 4096 * hdr["noBlocks"] and off + ln == buf.size
    assert all(o % 8 == 0 for o, _ in hdr["sections"].values())
    ids = buf[hdr["sections"]["BLOCK_IDS"][0]:][:4 * hdr["noBlocks"]].view(np.uint32)
    assert np.all(np.diff(ids.astype(np.int64)) > 0)


def _crafted(buf, hdr_edit=None, at=None, value=None, size=None):
    b = buf.copy()
    if hdr_edit is not None:
        h = b[:abi.CHECKPOINT_HEADER_BYTES].view(abi.CHECKPOINT_HEADER_DTYPE)
        hdr_edit(h)
    if at is not None:
        b[at:at + len(value)] = np.frombuffer(value, np.uint8)
    return b[:size] if size is not None else b


def rejection_cases(buf, hdr):
    sec = hdr["sections"]
    ids_off = sec["BLOCK_IDS"][0]
    hid = sec["HASH_INDEX"][0]

    def setf(k, v):
        def f(h):
            h[k] = v
        return f
    return {
        "bad magic": (_crafted(buf, at=0, value=b"B200CKPX"), 2),
        "bad version": (_crafted(buf, setf("version", 2)), 3),
        "truncated header": (buf[:100].copy(), 1),
        "truncated buffer": (buf[:-4096].copy(), 11),
        "trailing bytes": (np.concatenate([buf, np.zeros(16, np.uint8)]), 11),
        "section table disagrees": (_crafted(buf, setf("noEntries", hdr["noEntries"] - 1)), 10),
        "voxelSize": (_crafted(buf, setf("voxelSize", np.nextafter(np.float32(CFG.voxelSize), np.float32(1)))), 5),
        "mu": (_crafted(buf, setf("mu", 0.5)), 5),
        "geometry": (_crafted(buf, setf("img_w", hdr["img_w"] + 1)), 4),
        "optional buffers": (_crafted(buf, setf("flags", hdr["flags"] | abi.CK_HAS_SWAP_STATES)), 7),
        "block ids out of order": (_crafted(buf, at=ids_off, value=np.array([5, 5], np.uint32).tobytes()), 12),
        "entry index out of range": (_crafted(buf, at=hid, value=np.array([0x7fffffff], np.uint32).tobytes()), 12),
        "queue count": (_crafted(buf, at=sec["QUEUE_COUNTS"][0], value=np.array([-2], np.int32).tobytes()), 13),
        "visible count beyond the list": (_crafted(buf, setf("noVisibleBlocks", hdr["numBlocks"] + 1)), 9),
    }


def test_rejections_touch_nothing(run):
    b, buf = run["b"], run["buf"]
    before = K.volume_state(b)
    cases = rejection_cases(buf, run["hdr"])
    for name, (bad, why) in cases.items():
        assert K.oracle_load(b, bad) == (abi.ERR_INVALID, why), name
        K.assert_same(before, K.volume_state(b), f"{name}: ")
    # a target whose geometry or optional buffers differ
    other = K.host_volume(Cfg(scale=0.2, numBlocks=8192, numBuckets=0x4000, excessSize=0x2000), run["w"], run["h"])
    assert K.oracle_load(other, buf) == (abi.ERR_INVALID, 4)
    no_fwd = K.host_volume(CFG, run["w"], run["h"])
    no_fwd.rs.d_forwardProjection = None
    assert K.oracle_load(no_fwd, buf) == (abi.ERR_INVALID, 8)

