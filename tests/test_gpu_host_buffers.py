"""Host entries on caller buffers that share a memory page with a buffer an earlier call registered for DMA.

process_host registers the pages of a large input buffer (music_b200.cu, host_register), so the registration takes in
the first bytes of whatever the allocator put after it on the last page.  A later call whose input starts on that page
and runs past it (a smaller window buffer, or an antenna stream of the planar entry) must still be copied: the driver
refuses a copy from memory registered only in part.  Both layouts are built deterministically inside one allocation."""
import numpy as np
import pytest

from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_coarray import music_doa_coarray

pytestmark = pytest.mark.gpu

PAGE = 4096
M, SNAPS, K = 4, 256, 360
NS = M * SNAPS
W_BIG, W_SMALL = 160, 40  # 1.25 MiB (registered) and 320 KiB (not registered) of input


def make(kind):
    if kind == "plain":
        blk = music_doa(M, 1, NS, np.ones((K, M), np.complex64), K)
        blk.set_array_geometry([[0.5 * i, 0.0] for i in range(M)], 1.0)
        return blk
    blk = music_doa_coarray(M, 3, NS, K, [0, 1, 4, 6], (0.5, 0.0), 1.0)
    blk.set_peak_mode("esprit")
    return blk


def shared_page(first, rest, rng):
    """views of one allocation: `first` complex64 values ending 2048 bytes into a page, then `rest` values right after"""
    raw = (rng.standard_normal(first + rest + PAGE) + 1j * rng.standard_normal(first + rest + PAGE)).astype(np.complex64)
    off = (2048 - (raw.ctypes.data + 8 * first)) % PAGE // 8
    return raw[off:off + first], raw[off + first:off + first + rest]


def run(blk, x, W, planar):
    ang, lvl = np.zeros((W, blk.n), np.float32), np.zeros((W, blk.n), np.float32)
    if planar:
        streams = [x[a * W * SNAPS:(a + 1) * W * SNAPS] for a in range(M)]
        blk.work_planar(W, streams, [ang, lvl])
    else:
        blk.work(W, [x.reshape(W, NS)], [ang, lvl])
    return ang, lvl, blk.last_bins().copy()


@pytest.mark.parametrize("kind", ["plain", "coarray"])
@pytest.mark.parametrize("planar", [False, True], ids=["interleaved", "planar"])
def test_input_on_a_registered_page(kind, planar):
    big, small = shared_page(W_BIG * NS, W_SMALL * NS, np.random.default_rng(1))
    assert (big.ctypes.data + big.nbytes) % PAGE == 2048 and small.ctypes.data == big.ctypes.data + big.nbytes
    ref_blk = make(kind)  # a handle that has registered nothing
    ref = run(ref_blk, small, W_SMALL, planar)
    ref_blk.close()
    blk = make(kind)
    run(blk, big, W_BIG, False)  # registers big's pages, the first 2048 bytes of small with them
    got = run(blk, small, W_SMALL, planar)
    for g, r in zip(got, ref):
        assert np.array_equal(g, r)
    # and the registered buffer itself still runs
    run(blk, big, W_BIG, False)
    blk.close()
