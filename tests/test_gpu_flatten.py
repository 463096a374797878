"""GPU test of the step driver's bucket flatten (the warp-per-block copy of the partition rebuild), held to equality.

The flatten turns a block's cell buckets (64 rows of max_ppc slots, the first `count` of each filled) into the block's bucket:
cell-major, the tags of a cell in slot order, and the start of every cell.  It is integer data, so it must be the very bytes
that cb200_cell_bucket_to_block (the kernel-level entry, which searches the prefix per tag) and a numpy restatement produce,
and nothing behind a bucket's size may be written.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SENTINEL = -7
BLOCKS = 301


def _containers(max_ppc, seed):
    """cell counts [BLOCKS, 64] with cells of 0, 1, 7, 8, 9 and max_ppc tags (block 0 empty, block 1 full, block 2 one tag in its
    last cell), and cell buckets [BLOCKS, 64, max_ppc] whose filled slots hold distinct tags and whose other slots hold -1"""
    rng = np.random.default_rng(seed)
    pool = np.array([0, 0, 1, 7, 8, 8, 8, 9, max_ppc, max_ppc // 2 + 1], np.int32)
    counts = np.minimum(rng.choice(pool, size=(BLOCKS, 64)), max_ppc).astype(np.int32)
    sparse = rng.random(BLOCKS) < 0.3   # blocks at a body's surface: most cells empty
    counts[sparse] *= (rng.random((int(sparse.sum()), 64)) < 0.2).astype(np.int32)
    counts[0] = 0
    counts[1] = max_ppc
    counts[2] = 0
    counts[2, 63] = 1
    filled = np.arange(max_ppc)[None, None, :] < counts[:, :, None]
    tags = rng.permutation(BLOCKS * 64 * max_ppc).astype(np.int32).reshape(BLOCKS, 64, max_ppc)
    return counts, np.where(filled, tags, -1).astype(np.int32), filled


def _expected(counts, cellbuckets, filled, max_ppc):
    sizes = counts.sum(1).astype(np.int32)
    offs = (np.cumsum(counts, 1) - counts).astype(np.uint16)
    buckets = np.full((BLOCKS, 64 * max_ppc), SENTINEL, np.int32)
    for b in range(BLOCKS):
        buckets[b, : sizes[b]] = cellbuckets[b][filled[b]]   # row-major over (cell, slot): cell-major, slot order inside a cell
    return sizes, offs, buckets


@pytest.mark.parametrize("max_ppc", [8, 16, 32, 128])
def test_flatten_is_the_cell_major_slot_order(cuda_lib, max_ppc):
    import torch
    import claymore_b200 as cb
    counts, cellbuckets, filled = _containers(max_ppc, seed=max_ppc)
    want_sizes, want_offs, want_buckets = _expected(counts, cellbuckets, filled, max_ppc)
    cfg = cb.Config(domain_bits=8, max_ppc=max_ppc)
    dev = torch.device("cuda")
    t_counts, t_cells = torch.from_numpy(counts).to(dev), torch.from_numpy(cellbuckets).to(dev)

    def run(entry, *extra):
        sizes = torch.zeros(BLOCKS, dtype=torch.int32, device=dev)
        buckets = torch.full((BLOCKS, 64 * max_ppc), SENTINEL, dtype=torch.int32, device=dev)
        cb._capi.check(entry(C.byref(cfg), BLOCKS, t_counts.data_ptr(), t_cells.data_ptr(), sizes.data_ptr(), buckets.data_ptr(), *extra, None), "flatten")
        torch.cuda.synchronize()
        return sizes.cpu().numpy(), buckets.cpu().numpy()

    offs = torch.full((BLOCKS, 64), -1, dtype=torch.int16, device=dev)
    sizes, buckets = run(cuda_lib.cb200_test_warp_flatten, offs.data_ptr())
    ref_sizes, ref_buckets = run(cuda_lib.cb200_cell_bucket_to_block)
    assert np.array_equal(ref_sizes, want_sizes) and np.array_equal(ref_buckets, want_buckets), "the numpy restatement is not the kernel-level entry"
    assert np.array_equal(sizes, want_sizes), "bucket sizes"
    assert np.array_equal(offs.cpu().numpy().view(np.uint16), want_offs), "cell offsets"
    bad = np.flatnonzero((buckets != want_buckets).any(1))
    assert bad.size == 0, f"buckets differ in blocks {bad[:8].tolist()} (tags, or a write behind the bucket's size)"
