"""Index arithmetic the partitioned witness union relies on (csrc/shard_kernels.cuh: `part_lo`, `k_part_pack`, `k_part_bounds`),
restated in numpy and checked exhaustively: for every world size the library accepts (1..256) the owner the pack kernel computes for a
bucket, `(bucket * world) >> 16`, is the rank whose range `[part_lo(r), part_lo(r+1))` holds it, the ranges tile the 65 536 buckets in
rank order (so concatenating the partitions in rank order is the sorted set), and the default piece capacity never exceeds the
cannot-overflow capacity. A restatement — the kernels themselves run in tests/gpu_prims/shard_check.cu (tests/test_shard_check.py),
W simulated ranks on one GPU at world sizes 1 to 255 against CPU references, and in tests/test_parallel.py::test_sharded_call_over_nccl
where the GPUs for several ranks exist."""
import numpy as np

BUCKETS = 65536


def part_lo(r, world):
    return (r * BUCKETS + world - 1) // world


def test_owner_of_a_bucket_matches_the_partition_bounds():
    b = np.arange(BUCKETS, dtype=np.uint64)
    for world in range(1, 257):
        lo = np.array([part_lo(r, world) for r in range(world + 1)], dtype=np.uint64)
        assert lo[0] == 0 and lo[world] == BUCKETS and np.all(np.diff(lo.astype(np.int64)) > 0)
        owner_by_bounds = np.searchsorted(lo[1:], b, side="right")
        assert np.array_equal((b * world) >> 16, owner_by_bounds), world


def test_default_piece_capacity_is_bounded_by_the_safe_one():
    for world in (1, 2, 3, 4, 7, 8, 64, 256):
        for nw_max in (0, 1, 5, 1000, 146960, 10 ** 7):
            safe = nw_max + 1
            default = min(safe, 2 * ((nw_max + world - 1) // world) + 1024)
            assert 1 <= default <= safe
            # a perfectly balanced list always fits the default slots
            assert (nw_max + world - 1) // world <= default


def test_one_item_per_warp_launch_shape_covers_every_item_once():
    """k_read_slots / k_pass2 / k_verify_events / k_verify_storage: grid = ceil(32 n / 128) CTAs of 128 threads, lane 0 of warp w handles item w
    (`if (threadIdx.x & 31) return; t >>= 5; if (t >= n) return;`). Every item exactly once, for sizes around the CTA and warp boundaries."""
    def items(n, per_warp):
        threads = 128
        grid = -(-(n * 32 if per_warp else n) // threads)
        seen = []
        for b in range(grid):
            for tid in range(threads):
                t = b * threads + tid
                if per_warp:
                    if tid & 31:
                        continue
                    t >>= 5
                if t >= n:
                    continue
                seen.append(t)
        return seen
    for n in list(range(1, 20)) + [31, 32, 33, 127, 128, 129, 1020, 16384]:
        for per_warp in (True, False):
            if n == 16384 and not per_warp:
                continue
            assert items(n, per_warp) == list(range(n)), (n, per_warp)
