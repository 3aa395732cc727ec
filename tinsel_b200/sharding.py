"""Host-side image-plane sharding rules (the C ABI's, restated for hosts written in Python: bench.py's
per-rank bookkeeping and the gloo tests).

Rank r of n owns the 4-pixel-high tile rows t with t % n == r (tb200_set_shard; the device side is
decode_sample() in csrc/kernels.cu).  Every sample belongs to exactly one shard, so the sum of the
per-rank accumulators is the unsharded image (up to fp32 summation order)."""

TILE_ROWS = 4


def shard_rows(height, shard, num_shards):
    """Pixel rows whose samples shard `shard` of `num_shards` traces."""
    rows = []
    t = shard
    while t * TILE_ROWS < height:
        rows.extend(range(t * TILE_ROWS, min(height, (t + 1) * TILE_ROWS)))
        t += num_shards
    return rows


def shard_sample_count(width, height, shard, num_shards, spp=1):
    return len(shard_rows(height, shard, num_shards)) * width * spp


def slab_rows(height, member, num_members):
    """Owner-computes row slabs (tb200_create_multi / tb200_set_slab): (first_row, num_rows) of member k of n,
    contiguous and cut at tile rows.  Mirrors tb200_slab_rows (tested against it)."""
    tile_rows = (height + TILE_ROWS - 1) // TILE_ROWS

    def cut(k):
        return height if k >= num_members else min(height, (tile_rows * k // num_members) * TILE_ROWS)
    return cut(member), cut(member + 1) - cut(member)


def slab_traced_rows(height, first_row, num_rows, filter_width):
    """(first, count) of the pixel rows whose samples the owner of a slab traces: the slab plus the filter's
    reach, ceil(width) + 1 rows, on either side (render.cpp:404-407), with the width clamped to [0, 2^30] (NaN
    counts as 0).  Mirrors tb200_slab_traced_rows."""
    import math
    reach = int(math.ceil(min(max(0.0, filter_width), 1073741824.0))) + 1
    lo = max(0, min(first_row, height))
    hi = max(lo, min(first_row + max(0, num_rows), height))
    if hi <= lo:
        return max(0, lo - reach), 0
    t0 = max(0, lo - reach)
    return t0, min(height, hi + reach) - t0
