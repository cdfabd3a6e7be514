"""Model of the persistent tile schedule of ``group_gemm_kernel`` (csrc/group_gemm.cu): restates the device-side tile scan
(``s_tile_start`` from ``tokens_per_expert``) and ``decode(tile)`` and checks, for ragged expert sizes, that every 128-row x
BLOCK_N-column piece of the output is produced exactly once and that each CTA sees its tiles in non-decreasing order (the
monotone expert search relies on it).  Also records the wave quantisation of the C2 shapes on the 132 SMs of an H100."""
import random

import pytest

BM = 128
SMS = 132  # persistent CTAs of the kernel on an H100 ("cluster" below: one CTA)


def schedule(counts, n_tiles, n_clusters, mode_tn=False, m_out_tiles=0):
    E = len(counts)
    if mode_tn:
        total_tiles = E * m_out_tiles * n_tiles
    else:
        tile_start = [0]
        for c in counts:
            tile_start.append(tile_start[-1] + ((c + BM - 1) // BM) * n_tiles)
        total_tiles = tile_start[-1]

    def decode(tile, e_hint):
        if mode_tn:
            per_e = m_out_tiles * n_tiles
            e = tile // per_e
            local = tile - e * per_e
        else:
            while tile >= tile_start[e_hint + 1]:
                e_hint += 1
            e = e_hint
            local = tile - tile_start[e]
        return (e, local // n_tiles, local % n_tiles), e_hint

    per_cluster = []
    for c in range(n_clusters):
        e_hint, seq = 0, []
        for tile in range(c, total_tiles, n_clusters):
            t, e_hint = decode(tile, e_hint)
            seq.append(t)
        per_cluster.append(seq)
    return total_tiles, per_cluster


@pytest.mark.parametrize("n_tiles,n_clusters", [(6, SMS), (3, SMS), (8, SMS), (6, 5), (1, 3)])
def test_every_output_tile_is_produced_once(n_tiles, n_clusters):
    rng = random.Random(n_tiles * 100 + n_clusters)
    for trial in range(20):
        E = rng.choice([1, 3, 8])
        counts = [rng.choice([0, 1, 255, 256, 257, 2048, rng.randrange(0, 3000)]) for _ in range(E)]
        total_tiles, per_cluster = schedule(counts, n_tiles, n_clusters)
        cover = {}
        for seq in per_cluster:
            assert seq == sorted(seq), "a cluster must see tiles in non-decreasing order"
            for e, m, n in seq:
                assert m * BM < counts[e], "tile beyond the expert's rows"
                cover[(e, m, n)] = cover.get((e, m, n), 0) + 1
        want = {(e, m, n) for e, c in enumerate(counts) for m in range((c + BM - 1) // BM) for n in range(n_tiles)}
        assert set(cover) == want and all(v == 1 for v in cover.values())
        assert sum(len(s) for s in per_cluster) == total_tiles


def test_c2_wave_quantisation():
    """At C2 (8 experts x 2048 rows = 16 row blocks each, 132 CTAs, 256-column tiles) every product runs a multiple of 384
    tiles: 2.9 waves of work per 3 waves, 97 % wave efficiency."""
    uniform = [2048] * 8
    waves = lambda tiles: -(-tiles // SMS)  # noqa: E731
    for n_tiles, tiles in [(6, 768), (3, 384), (8, 1024)]:  # w13 NT (I=768: 128 features per tile), dX of w2 (768), w2 NT / dX of w13 (2048)
        total, _ = schedule(uniform, n_tiles, SMS)
        assert total == tiles
    assert round(384 / SMS / waves(384), 3) == 0.97 and round(768 / SMS / waves(768), 3) == 0.97
    assert round(1024 / SMS / waves(1024), 3) == 0.97
    total, _ = schedule(uniform, 8, SMS, mode_tn=True, m_out_tiles=12)  # dW13: 8 experts x 12 x 8
    assert total == 768


def schedule_tn_pair(E, geo_a, geo_b, n_clusters):
    """decode() of the two-product TN launch (xtb_group_gemm_tn_pair): the first product's tiles, then the second's;
    geo = (m_out_tiles, n_tiles).  Returns per cluster the list of (product, expert, m_blk, n_blk)."""
    tiles0 = E * geo_a[0] * geo_a[1]
    tiles1 = E * geo_b[0] * geo_b[1]

    def decode(tile):
        prob, (mt, nu) = 0, geo_a
        if tile >= tiles0:
            tile -= tiles0
            prob, (mt, nu) = 1, geo_b
        per_e = mt * nu
        e = tile // per_e
        local = tile - e * per_e
        return prob, e, local // nu, local - (local // nu) * nu

    return tiles0 + tiles1, [[decode(t) for t in range(c, tiles0 + tiles1, n_clusters)] for c in range(n_clusters)]


@pytest.mark.parametrize("E,geo_a,geo_b,n_clusters", [(8, (16, 3), (12, 8), SMS), (4, (4, 2), (4, 4), SMS), (5, (1, 2), (2, 1), 3)])
def test_tn_pair_tile_list_covers_both_products_once(E, geo_a, geo_b, n_clusters):
    total, per_cluster = schedule_tn_pair(E, geo_a, geo_b, n_clusters)
    seen = [t for seq in per_cluster for t in seq]
    want = {(p, e, m, n) for p, (mt, nu) in enumerate((geo_a, geo_b)) for e in range(E) for m in range(mt) for n in range(nu)}
    assert len(seen) == total == len(want) and set(seen) == want
    # balance: no cluster has more than one tile above any other (equal cost per tile: same token groups)
    sizes = [len(s) for s in per_cluster]
    assert max(sizes) - min(sizes) <= 1


def test_tn_pair_never_needs_more_waves_than_two_launches():
    """One tile list over both weight gradients never takes more waves than the two launches, and saves one whenever the
    two last waves fit into one.  At C2 on 132 CTAs (384 + 768 tiles) both ways take 9 waves."""
    waves = lambda tiles: -(-tiles // SMS)  # noqa: E731
    for E, geo_a, geo_b in [(8, (16, 3), (12, 8)), (8, (8, 3), (6, 8)), (4, (4, 2), (4, 4)), (3, (2, 2), (1, 5))]:
        ta, tb = E * geo_a[0] * geo_a[1], E * geo_b[0] * geo_b[1]
        total, _ = schedule_tn_pair(E, geo_a, geo_b, SMS)
        assert total == ta + tb and waves(total) <= waves(ta) + waves(tb)
        if (ta % SMS) and (tb % SMS) and (ta % SMS) + (tb % SMS) <= SMS:
            assert waves(total) == waves(ta) + waves(tb) - 1
    total, _ = schedule_tn_pair(8, (16, 3), (12, 8), SMS)
    assert total == 1152 and waves(384) + waves(768) == 9 and waves(total) == 9
