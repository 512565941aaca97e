"""Host-side model of the work schedule of the chained hidden-layer launch (csrc/gemm_planes.cu: gemm_chain_kernel -- the `unit_of` enumeration
every role of a CTA walks).  Checks, for the shapes the update uses and for ragged ones, what the kernel relies on and what DESIGN.md
section 4.6 claims:
  * every (chain, tile, layer) unit is processed exactly once over all pairs, all layers of a (chain, tile) by the SAME pair (the next layer
    re-loads what the pair itself stored), in layer order, and the lane of a unit -- the `stored[lane]` barrier its producer waits on -- is the
    lane of its predecessor;
  * the dependency distance (units between two layers of a lane) is 4 with full groups, never 0;
  * with two chains the per-chain rotation leaves every pair with 4 + 3 or 3 + 3 tiles at the north-star row count (256 tiles on 74 pairs),
    where one shared assignment would give 4 + 4 to 34 pairs."""

import itertools

from tests.chain_tiles import chain_tiles

LANES = 4


def schedule(n_tiles, n_pairs, n_chains, n_layers, rotate=True):
    """[(pair, [(chain, tile, layer, lane), ...])] exactly as gemm_chain_kernel enumerates them."""
    n_units = min(n_tiles, n_pairs)
    tpg = LANES // n_chains
    out = []
    for unit in range(n_units):
        tiles = chain_tiles(n_tiles, n_units, n_chains, unit, rotate)
        n_groups = (max(map(len, tiles)) + tpg - 1) // tpg
        seq = []
        for gi, l, ln in itertools.product(range(n_groups), range(n_layers), range(LANES)):
            c, ti = ln % n_chains, gi * tpg + ln // n_chains
            if ti < len(tiles[c]):
                seq.append((c, tiles[c][ti], l, ln))
        out.append((unit, seq))
    return out


def check(n_tiles, n_pairs, n_chains, n_layers):
    sched = schedule(n_tiles, n_pairs, n_chains, n_layers)
    seen = {}
    for pair, seq in sched:
        last = {}
        for pos, (c, t, l, ln) in enumerate(seq):
            assert (c, t, l) not in seen, "unit processed twice"
            seen[(c, t, l)] = pair
            if l > 0:
                p_pos, p_ln = last[(c, t)]
                assert seen[(c, t, l - 1)] == pair and p_ln == ln and pos - p_pos >= 1
            last[(c, t)] = (pos, ln)
    assert len(seen) == n_chains * n_tiles * n_layers, "a unit is missing"
    return sched


def test_every_unit_once_in_layer_order_on_one_pair():
    for n_tiles, n_chains, n_layers in [(256, 2, 3), (256, 1, 3), (256, 1, 4), (150, 2, 2), (5, 1, 3), (4, 2, 3), (2, 1, 1), (75, 2, 4), (32, 2, 3), (1, 1, 2)]:
        check(n_tiles, 74, n_chains, n_layers)


def test_dependency_distance_is_four_with_full_groups():
    for n_chains in (1, 2):
        for pair, seq in check(296, 74, n_chains, 3):  # 4 tiles per pair and chain: every group is full
            pos = {}
            for i, (c, t, l, ln) in enumerate(seq):
                if l > 0:
                    assert i - pos[(c, t, l - 1)] == LANES
                pos[(c, t, l)] = i


def test_two_chain_rotation_balances_the_north_star_launch():
    def tiles_per_pair(rotate):
        per = {}
        for pair, seq in schedule(256, 74, 2, 3, rotate):
            per[pair] = len({(c, t) for c, t, _, _ in seq})
        return per

    rotated, shared = tiles_per_pair(True), tiles_per_pair(False)
    assert set(rotated.values()) == {6, 7} and sum(rotated.values()) == 512
    assert max(shared.values()) == 8 and sum(shared.values()) == 512  # 34 pairs with 4 + 4 tiles: the launch lasted 8/6.92 of the balanced time
    single = {pair: len({(c, t) for c, t, _, _ in seq}) for pair, seq in schedule(256, 74, 1, 3)}
    assert set(single.values()) == {3, 4}  # a single chain cannot be balanced at tile granularity (DESIGN 4.6 / 7)
