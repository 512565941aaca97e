"""Host-side model of the work schedule of the resident chain kernel (csrc/gemm_planes.cu: gemm_chain_resident_kernel): a CTA takes each
of its tiles through every layer of chain 0, then the tile of the same index through every layer of chain 1, while its activation tile stays
in shared memory.  Checks that every (chain, tile, layer) unit is processed exactly once, all layers of a (chain, tile) consecutively on one
CTA in layer order, and that the per-chain rotation balances the two-chain launch at the update's row count."""

import itertools

from tests.chain_tiles import chain_tiles


def schedule(n_tiles, n_sms, n_chains, n_layers):
    """[(cta, [(chain, tile, layer), ...])] exactly as gemm_chain_resident_kernel enumerates them."""
    n_units = min(n_tiles, n_sms)
    out = []
    for unit in range(n_units):
        tiles = chain_tiles(n_tiles, n_units, n_chains, unit)
        seq = []
        for ti, c in itertools.product(range(max(map(len, tiles))), range(n_chains)):
            if ti < len(tiles[c]):
                seq += [(c, tiles[c][ti], l) for l in range(n_layers)]
        out.append((unit, seq))
    return out


def check(n_tiles, n_sms, n_chains, n_layers):
    sched = schedule(n_tiles, n_sms, n_chains, n_layers)
    seen = set()
    for _, seq in sched:
        for i, (c, t, l) in enumerate(seq):
            assert (c, t, l) not in seen, "unit processed twice"
            seen.add((c, t, l))
            if l > 0:
                assert seq[i - 1] == (c, t, l - 1), "a layer does not directly follow its predecessor on the resident tile"
    assert len(seen) == n_chains * n_tiles * n_layers, "a unit is missing"
    return sched


def test_every_unit_once_layers_consecutive():
    for n_sms in (132, 74):
        for n_tiles, n_chains, n_layers in [(512, 2, 3), (512, 1, 3), (512, 1, 4), (300, 2, 2), (5, 1, 3), (4, 2, 3), (2, 1, 1), (75, 2, 4), (8, 2, 3)]:
            check(n_tiles, n_sms, n_chains, n_layers)


def test_two_chain_rotation_balances_the_update_launch():
    # 65,536 rows = 512 tiles on 132 SMs: 1,024 (chain, tile) pairs -> 7 or 8 per CTA with the rotation
    per = {cta: len({(c, t) for c, t, _ in seq}) for cta, seq in schedule(512, 132, 2, 3)}
    assert set(per.values()) == {7, 8} and sum(per.values()) == 1024
