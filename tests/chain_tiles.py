"""Host-side model of ChainTiles (csrc/gemm_planes.cu), the tile rotation both chain kernels share: tile t of chain c goes to CTA
(t + offset_c) mod n_units, chain 1 rotated by half the grid."""


def chain_tiles(n_tiles, n_units, n_chains, unit, rotate=True):
    """[[tile, ...] for each chain]: the tiles of every chain on CTA `unit`, by tile index, exactly as ChainTiles computes them
    (rotate=False: chain 1 without its rotation)."""
    cu = [unit, (unit + n_units // 2) % n_units if rotate else unit]
    mt = [(n_tiles - c + n_units - 1) // n_units if c < n_tiles else 0 for c in cu]
    return [[cu[c] + ti * n_units for ti in range(mt[c])] for c in range(n_chains)]
