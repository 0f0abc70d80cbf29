"""CPU: the row-block schedule of the fused FFN kernel's 2-CTA clusters restated (csrc/ffn_tc.cu): cluster c walks the row
block pairs c, c + clusters, ...; CTA `rank` of the pair owns row block 2 pair + rank.  Every row block is owned exactly once,
both CTAs of a cluster walk the same number of pairs (they share every weight K-block and every stage release), and the only
CTA without rows is the second of the last pair at an odd number of row blocks: it loads the last block's rows (in range)
and its row indices are all >= M, so it stores nothing."""
import pytest

FM, CLUSTER = 64, 2


def schedule(M, clusters_resident):
    nrb = -(-M // FM)
    npairs = -(-nrb // CLUSTER)
    clusters = min(npairs, clusters_resident)                  # grid = CLUSTER x clusters
    walk = {}
    for c in range(clusters):
        for rank in range(CLUSTER):
            walk[c, rank] = [(p * CLUSTER + rank, min(p * CLUSTER + rank, nrb - 1) * FM) for p in range(c, npairs, clusters)]
    return nrb, clusters, walk


@pytest.mark.parametrize("clusters_resident", [1, 2, 60, 62, 64, 66])
@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 128, 129, 64 * 125, 7936, 8448, 8449, 20000])
def test_cluster_schedule_owns_every_row_block_once(M, clusters_resident):
    nrb, clusters, walk = schedule(M, clusters_resident)
    assert clusters >= 1
    owned = sorted(rb for steps in walk.values() for rb, _ in steps if rb < nrb)
    assert owned == list(range(nrb))
    idle = [(c, rank, rb, m0) for (c, rank), steps in walk.items() for rb, m0 in steps if rb >= nrb]
    assert len(idle) == nrb % CLUSTER
    for c, rank, rb, m0 in idle:
        assert (rank, rb) == (1, nrb) and rb * FM >= M               # every row the consumers would store is >= M
        assert 0 <= m0 < M                                           # the X box it loads starts inside the tensor
    for c in range(clusters):
        a, b = walk[c, 0], walk[c, 1]
        assert len(a) == len(b)                                      # same trip count: same K-block sequence
        assert all(rb1 == rb0 + 1 and rb0 % CLUSTER == 0 for (rb0, _), (rb1, _) in zip(a, b))
