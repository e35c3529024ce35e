"""The persistent GRU chain kernels walk their units in an order in which everything a unit waits for has a smaller
index (round-robin over co-resident blocks then cannot deadlock).  Both chains take the order from ChainOrder
(pnb_chain.cuh): hop-major, or anti-diagonal, which the fp32 chain always uses.  This defines the anti-diagonal order
as a table, restates the closed-form decode both kernels run (chain_decode_diag) and checks the property, the coverage
(every unit exactly once) and the decode against the table; and it checks the property for the hop-major order."""
import itertools

import pytest

DEP = (-1, 0, 1, 2, 2)           # chain_dep: layer whose fresh state is a layer's input (-1: conv2 output, ready before the launch)
DEPTH = tuple(d + 1 for d in DEP)  # (0, 1, 2, 3, 3) for gru1, gru2, gru3, gru_gb, gru_rb (gru_rb reads gru3 like gru_gb does)


def diag_table(n_hops, units):   # the definition: entries (t, l) sorted by diagonal, then layer
    order = []
    for d in range(n_hops + 3):
        for l in range(5):
            t = d - DEPTH[l]
            if 0 <= t < n_hops:
                order.append((t, l))
    first, u = {}, 0
    for t, l in order:
        first[(t, l)] = u
        u += units[l]
    return order, first, u


def decode_diag_closed_form(u, n_hops, units):   # chain_decode_diag
    per_hop = sum(units)

    def size(d):
        return sum(units[l] for l in range(5) if 0 <= d - DEPTH[l] < n_hops)
    d, r, found = 0, u, False
    while d < 3:
        if r < size(d):
            found = True
            break
        r -= size(d)
        d += 1
    if not found and n_hops > 3:
        q = r // per_hop
        if q < n_hops - 3:
            d, r, found = 3 + q, r - q * per_hop, True
        else:
            r -= (n_hops - 3) * per_hop
            d = n_hops
    while not found:
        if r < size(d):
            break
        r -= size(d)
        d += 1
    for l in range(5):
        t = d - DEPTH[l]
        nl = units[l] if 0 <= t < n_hops else 0
        if r < nl:
            return t, l, r
        r -= nl
    raise AssertionError("unit index out of range")


@pytest.mark.parametrize("n_hops", [1, 2, 3, 4, 5, 8, 13, 32])
@pytest.mark.parametrize("units", [(8, 8, 8, 8, 2), (128, 128, 128, 128, 32), (1, 1, 1, 1, 1)])
def test_anti_diagonal_order_is_topological_and_decodes(n_hops, units):
    order, first, total = diag_table(n_hops, units)
    assert len(order) == 5 * n_hops and total == n_hops * sum(units)
    for (t, l) in order:
        lo = first[(t, l)]
        if DEP[l] >= 0:                                    # the layer below at this hop: all of its units come earlier
            assert first[(t, DEP[l])] + units[DEP[l]] <= lo
        if t > 0:                                          # the layer's own previous hop
            assert first[(t - 1, l)] + units[l] <= lo
    seen = set()
    for u in range(total):
        t, l, r = decode_diag_closed_form(u, n_hops, units)
        assert first[(t, l)] + r == u and 0 <= r < units[l]
        seen.add((t, l, r))
    assert len(seen) == total


@pytest.mark.parametrize("n_hops", [1, 2, 7])
def test_hop_major_order_is_topological(n_hops):
    units = (8, 8, 8, 8, 2)
    idx = {}
    u = 0
    for t, l in itertools.product(range(n_hops), range(5)):
        idx[(t, l)] = u
        u += units[l]
    for (t, l), lo in idx.items():
        if DEP[l] >= 0:
            assert idx[(t, DEP[l])] + units[DEP[l]] <= lo
        if t > 0:
            assert idx[(t - 1, l)] + units[l] <= lo


def chain_is_diagonal(n_active, sm):         # tc_gru_chain: a.diag = (tiles_mp * (512 / HT) < sm_count), HT = 64
    return -(-n_active // 128) * (512 // 64) < sm


@pytest.mark.parametrize("sm,first", [(132, 2049), (114, 1793), (128, 1921), (136, 2049), (8, 1)])
def test_first_hop_major_size(sm, first):
    """tests/util.first_hop_major, which the GPU tests size their hop-major cases with, is the chain's switch: H100 SXM
    (132 SMs) and PCIe (114 SMs), and SM counts on and next to a multiple of 8."""
    from util import first_hop_major
    assert first_hop_major(sm) == first
    assert not chain_is_diagonal(first, sm)
    assert first == 1 or chain_is_diagonal(first - 1, sm)
    assert not chain_is_diagonal(16384, sm)
