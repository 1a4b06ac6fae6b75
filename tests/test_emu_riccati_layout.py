"""The shared-memory layouts of the generic Riccati kernels (riccati_layout_padded for riccati_kernel, riccati_layout for riccati_cluster_kernel)
on the CPU harness (tests/emu/bld_emu.cu), for every (nx, nu_max) with 0 < nx <= 64 and 0 < nu_max <= 32: each region holds the largest
operand the kernels write into it, the regions tile the block's dynamic shared memory, and b200sqp_qp_create accepts exactly the sizes whose
layouts fit one block in both variants.  The extents below are restated from the operand shapes of the kernels' GEMM calls and copies.

This is the guard of the layout: a [K | k] that runs past W into Y[0] changes the cluster kernel's results only at a few sizes (the overflow
lands in columns of Y[0] that the writing CTA does not read, while a cp.async into Y[0] may still be in flight), so the GPU tests alone would
not hold it."""
import itertools

import pytest

import bld_emu_lib

SIZES = list(itertools.product(range(1, 65), range(1, 33)))
LIMIT = 227 * 1024 - 16   # a block's opt-in shared memory on sm_90, less the kernels' 16 bytes of static shared memory
# sizes whose one-CTA layout takes at most 227 KB but whose cluster layout does not fit
CLUSTER_TOO_BIG = [(57, 28), (58, 26), (58, 27), (58, 28), (59, 25), (59, 26), (59, 27), (59, 28), (60, 24), (60, 25), (60, 26), (60, 27)]


def even_up(n):
    return (n + 1) & ~1


def extent(rows, cols, ld):
    """doubles spanned by a column-major rows x cols block at leading dimension ld"""
    return (cols - 1) * ld + rows


def regions(L, cluster):
    """the kernel's regions in the order it carves them from its dynamic shared memory (name, size)"""
    r = [("PQ0", L["pq"]), ("PQ1", L["pq"]), ("AB0", L["ab"]), ("AB1", L["ab"]), ("W", L["w"]), ("Y0", L["y"]), ("Y1", L["y"]),
         ("Rs0", L["rs"]), ("Rs1", L["rs"]), ("Linv", L["linv"]), ("vec", L["vec"])]
    return r + [("Rg", L["rs"]), ("Yg", L["y"])] if cluster else r


def check_layout(nx, nm, L, lx, lm, cluster):
    """every write of the kernel into its regions stays inside them; lx / lm: the leading dimensions of the nx-row / nm-row operands of the
    backward sweep"""
    nx1 = nx + 1
    need = {
        # [P | p] and the prefetched [Q | q]
        "pq": extent(nx, nx1, lx),
        # backward [A | b | B] at ld lx; the forward sweep's dense [A | b | B]
        "ab": max(extent(nx, nx1 + nm, lx), nx * (nx1 + nm)),
        # backward [S | r] (and S~, r~) at ld lm; the forward sweep's dense K
        "y": max(extent(nm, nx1, lm), nm * nx),
        # R~ and L^-1
        "rs": extent(nm, nm, lm),
        "linv": extent(nm, nm, lm),
        # x, x+, u, k (double-buffered)
        "vec": 2 * even_up(nx) + 3 * even_up(nm),
    }
    for key, n in need.items():
        assert L[key] >= n, (nx, nm, cluster, key, L[key], n)
    # W: first P [A | b | B] (ld lx); later [Yl | yl] (ld lm) at 0, read while [K | k] (ld nm) is written at kout
    assert L["w"] >= extent(nx, nx1 + nm, lx), (nx, nm, cluster, "W = P [A|b|B]")
    assert L["kout"] >= extent(nm, nx1, lm), (nx, nm, cluster, "[Yl | yl] runs into [K | k]")
    assert L["kout"] + extent(nm, nx1, nm) <= L["w"], (nx, nm, cluster, "[K | k] runs past W", L["kout"], L["w"])
    if cluster:   # the gathered R~ and [S~ | r~]
        assert L["rs"] >= extent(nm, nm, nm) and L["y"] >= extent(nm, nx1, nm), (nx, nm)
    # the regions are carved one after another: disjoint, each starting on a 16-byte boundary (the prefetch's wide cp.async), summing to total
    regs = regions(L, cluster)
    assert all(n % 2 == 0 for _, n in regs), (nx, nm, cluster, regs)
    assert L["kout"] % 2 == 0
    base = sum(n for name, n in regs if name not in ("Rg", "Yg"))
    assert L["total"] == base, (nx, nm, cluster)
    return sum(n for _, n in regs)


@pytest.fixture(scope="module")
def layouts():
    return {s: bld_emu_lib.riccati_layout(*s) for s in SIZES}


def test_every_region_holds_its_largest_operand(layouts):
    for (nx, nm), d in layouts.items():
        lx, lm = d["lx"], d["lm"]
        assert lx >= nx and lm >= nm and lx % 8 == 4 and lm % 8 == 4, (nx, nm, lx, lm)
        assert d["one_doubles"] == check_layout(nx, nm, d["one"], lx, lm, cluster=False)
        assert d["cluster_doubles"] == check_layout(nx, nm, d["cluster"], nx, nm, cluster=True)


def test_qp_create_accepts_exactly_the_sizes_that_fit_both_variants(layouts):
    accepted = set()
    for (nx, nm), d in layouts.items():
        assert d["limit"] == LIMIT
        fits = d["one_doubles"] * 8 <= LIMIT and d["cluster_doubles"] * 8 <= LIMIT
        assert d["supported"] == fits, (nx, nm, d["one_doubles"] * 8, d["cluster_doubles"] * 8)
        if fits:
            accepted.add((nx, nm))
    assert len(accepted) == 1948
    for s in CLUSTER_TOO_BIG:
        d = layouts[s]
        assert d["one_doubles"] * 8 <= 227 * 1024 and d["cluster_doubles"] * 8 > LIMIT and s not in accepted, s
    for s in [(52, 32), (64, 15), (56, 24), (57, 24), (58, 23), (4, 4), (36, 32), (3, 32)]:
        assert s in accepted, s
    for nx, nm in [(0, 1), (1, 0), (65, 1), (1, 33), (-1, 4), (64, 16)]:
        assert not bld_emu_lib.riccati_layout(nx, nm)["supported"], (nx, nm)


def test_whole_body_layout_is_unchanged(layouts):
    """the compile-time layout of the <58, 23> instantiations: their shared memory, and with it the kernels, stay as they are"""
    d = layouts[(58, 23)]
    assert (d["lx"], d["lm"]) == (60, 28)
    assert d["one"]["w"] == d["one"]["ab"] == 4920 and d["one"]["kout"] == 1652 and d["one_doubles"] == 27272
    assert d["cluster"]["w"] == d["cluster"]["ab"] == 4756 and d["cluster"]["kout"] == 1358 and d["cluster_doubles"] == 27502
