"""The shared-memory map of riccati_bwd_kernel (riccati_wb.cuh), read from the header on the CPU (tests/emu/ricwb_layout_emu.cu).  Each of the
kernel's two lanes carves one map: [P | p] (later [Q~ | q~]), [A | b | B], W (later Yl, [K | k] and, in the columns of W_B, [S~ | r~]), R~
(later L^-1) and the landing buffer of R; one mbarrier per lane follows the two maps.  Every region holds the largest operand the kernel
writes into it, the operands that share a region never overlap while both are live, and two lanes fit one block.  The extents are restated
from the operand shapes of the kernel's GEMM calls and copies."""
import ctypes as C

import numpy as np
import pytest

from emu_build import build

NX, NM = 58, 23
NX1 = NX + 1
LIMIT = 227 * 1024   # a block's opt-in shared memory on sm_90, static shared memory included
FIELDS = ("lanes", "lane_d", "pq_off", "ab_off", "w_off", "rt_off", "rin_off", "smem_d", "smem_bytes", "static_bytes", "ldw", "ldm", "yl_d",
          "kout_off", "y_off", "threads", "lane_threads")


def extent(rows, cols, ld):
    """doubles spanned by a column-major rows x cols block at leading dimension ld"""
    return (cols - 1) * ld + rows


@pytest.fixture(scope="module")
def L():
    lib = C.CDLL(str(build("ricwb_layout_emu.cu", "libricwbemu.so")))
    out = np.zeros(len(FIELDS), np.int64)
    lib.emu_ricwb_layout(out.ctypes.data_as(C.POINTER(C.c_longlong)))
    return dict(zip(FIELDS, (int(x) for x in out)))


def regions(L):
    """(name, start, size) of one lane's regions, in the order the kernel carves them"""
    names = ["pq", "ab", "w", "rt", "rin"]
    starts = [L[f"{n}_off"] for n in names] + [L["lane_d"]]
    return [(n, starts[i], starts[i + 1] - starts[i]) for i, n in enumerate(names)]


def test_every_region_holds_its_largest_operand(L):
    lx, lm = L["ldw"], L["ldm"]
    size = {n: s for n, _, s in regions(L)}
    assert size["pq"] >= extent(NX, NX1, NX)                 # [P | p] and [Q~ | q~], dense (ld 58)
    assert size["ab"] >= extent(NX, NX1 + NM, NX)            # [A | b | B] as the bulk copy lands it (ld 58)
    assert size["w"] >= extent(NX, NX1 + NM, lx)             # W = P [A | b | B]
    assert size["rt"] >= extent(NM, NM, lm)                  # R~, then L^-1
    assert size["rin"] >= extent(NM, NM, lm)                 # R from the cp.async
    assert lx >= NX and lm >= NM and lx % 8 == 4 and lm % 8 == 4


def test_operands_sharing_w_do_not_overlap(L):
    """[S~ | r~] (ld 23) is written into the columns of W_B once R~ is formed, and is read by P3 while [Yl | yl] (ld 28, at 0) is written;
    P4 reads Yl while [K | k] (ld 23, at kout) is written; P5 reads [K | k].  None of them may reach another."""
    lx, lm = L["ldw"], L["ldm"]
    w = regions(L)[2][2]
    assert L["y_off"] == lx * NX1                                        # the first column of W_B: W_A and the column b stay intact
    assert L["y_off"] + extent(NM, NX1, NM) <= extent(NX, NX1 + NM, lx)  # S~ fits the W_B columns
    assert L["yl_d"] >= extent(NM, NX1, lm) and L["kout_off"] >= L["yl_d"]
    assert L["kout_off"] + extent(NM, NX1, NM) <= L["y_off"]            # [K | k] stays below S~
    assert L["y_off"] + extent(NM, NX1, NM) <= w


def test_two_lanes_fit_one_block(L):
    assert L["lanes"] == 2 and L["threads"] == L["lanes"] * L["lane_threads"] == 320
    regs = regions(L)
    assert regs[0][1] == 0 and all(a[1] + a[2] == b[1] for a, b in zip(regs, regs[1:]))
    # every region and every lane starts on a 16-byte boundary (the bulk copies); the mbarriers (8 bytes each) follow the lanes
    assert all(start % 2 == 0 for _, start, _ in regs) and L["lane_d"] % 2 == 0
    assert L["smem_d"] == L["lanes"] * L["lane_d"] + L["lanes"]
    assert L["smem_bytes"] == 8 * L["smem_d"]
    assert L["smem_bytes"] + L["static_bytes"] <= LIMIT, (L["smem_bytes"], L["static_bytes"])
