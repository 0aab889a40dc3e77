"""Host-side planning for the grouped sm_90a kernels.

Turns a model's parameter list into the descriptor tables the kernels walk
(``csrc/common.cuh``: ``LayerDesc``, ``TileDesc``, ``Ctrl``) and the slot layout
of a worker's arena in PS peer memory.  Pure Python — unit-testable on CPU.

Routing (what the reference does per tensor vs. what is sent here):

* matricization follows ``codings.svd.matricize_shape`` (svd.py:12-28);
* the factorization always works on the *tall* orientation (rows >= cols); a
  wide matrix such as fc ``(10, 512)`` is handled as its transpose through the
  ``row_stride/col_stride`` fields, no copy;
* ``cols <= 32`` (or ``<= 64`` when really tall) -> ``ROUTE_SVD_TS``: complete
  Gram/Jacobi SVD (every 3x3 / 5x5 conv of the model zoo: cols = 18 / 50);
* 1-D tensors (BN, biases; rank <= 2) travel dense: coding them costs more
  bytes than the tensor itself (SURVEY.md 2.4, consequence 2);
* square-ish layers (fc, 1x1 convs) -> ``ROUTE_LOWRANK_EXT`` when ``subspace``
  is on: randomized range finder of width ``sketch`` on the wgmma skinny
  GEMMs, then the same Gram/Jacobi machinery on auxiliary plans (``ExtPlan``);
  otherwise dense.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

from ..codings.svd import matricize_shape

ROUTE_DENSE, ROUTE_SVD_TS, ROUTE_LOWRANK_EXT = 0, 1, 2
RCAP_MAX = 32
TS_MAX_COLS = 64
PS_TILE_ELEMS = 4096
PS_MAX_ROWS = 256
PS_DENSE_ELEMS = 4096
ALIGN_ELEMS = 32

LAYER_FMT = "<qqq12i"   # 72 bytes, mirrors struct LayerDesc
TILE_FMT = "<4i"        # 16 bytes, mirrors struct TileDesc
CTRL_FMT = "<iiffffiiQIIII"  # 56 bytes, mirrors struct Ctrl
LAYER_BYTES = struct.calcsize(LAYER_FMT)
TILE_BYTES = struct.calcsize(TILE_FMT)
CTRL_BYTES = struct.calcsize(CTRL_FMT)


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


def slot_u_off(rcap: int, cols: int) -> int:
    return _round_up(4 + rcap + rcap * cols, 4)


def slot_floats(rows: int, cols: int, rcap: int) -> int:
    return _round_up(slot_u_off(rcap, cols) + rows * rcap, 32)


def slot_capacity(cols: int, rank: int, systematic: bool) -> int:
    """Atoms a slot must hold.  Bernoulli sampling has a random count with
    mean <= rank; the kernel resamples on overflow, so 2r+2 keeps that rare."""
    if rank <= 0:
        cap = cols
    elif systematic:
        cap = min(cols, rank)
    else:
        cap = min(cols, 2 * rank + 2)
    return min(_round_up(max(cap, 1), 4), RCAP_MAX)


@dataclass
class Layer:
    index: int
    shape: Tuple[int, ...]
    off: int
    numel: int
    rows: int
    cols: int
    row_stride: int
    col_stride: int
    route: int
    rcap: int = 0
    slot_off: int = 0
    gpart_off: int = 0
    ts_index: int = -1
    tile0: int = 0
    ntiles: int = 0
    vec_ok: int = 0
    ps_rows: int = 0
    sketch: int = 0      # ROUTE_LOWRANK_EXT: subspace width l
    ext_index: int = -1

    def pack(self) -> bytes:
        return struct.pack(LAYER_FMT, self.off, self.slot_off, self.gpart_off, self.numel, self.rows, self.cols,
                           self.row_stride, self.col_stride, self.route, self.rcap, self.ts_index, self.tile0,
                           self.ntiles, self.vec_ok, self.ps_rows)


@dataclass
class Plan:
    layers: List[Layer]
    enc_tiles: List[Tuple[int, int, int, int]]    # tall-skinny encode tiles (layer,row0,nrows,0)
    ps_tiles: List[Tuple[int, int, int, int]]     # PS update tiles (low-rank + dense)
    dense_tiles: List[Tuple[int, int, int, int]]  # every layer tiled flat (entry-wise / dense-only configs)
    ts_layers: List[int]
    total_elems: int
    arena_floats: int
    gpart_floats: int
    code: str
    rank: int
    ext: Optional["ExtPlan"] = None

    def layers_bytes(self) -> bytes:
        return b"".join(l.pack() for l in self.layers)

    @staticmethod
    def tiles_bytes(tiles) -> bytes:
        return b"".join(struct.pack(TILE_FMT, *t) for t in tiles)

    def factor_bytes_per_worker(self) -> int:
        """Bytes one worker pushes per step on the low-rank routes (expected, at slot capacity)."""
        return sum(4 * (4 + l.rcap + l.rcap * l.cols + l.rows * l.rcap) for l in self.layers if l.route != ROUTE_DENSE)

    def dense_bytes(self) -> int:
        return sum(4 * l.numel for l in self.layers if l.route == ROUTE_DENSE)


def tall_orientation(shape: Sequence[int]):
    """(rows, cols, row_stride, col_stride) of the tall view of the matricized tensor."""
    m, n = matricize_shape(shape)
    if n <= m:
        return m, n, n, 1
    return n, m, 1, n


def _ps_rows_for(cols: int) -> int:
    nc4 = (min(cols, TS_MAX_COLS) + 3) // 4
    r = min(PS_MAX_ROWS, PS_TILE_ELEMS // max(cols, 1), 1024 // nc4)
    return max(4, r & ~3)


def _enc_rows_for(cols: int) -> int:
    r = max(64, min(2048, 16384 // max(cols, 1)))
    return r // 64 * 64


def build_plan(shapes: Sequence[Sequence[int]], code: str = "svd", rank: int = 3, systematic: bool = False,
               dense_vectors: bool = True, offsets: Optional[Sequence[int]] = None, subspace: bool = False,
               ext_min_numel: int = 16384) -> Plan:
    layers: List[Layer] = []
    off = 0
    for i, shape in enumerate(shapes):
        shape = tuple(int(d) for d in shape)
        numel = 1
        for d in shape:
            numel *= d
        this_off = offsets[i] if offsets is not None else off
        rows, cols, rs, cs = tall_orientation(shape)
        route = ROUTE_DENSE
        if code == "svd":
            is_vector = len(shape) <= 1
            # tall-skinny Gram/Jacobi path: cols <= 32 always; 32 < cols <= 64 only when really
            # tall (the Jacobi cost grows ~cols^3 and sits on the critical path)
            skinny = cols <= 32 or (cols <= TS_MAX_COLS and rows >= 8 * cols)
            if not (is_vector and dense_vectors) and cols >= 2 and rows >= cols and skinny:
                route = ROUTE_SVD_TS
            elif (not is_vector) and subspace and cols > 32 and numel >= ext_min_numel:
                route = ROUTE_LOWRANK_EXT
        layers.append(Layer(i, shape, this_off, numel, rows, cols, rs, cs, route))
        off = this_off + _round_up(numel, ALIGN_ELEMS)
    total = max(off, ALIGN_ELEMS)

    enc_tiles, ps_tiles, dense_tiles, ts_layers, ext_layers = [], [], [], [], []
    slot_off, gpart_off = 0, 0
    for l in layers:
        if l.route == ROUTE_SVD_TS:
            l.rcap = slot_capacity(l.cols, rank, systematic)
            l.slot_off = slot_off
            slot_off += slot_floats(l.rows, l.cols, l.rcap)
            l.ts_index = len(ts_layers)
            ts_layers.append(l.index)
            er = _enc_rows_for(l.cols)
            l.tile0 = len(enc_tiles)
            for r0 in range(0, l.rows, er):
                enc_tiles.append((l.index, r0, min(er, l.rows - r0), 0))
            l.ntiles = len(enc_tiles) - l.tile0
            l.gpart_off = gpart_off
            gpart_off += l.ntiles * l.cols * l.cols
            l.vec_ok = 1 if (l.col_stride == 1 and l.row_stride == l.cols and l.off % 4 == 0) else 0
            l.ps_rows = _ps_rows_for(l.cols)
            for r0 in range(0, l.rows, l.ps_rows):
                ps_tiles.append((l.index, r0, min(l.ps_rows, l.rows - r0), 0))
        elif l.route == ROUTE_LOWRANK_EXT:
            l.sketch = 16 if rank <= 6 else 32
            l.rcap = slot_capacity(l.sketch, rank, systematic)
            l.slot_off = slot_off
            slot_off += slot_floats(l.rows, l.cols, l.rcap)
            l.ext_index = len(ext_layers)
            ext_layers.append(l)
            # vectorised epilogue along whichever direction is contiguous in memory
            if l.col_stride == 1:
                l.vec_ok = 2 if (l.cols % 4 == 0 and l.row_stride % 4 == 0 and l.off % 4 == 0) else 0
            else:
                l.vec_ok = 3 if (l.row_stride == 1 and l.col_stride % 4 == 0 and l.off % 4 == 0) else 0
            l.ps_rows = _ps_rows_for(TS_MAX_COLS)
            for r0 in range(0, l.rows, l.ps_rows):
                for c0 in range(0, l.cols, TS_MAX_COLS):
                    ps_tiles.append((l.index, r0, min(l.ps_rows, l.rows - r0), c0))
        else:
            for e0 in range(0, l.numel, PS_DENSE_ELEMS):
                ps_tiles.append((l.index, e0 // 4, min(PS_DENSE_ELEMS, l.numel - e0), 0))
        for e0 in range(0, l.numel, PS_DENSE_ELEMS):
            dense_tiles.append((l.index, e0 // 4, min(PS_DENSE_ELEMS, l.numel - e0), 0))
    plan = Plan(layers, enc_tiles, ps_tiles, dense_tiles, ts_layers, total, max(slot_off, 32), max(gpart_off, 1),
                code, rank)
    if ext_layers:
        plan.ext = build_ext_plan(ext_layers, rank, systematic)
    return plan


# ----------------------------------------------------------------------------------------------
# Subspace-iteration route (ROUTE_LOWRANK_EXT): square-ish layers (fc, 1x1 convs)
# ----------------------------------------------------------------------------------------------
EXT_FMT = "<8q8i"  # mirrors struct ExtDesc (96 bytes)
EXT_BYTES = struct.calcsize(EXT_FMT)
FIN_ROWS = 256


@dataclass
class ExtPlan:
    """Scratch layout + auxiliary tall-skinny plans for the randomized range finder.

    Per layer A (m x n, tall view):  Y = A X (m x l)  ->  Q = orth(Y)  ->  B = A^T Q (n x l)
    ->  B = Ub S Vb^T  (complete SVD of the skinny B through the Gram/Jacobi kernels, atoms sampled
    there)  ->  A ~ (Q Vb) S Ub^T.  ``aux_y`` / ``aux_b`` describe Y and B as tall-skinny "layers" of
    a scratch buffer so the SAME gram / eig_sample / project kernels orthonormalise and factorise them.
    """
    layers: List[Layer]
    descs: List[tuple]
    aux_y: "Plan"
    aux_b: "Plan"
    scratch_floats: int
    local_arena_floats: int
    fin_tiles: List[Tuple[int, int, int, int]]
    xt_range: Tuple[int, int] = (0, 0)
    y_range: Tuple[int, int] = (0, 0)
    b_range: Tuple[int, int] = (0, 0)

    def descs_bytes(self) -> bytes:
        return b"".join(struct.pack(EXT_FMT, *d) for d in self.descs)


def _aux_plan(entries, rank, systematic, topk_all: bool) -> Plan:
    """entries: (off, rows, cols, rcap). Builds a TS-only plan over a scratch buffer."""
    layers, enc_tiles, ts_layers = [], [], []
    slot_off = gpart_off = 0
    for i, (off, rows, cols, rcap) in enumerate(entries):
        l = Layer(i, (rows, cols), off, rows * cols, rows, cols, cols, 1, ROUTE_SVD_TS)
        l.rcap = rcap
        l.slot_off = slot_off
        slot_off += slot_floats(rows, cols, rcap)
        l.ts_index = i
        ts_layers.append(i)
        er = _enc_rows_for(cols)
        l.tile0 = len(enc_tiles)
        for r0 in range(0, rows, er):
            enc_tiles.append((i, r0, min(er, rows - r0), 0))
        l.ntiles = len(enc_tiles) - l.tile0
        l.gpart_off = gpart_off
        gpart_off += l.ntiles * cols * cols
        layers.append(l)
    total = max([l.off + l.numel for l in layers] + [ALIGN_ELEMS])
    return Plan(layers, enc_tiles, [], [], ts_layers, total, max(slot_off, 32), max(gpart_off, 1), "svd", rank)


def build_ext_plan(ext_layers: List[Layer], rank: int, systematic: bool) -> ExtPlan:
    # scratch = [all X^T | all Y | all B]: each group can be (re)initialised with ONE launch
    xt_total = sum(_round_up(l.sketch * l.cols, ALIGN_ELEMS) for l in ext_layers)
    y_total = sum(_round_up(l.rows * l.sketch, ALIGN_ELEMS) for l in ext_layers)
    b_total = sum(_round_up(l.cols * l.sketch, ALIGN_ELEMS) for l in ext_layers)
    xt_cur, y_cur, b_cur = 0, xt_total, xt_total + y_total
    scratch = xt_total + y_total + b_total
    descs, y_entries, b_entries, fin_tiles = [], [], [], []
    for l in ext_layers:
        sk = l.sketch
        xt_off = xt_cur; xt_cur += _round_up(sk * l.cols, ALIGN_ELEMS)
        y_off = y_cur; y_cur += _round_up(l.rows * sk, ALIGN_ELEMS)
        b_off = b_cur; b_cur += _round_up(l.cols * sk, ALIGN_ELEMS)
        y_entries.append((y_off, l.rows, sk, sk))        # orthonormalise: keep all l atoms
        b_entries.append((b_off, l.cols, sk, l.rcap))    # factorise + sample
        descs.append([l.off, xt_off, y_off, b_off, 0, 0, l.slot_off, 0,
                      l.rows, l.cols, l.row_stride, l.col_stride, sk, l.rcap, l.index, 0])
        for r0 in range(0, l.rows, FIN_ROWS):
            fin_tiles.append((l.ext_index, r0, min(FIN_ROWS, l.rows - r0), 0))
    aux_y = _aux_plan(y_entries, rank, systematic, True)
    aux_b = _aux_plan(b_entries, rank, systematic, False)
    for d, ly, lb in zip(descs, aux_y.layers, aux_b.layers):
        d[4], d[5] = ly.slot_off, lb.slot_off  # Q slot / B slot inside their local arenas
    ep = ExtPlan(ext_layers, [tuple(d) for d in descs], aux_y, aux_b, max(scratch, 32),
                 aux_y.arena_floats + aux_b.arena_floats, fin_tiles)
    ep.xt_range, ep.y_range, ep.b_range = (0, xt_total), (xt_total, xt_total + y_total), (xt_total + y_total, scratch)
    return ep


def dense_only_plan(shapes, offsets=None) -> Plan:
    return build_plan(shapes, code="sgd", offsets=offsets)


def pack_ctrl(step: int = 1, lr: float = 0.01, momentum: float = 0.0, dampening: float = 0.0,
              weight_decay: float = 0.0, nesterov: bool = False, first_step: int = 1, seed: int = 1) -> bytes:
    return struct.pack(CTRL_FMT, step, 0, lr, momentum, dampening, weight_decay, int(nesterov), first_step,
                       seed & 0xFFFFFFFFFFFFFFFF, 0, 0, 0, 0)
