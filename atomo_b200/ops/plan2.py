"""Planner of the overlapped / sharded bf16 engine (``runtime/shadow_engine.py``, kernels ``csrc/v2_*.cu``).

What changes against ``ops/plan.py`` (the fp32-flat plan of round 1):

* **Where the bytes live.**  Conv / linear weights are bf16 *leaf* tensors in the memory format cuDNN wants
  (``channels_last``: physical ``[O][kh*kw][I]``), carved out of one symmetric-heap region (``wshadow``); the
  fp32 master copy and the optimizer state exist only on the parameter-server owner of each tile.  1-D
  parameters (BN, biases) stay fp32 (``vparams`` / ``vgrads`` regions).  Weight gradients are read by the
  coding kernels *where autograd leaves them* (bf16, same physical layout, address taken from a pointer
  table): no cast / re-layout / accumulate kernels between cuDNN and the coder.
* **Coding units.**  The reference matricizes a conv gradient ``(O,I,kh,kw)`` to ``(O*I/2, 2*kh*kw)``
  (``/root/reference/src/codings/svd.py:12-28``).  In the ``[O][K][I]`` layout one output channel is a
  contiguous *slab* of ``K*I`` values holding ``I/2`` rows of that matrix (row ``(o, ri)``, column ``(b, k)``
  = ``X_o[k][2*ri + b]``): kind ``SLAB``.  2-D tensors (fc, 1x1 convs) are handled in their tall orientation
  and cut into column blocks of <= 64 columns, each block an independent unit (kind ``MAT``) whose complete
  Gram/Jacobi SVD is exact — a block-spectral atomic decomposition (atoms of different blocks are orthogonal
  in the Frobenius inner product), so the ATOMO estimator stays exactly unbiased for square-ish layers
  without a truncated range finder.  Odd-``I`` convs (the 3-channel stem) and anything skinny travel dense.
* **Groups.**  Units are grouped by backward order; each group is encoded and pushed as soon as its last
  gradient exists, while backward continues (the reference's only overlap design,
  ``/root/reference/src/model_ops/resnet_split.py:259-360``).
* **Owners.**  Parameter-server work is sharded: PS tile ``j`` of a group belongs to owner ``j % n_owners``;
  a worker stores the ``U`` rows of a tile into that owner's arena only.  ``n_owners == 1`` is the
  reference's centralized PS.
* **Quantizing codes** (``code="qsgd" | "terngrad"``, see :func:`build_plan2`): every >= 2-D weight is one
  ``QSGD`` unit whose buckets are quantized and bit-packed by the workers straight into the owners' arenas; the
  owners decode, sum and step the optimizer in one launch per group.
* **Scaled sign** (``code="sign"``): every >= 2-D weight is one ``SIGN`` unit whose buckets are sent as one bit per
  element and one fp32 scale, in the slot and tile geometry of the quantizing codes.
* **FP8** (``code="fp8"``): every >= 2-D weight is one ``FP8`` unit whose buckets are sent as one e4m3 byte per
  element (stochastically rounded) and one power-of-two fp32 scale, in the geometry of the sign units.
* **PowerSGD** (``code="powersgd"``): every >= 2-D weight with ``r (O + C) < O C`` is one ``POWER`` unit, the whole
  ``[O][C]`` matrix of its physical layout, sent as a rank-``r`` pair ``P_hat`` / ``Q'`` from one warm-started power
  step; the owners reconstruct ``P_hat Q'^T`` and step the optimizer.
* **Entry-wise ATOMO** (``code="entrywise"``): every >= 2-D weight is one ``ENTRY`` unit whose sampled entries are
  compacted by the workers into 4-byte words in the owners' arenas; the owners scatter-add, average and step the
  optimizer in one launch per group.

Pure Python (unit-testable on CPU).  Struct layouts mirror ``csrc/v2_common.cuh``.
"""
from __future__ import annotations

import math
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

KIND_SLAB, KIND_MAT, KIND_DENSE16, KIND_VEC, KIND_QSGD, KIND_ENTRY, KIND_SIGN, KIND_POWER, KIND_FP8 = \
    1, 2, 3, 4, 5, 6, 7, 8, 9
RCAP_MAX = 32
MAX_COLS = 64
BLOCK_COLS = 32               # column-block width of MAT units (Jacobi cost ~ cols^3 sits in the encode launch)
PS_TILE_ELEMS = 4608          # >= one slab of a 512-channel 3x3 conv
PS_MAX_ROWS = 256
DENSE_TILE_ELEMS = 4096
ENC_TILE_BYTES = 18432        # target bytes of gradient per encode tile
MAX_WORKERS = 16
MAX_GROUPS = 8
W_ALIGN = 64                  # bf16 elements (128 B)
V_ALIGN = 32                  # fp32 elements (128 B)
QSGD_TILE_ELEMS = 4096        # a QSGD PS / encode tile holds max(1, 4096 // bucket) whole buckets
QSGD_MAX_BUCKET = 1024        # one warp quantizes one bucket, staged in shared memory
QSGD_MAX_LEVEL = 14           # (sign + 1) << q | level must fit 16 bits
SIGN_MIN_BUCKET, SIGN_MAX_BUCKET = 64, 4096   # scaled sign and fp8: whole 64-bit words, at most one tile
ENTRY_TILE_ELEMS = 4096       # entry-wise PS / encode tile: the element offset of an entry fits 12 bits
TOPK_STATE_INTS, TOPK_HI_BINS, TOPK_LO_BINS = 8, 256, 128   # top-k selection state / histograms (csrc/v2_common.cuh)
POWER_MAX_RANK = 4            # PowerSGD: rank r in [1, 4] (csrc/v2_powersgd.cu keeps r x 8 accumulators per thread)
PW_ENC_ROWS = 8               # PowerSGD pass A (P = M Q_w, Gram partial) and the EF / stats passes: rows per tile
PW_COL_BLOCK = 256            # PowerSGD pass B (Q' = M^T P_hat): columns per CTA, every row summed inside the CTA
PW_PS_ROWS = 4                # PowerSGD PS tile: rows of the reconstructed matrix
PW_GRAM = 16                  # fp64 Gram partial per pass-A tile (4 x 4)

UNIT_FMT = "<4q20i"           # 112 bytes, mirrors struct Unit2
TILE_FMT = "<4i"              # unit, a, b, owner
UNIT_BYTES = struct.calcsize(UNIT_FMT)
TILE_BYTES = struct.calcsize(TILE_FMT)
CTRL2_FMT = "<iiffffiiQffffiiii"   # mirrors struct Ctrl2 (72 bytes)
CTRL2_BYTES = struct.calcsize(CTRL2_FMT)


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


def slot_u_off(rcap: int, cols: int) -> int:
    return _round_up(4 + rcap + rcap * cols, 4)


def slot_floats(rows: int, cols: int, rcap: int, ubits: int = 0) -> int:
    """Slot size in floats.  ``ubits == 8`` (QSVD): U is stored as int8 [rows][rcap] followed by one fp32 scale per
    row instead of fp32 [rows][rcap]."""
    if ubits == 8:
        return _round_up(slot_u_off(rcap, cols) + _round_up(rows * rcap // 4, 4) + rows, 32)
    return _round_up(slot_u_off(rcap, cols) + rows * rcap, 32)


def slot_scale_off(rows: int, cols: int, rcap: int) -> int:
    """Float offset (inside the slot) of the per-row scales of an int8 U."""
    return slot_u_off(rcap, cols) + _round_up(rows * rcap // 4, 4)


def qsgd_words_per_bucket(bucket: int, q: int) -> int:
    """``L = ceil(bucket / E)`` 64-bit words per bucket, ``E = 64 // (2 + q)`` codes per word (codings/qsgd.py)."""
    e = 64 // (2 + q)
    return (bucket + e - 1) // e


def qsgd_norms_off(n_ps: int) -> int:
    """Float offset (inside a QSGD slot) of the bucket norms: after one int32 step stamp per PS tile."""
    return _round_up(n_ps, 4)


def qsgd_words_off(n_ps: int, buckets: int) -> int:
    """Float offset (inside a QSGD slot) of the uint64 words (16-byte aligned)."""
    return qsgd_norms_off(n_ps) + _round_up(buckets, 4)


def qsgd_slot_floats(n_ps: int, buckets: int, words_per_bucket: int) -> int:
    return _round_up(qsgd_words_off(n_ps, buckets) + 2 * buckets * words_per_bucket, 32)


def pw_phat_off(n_ps: int) -> int:
    """Float offset (inside a PowerSGD slot) of ``P_hat^T`` (``[r][round4(O)]``): after one int32 step stamp per PS
    tile."""
    return _round_up(n_ps, 4)


def pw_q_off(n_ps: int, rows: int, rank: int) -> int:
    """Float offset (inside a PowerSGD slot) of ``Q'^T`` (``[r][round4(C)]``)."""
    return pw_phat_off(n_ps) + rank * _round_up(rows, 4)


def pw_slot_floats(n_ps: int, rows: int, cols: int, rank: int) -> int:
    return _round_up(pw_q_off(n_ps, rows, rank) + rank * _round_up(cols, 4), 32)


def pw_scratch_floats(rows: int, cols: int, rank: int) -> int:
    """Worker-local fp32 state of a PowerSGD unit (from ``gpart_off``): ``P^T``, ``P_hat^T`` (``[r][round4(O)]`` each),
    ``Q'^T`` and the warm ``Q_w^T`` (``[r][round4(C)]`` each)."""
    return 2 * rank * (_round_up(rows, 4) + _round_up(cols, 4))


def entry_hdr_off(j: int) -> int:
    """Float offset (inside an entry slot) of PS tile ``j``'s header {int32 step stamp, int32 count, fp32 scale, pad}."""
    return 4 * j


def entry_words_off(n_ps: int, j: int, ps_rows: int = ENTRY_TILE_ELEMS) -> int:
    """Float offset (inside an entry slot) of PS tile ``j``'s uint32 entries (16-byte aligned)."""
    return 4 * n_ps + j * ps_rows


def entry_slot_floats(numel: int, n_ps: int, ps_rows: int = ENTRY_TILE_ELEMS) -> int:
    """Headers, then room for one entry per element of every tile (a tile never overflows)."""
    last = numel - (n_ps - 1) * ps_rows
    return _round_up(entry_words_off(n_ps, n_ps - 1, ps_rows) + _round_up(last, 4), 32)


def entry_atoms(budget: float, numel: int) -> float:
    """Expected atoms ``s`` of a tensor: ``budget * numel`` for a fraction, else ``budget``, clamped to
    ``[1, numel]`` (``codings.entrywise.EntryWise.atoms_for``)."""
    s = budget * numel if budget < 1.0 else budget
    return float(min(max(s, 1.0), numel))


def topk_atoms(budget: float, numel: int) -> int:
    """``k`` of a top-k unit: ``floor(s)`` of :func:`entry_atoms` (``codings.topk.TopK.k_for``), at least 1."""
    return int(math.floor(entry_atoms(budget, numel)))


def slot_capacity(cols: int, rank: int, systematic: bool) -> int:
    if rank <= 0:
        cap = cols
    elif systematic:
        cap = min(cols, rank)
    else:
        cap = min(cols, 2 * rank + 2)
    return min(_round_up(max(cap, 1), 4), RCAP_MAX)


@dataclass
class Param2:
    """One model parameter as the engine stores it."""
    index: int
    shape: Tuple[int, ...]
    is_w: bool              # bf16 shadow (dim >= 2) vs fp32 vector
    off: int                # element offset in wshadow (bf16) or vparams (fp32)
    numel: int
    widx: int = -1          # index among W params (gradient pointer table)
    group: int = 0

    def phys_strides(self) -> Tuple[int, ...]:
        """Element strides of the bf16 leaf tensor inside wshadow (channels_last for 4-D)."""
        s = self.shape
        if len(s) == 4:
            o, i, kh, kw = s
            return (i * kh * kw, 1, kw * i, i)
        st, acc = [], 1
        for d in reversed(s):
            st.append(acc)
            acc *= d
        return tuple(reversed(st))


@dataclass
class Unit2:
    index: int
    kind: int
    param: int              # Param2.index
    pidx: int               # gradient pointer table index (W params) or -1
    w_off: int              # element offset of the unit's base in wshadow / master (or vparams for VEC)
    g_off: int              # element offset inside the parameter's own gradient tensor
    rows: int = 0
    cols: int = 0
    K: int = 0
    I: int = 0
    rs: int = 0
    cs: int = 0
    rcap: int = 0
    budget: float = 0.0
    numel: int = 0
    group: int = 0
    slot_off: int = 0
    gpart_off: int = 0
    enc_tile0: int = 0
    n_enc: int = 0
    ps_rows: int = 0
    own0: int = 0
    ps_tile0: int = 0
    n_ps: int = 0
    ts_index: int = -1      # index among coded units (vsel / selcount / counters); QSGD / ENTRY: among those units
    ubits: int = 0          # 0: U stored fp32; 8: QSVD, U stochastically rounded to int8 with a per-row scale

    def pack(self) -> bytes:
        return struct.pack(UNIT_FMT, self.w_off, self.g_off, self.slot_off, self.gpart_off, self.kind, self.pidx,
                           self.rows, self.cols, self.K, self.I, self.rs, self.cs, self.rcap,
                           struct.unpack("<i", struct.pack("<f", self.budget))[0], self.numel, self.group,
                           self.enc_tile0, self.n_enc, self.ps_rows, self.own0, self.ps_tile0, self.n_ps,
                           self.ts_index, self.ubits)

    @property
    def coded(self) -> bool:
        return self.kind in (KIND_SLAB, KIND_MAT)


@dataclass
class Plan2:
    params: List[Param2]
    units: List[Unit2]
    enc_tiles: List[Tuple[int, int, int, int]]        # (unit, a, b, idx in unit)  SLAB: slab0, nslabs; MAT: row0, nrows;
    #                                                                       DENSE16: elem0, nelem (staging copy)
    ps_tiles: List[Tuple[int, int, int, int]]         # (unit, a, b, owner) sorted by (group, owner)
    enc_range: List[Tuple[int, int]]                  # per group: (first tile, count)
    ps_range: List[List[Tuple[int, int]]]             # [group][owner] -> (first tile, count)
    group_units: List[List[int]]
    n_groups: int
    n_owners: int
    w_total: int            # bf16 elements of wshadow
    v_total: int            # fp32 elements of vparams / vgrads
    stage_total: int        # bf16 elements of the dense-16 staging region
    arena_floats: int
    gpart_floats: int
    n_coded: int            # units with per-unit device state (coded SLAB / MAT units, or the QSGD / ENTRY / SIGN / FP8 units)
    rank: int
    code: str
    pw_tiles: List[Tuple[int, int, int, int]] = field(default_factory=list)   # PowerSGD pass B: (unit, col0, ncols, j)
    pw_range: List[Tuple[int, int]] = field(default_factory=list)             # per group: (first pw tile, count)

    def units_bytes(self) -> bytes:
        return b"".join(u.pack() for u in self.units)

    @staticmethod
    def tiles_bytes(tiles) -> bytes:
        return b"".join(struct.pack(TILE_FMT, *t) for t in tiles) or b"\0" * TILE_BYTES

    def factor_bytes_per_worker(self) -> int:
        return sum(4 * (4 + u.rcap + u.rcap * u.cols) + (u.rows * (u.rcap + 4) if u.ubits == 8 else 4 * u.rows * u.rcap)
                   for u in self.units if u.coded)

    def qsgd_bytes(self) -> int:
        """Bytes of quantized gradient a worker pushes per step: the uint64 words and fp32 norms of every bucket
        (the same sizes as ``codings.qsgd``'s ``words`` and ``norms``; for sign units ``codings.sign``'s ``words`` and
        ``scales``; for fp8 units ``codings.fp8``'s ``bytes`` and ``scales``)."""
        return sum(8 * u.rows * u.cols + 4 * u.rows for u in self.units if u.kind in (KIND_QSGD, KIND_SIGN, KIND_FP8))

    def powersgd_bytes(self) -> int:
        """Bytes of PowerSGD factors a worker pushes per step: ``4 r (O + C)`` per coded tensor, ``P_hat`` and ``Q'``
        sent once to the tensor's single owner, for any number of owners.  The 4-byte step stamps per PS tile are not
        counted."""
        return sum(4 * u.rcap * (u.rows + u.cols) for u in self.units if u.kind == KIND_POWER)

    def entry_bytes(self) -> float:
        """Bytes of entry-wise code a worker pushes per step: 4 per expected atom and a 16-byte header per PS tile.
        An upper bound on the expectation (``sum(p_i) <= s``), exact when no ``p_i`` is clamped to 1.  Top-k: an
        upper bound on the realized bytes, exact when every tensor has at least ``k`` non-zero entries."""
        return sum(4.0 * u.budget + 16.0 * u.n_ps for u in self.units if u.kind == KIND_ENTRY)

    def expected_factor_bytes(self) -> float:
        """Bytes actually stored per worker and step for the expected number of atoms (U is written in groups
        of 4 atoms); for the quantizing codes the words and norms of the QSGD units; for entry-wise ATOMO the
        entries and tile headers."""
        tot = float(self.qsgd_bytes()) + self.entry_bytes() + float(self.powersgd_bytes())
        for u in self.units:
            if u.coded:
                atoms = min(u.budget if u.budget > 0 else u.cols, u.cols)
                a4 = min(u.rcap, _round_up(int(atoms + 0.999), 4))
                tot += 4 * (4 + u.rcap + u.rcap * u.cols) + (u.rows * (a4 + 4) if u.ubits == 8 else 4 * u.rows * a4)
        return tot

    def dense_bytes(self) -> int:
        return sum((2 if u.kind == KIND_DENSE16 else 4) * u.numel for u in self.units
                   if not u.coded and u.kind not in (KIND_QSGD, KIND_ENTRY, KIND_SIGN, KIND_POWER, KIND_FP8))


def default_groups(shapes: Sequence[Sequence[int]], n_groups: int) -> List[int]:
    """Assign parameters to backward groups.  ``parameters()`` order ~ forward order, so the LAST parameters
    form group 0 (their gradients exist first).

    What matters is what is left on the critical path after the last ``wgrad``: the encode -> project -> PS chain
    of the FINAL group.  So the final group is only the first weight tensor of the network (for the CNNs here the
    3-channel stem, which travels dense: a staging copy + two PS tiles), the group before it is the next few
    percent of the weights (its chain hides behind the stem's backward), and the early groups — where almost all
    bytes are — close once the share still to come drops below ``0.5 * 0.3**g``.  A 1-D parameter (BN, bias)
    joins the group of the weight tensor that precedes it in forward order (its gradient exists earlier)."""
    numels = []
    for s in shapes:
        n = 1
        for d in s:
            n *= int(d)
        numels.append(n if len(s) >= 2 else 0)
    total = sum(numels) or 1
    n_groups = max(1, min(n_groups, MAX_GROUPS))
    w_idx = [i for i, n in enumerate(numels) if n > 0]
    groups = [0] * len(shapes)
    reserve_last = n_groups >= 3 and len(w_idx) >= n_groups
    body = n_groups - 1 if reserve_last else n_groups
    acc, g = 0, 0
    for i in range(len(shapes) - 1, -1, -1):
        groups[i] = g
        acc += numels[i]
        if numels[i] > 0 and g < body - 1 and (total - acc) / total <= 0.5 * 0.3 ** g:
            g += 1
    if reserve_last:
        groups[w_idx[0]] = g + 1
    last_w = None
    for i, s in enumerate(shapes):
        if len(s) >= 2:
            last_w = groups[i]
        elif last_w is not None:
            groups[i] = last_w
    used = sorted(set(groups))
    remap = {g: k for k, g in enumerate(used)}
    return [remap[g] for g in groups]


def build_plan2(shapes: Sequence[Sequence[int]], code: str = "svd", rank: int = 3, systematic: bool = False,
                n_owners: int = 1, n_groups: int = 4, groups: Optional[Sequence[int]] = None,
                block_cols: int = BLOCK_COLS, min_coded_numel: int = 256, quantization_level: int = 4,
                bucket_size: int = 512, entry_budget: float = 0.05) -> Plan2:
    """Plan of the bf16 engine for ``code`` in ``svd | qsvd | sgd | qsgd | terngrad | entrywise | topk | sign |
    powersgd | fp8``.

    ``qsgd`` / ``terngrad``: every >= 2-D weight (the 3-channel stem and the fc layers included) is exactly one
    ``KIND_QSGD`` unit; there are no ``DENSE16`` units.  1-D parameters stay ``KIND_VEC`` (fp32, summed by
    ``multimem.ld_reduce``) exactly as under ``svd`` — unlike the round-1 engine, which quantizes the BN and bias
    vectors too.  Per tensor:

    * buckets run over the PHYSICAL element order of the bf16 weight (``[O][kh][kw][I]`` for convs, the order
      of ``wshadow`` and of the gradients); ``bucket = min(bucket_size, numel)`` exactly as
      ``codings/qsgd.py::_bucketize``, the tail bucket is zero-padded;
    * packing is the coder's: ``E = 64 // (2 + q)`` codes per word, section-major, ``L = ceil(bucket / E)``
      words per bucket.  The result is the coder's estimator applied to the physical-order flat tensor: it is
      not bit-identical to the round-1 path, which buckets the logical OIHW order;
    * one PS tile (also one encode CTA) holds ``max(1, 4096 // bucket)`` whole buckets; tile ``j`` of a group
      belongs to owner ``j % n_owners`` as for every other kind.  ``ps_tiles`` entries are (unit, first element,
      element count, owner);
    * the unit's slot in a worker arena (same offset in every owner's arena; a worker writes only the tiles that
      owner owns) holds one int32 step stamp per PS tile, the fp32 norms of all buckets and the 16-byte aligned
      uint64 words of all buckets (``qsgd_norms_off`` / ``qsgd_words_off``).

    ``Unit2`` fields of a QSGD unit: ``K`` = bucket, ``I`` = q, ``rows`` = buckets, ``cols`` = words per bucket,
    ``rs`` = 1 for TernGrad, ``cs`` = buckets per tile, ``ps_rows`` = elements per tile (``csrc/v2_common.cuh``).

    ``entrywise``: every >= 2-D weight is exactly one ``KIND_ENTRY`` unit; 1-D parameters stay ``KIND_VEC`` as above
    (the round-1 engine samples them too).  Per tensor:

    * ``budget`` = the expected atom count ``s`` of ``codings.entrywise`` (:func:`entry_atoms` of ``entry_budget``);
    * tiles of ``ENTRY_TILE_ELEMS`` elements run over the physical element order; encode tile == PS tile, and tile
      ``j`` of a group belongs to owner ``j % n_owners``.  ``ps_tiles`` entries are (unit, first element, element
      count, owner);
    * the slot holds a 16-byte header per tile, then room for one uint32 entry per element of every tile
      (:func:`entry_hdr_off` / :func:`entry_words_off`), so a tile cannot overflow.

    ``topk``: the units, tiles, owners, slots and headers of ``entrywise``, with ``budget = k`` (:func:`topk_atoms`, an
    integer: the exact number of entries pushed when the tensor has at least ``k`` non-zeros).

    ``sign``: every >= 2-D weight is exactly one ``KIND_SIGN`` unit; 1-D parameters stay ``KIND_VEC``.  Buckets, tiles,
    owners and slots are those of ``qsgd`` with ``bucket = min(bucket_size, numel)`` (``bucket_size`` a multiple of 64
    in ``[64, 4096]``) and ``L = ceil(bucket / 64)`` words per bucket: one bit per element (``codings/sign.py``) in
    place of the quantized codes and one fp32 scale per bucket in place of the norm.  ``Unit2`` fields: ``K`` = bucket,
    ``rows`` = buckets, ``cols`` = L, ``cs`` = buckets per tile, ``ps_rows`` = elements per tile, ``I`` = ``rs`` = 0.

    ``fp8``: the units, buckets, tiles, owners and slots of ``sign`` (kind ``KIND_FP8``) with ``cols`` =
    ``ceil(bucket / 8)`` uint64 words per bucket: one e4m3 byte per element in element order, bucket ``j`` starting at
    byte ``8 j cols``, and one power-of-two fp32 scale per bucket in place of the norm (``codings/fp8.py``).

    ``powersgd`` (``rank`` = r in ``[1, 4]``): every >= 2-D weight with ``r (O + C) < O C`` is exactly one ``KIND_POWER``
    unit (``codings/powersgd.py``), the others travel ``DENSE16``; 1-D parameters stay ``KIND_VEC``.  Per unit:

    * ``rows`` = O, ``cols`` = C = numel / O (row ``o`` is the contiguous physical slab of output channel ``o``),
      ``rcap`` = ``budget`` = r, ``K`` = pass-B tiles;
    * pass-A encode tiles (``enc_tiles``) of ``PW_ENC_ROWS`` rows: (unit, first row, rows, index in unit); each leaves a
      16-double Gram partial (indexed by global encode tile) that the unit's last tile sums in tile order;
    * pass-B tiles (``pw_tiles`` / ``pw_range``) of ``PW_COL_BLOCK`` columns: (unit, first column, columns, index in
      unit); each sums ``Q' = M^T P_hat`` over all rows of its columns inside one CTA, so no ``Q'`` partials exist;
    * PS tiles of ``PW_PS_ROWS`` rows: (unit, first row, rows, owner).  Every PS tile of a unit belongs to ONE owner,
      ``own0`` (every tile needs all of ``Q'``, so spreading a unit over owners would send ``Q'`` to each of them); the
      units of a group go to the owner with the fewest PowerSGD elements of that group so far (lowest index on ties);
    * the slot holds one int32 step stamp per PS tile, ``P_hat^T`` and ``Q'^T`` (:func:`pw_phat_off` /
      :func:`pw_q_off`), written into owner ``own0``'s arena only;
    * ``gpart_off`` locates the worker-local scratch (:func:`pw_scratch_floats`) inside the ``gpart`` region.
    """
    shapes = [tuple(int(d) for d in s) for s in shapes]
    quant = code in ("qsgd", "terngrad")
    entry = code in ("entrywise", "topk")
    sign = code == "sign"
    fp8 = code == "fp8"
    if entry and not entry_budget > 0:
        raise ValueError("entry_budget must be positive (a fraction of numel below 1, else an atom count)")
    if quant:
        q, bsz = int(quantization_level), int(bucket_size)
        if not 1 <= q <= QSGD_MAX_LEVEL:
            raise ValueError("quantization_level must be in [1, %d]" % QSGD_MAX_LEVEL)
        if not (32 <= bsz <= QSGD_MAX_BUCKET and bsz % 8 == 0):
            raise ValueError("bucket_size must be a multiple of 8 in [32, %d]" % QSGD_MAX_BUCKET)
    if sign or fp8:
        sbsz = int(bucket_size)
        if not (SIGN_MIN_BUCKET <= sbsz <= SIGN_MAX_BUCKET and sbsz % 64 == 0):
            raise ValueError("%s: bucket_size must be a multiple of 64 in [%d, %d]"
                             % (code, SIGN_MIN_BUCKET, SIGN_MAX_BUCKET))
    power = code == "powersgd"
    if power and not 1 <= int(rank) <= POWER_MAX_RANK:
        raise ValueError("powersgd: svd_rank must be in [1, %d] (got %r)" % (POWER_MAX_RANK, rank))
    ubits = 0
    if code == "qsvd":          # QSVD: spectral atoms with quantized left factors (README.md:141-142 of the reference)
        code, ubits = "svd", 8
    if groups is None:
        groups = default_groups(shapes, n_groups)
    n_groups = max(groups) + 1 if groups else 1
    params: List[Param2] = []
    w_off = v_off = 0
    widx = 0
    for i, s in enumerate(shapes):
        numel = 1
        for d in s:
            numel *= d
        if len(s) >= 2:
            params.append(Param2(i, s, True, w_off, numel, widx, groups[i]))
            w_off += _round_up(numel, W_ALIGN)
            widx += 1
        else:
            params.append(Param2(i, s, False, v_off, numel, -1, groups[i]))
            v_off += _round_up(numel, V_ALIGN)

    units: List[Unit2] = []
    stage_off = 0

    def add(u: Unit2):
        u.index = len(units)
        units.append(u)

    for p in params:
        if not p.is_w:
            add(Unit2(0, KIND_VEC, p.index, -1, p.off, 0, numel=p.numel, group=p.group))
            continue
        s = p.shape
        if quant:
            bucket = min(bsz, p.numel)
            nb = (p.numel + bucket - 1) // bucket
            bpt = max(1, QSGD_TILE_ELEMS // bucket)
            add(Unit2(0, KIND_QSGD, p.index, p.widx, p.off, 0, rows=nb, cols=qsgd_words_per_bucket(bucket, q),
                      K=bucket, I=q, rs=1 if code == "terngrad" else 0, cs=bpt, numel=p.numel, group=p.group,
                      ps_rows=bpt * bucket))
            continue
        if sign:
            bucket = min(sbsz, p.numel)
            bpt = max(1, QSGD_TILE_ELEMS // bucket)
            add(Unit2(0, KIND_SIGN, p.index, p.widx, p.off, 0, rows=(p.numel + bucket - 1) // bucket,
                      cols=(bucket + 63) // 64, K=bucket, cs=bpt, numel=p.numel, group=p.group, ps_rows=bpt * bucket))
            continue
        if fp8:
            bucket = min(sbsz, p.numel)
            bpt = max(1, QSGD_TILE_ELEMS // bucket)
            add(Unit2(0, KIND_FP8, p.index, p.widx, p.off, 0, rows=(p.numel + bucket - 1) // bucket,
                      cols=(bucket + 7) // 8, K=bucket, cs=bpt, numel=p.numel, group=p.group, ps_rows=bpt * bucket))
            continue
        if power:
            o = s[0]
            c = p.numel // o
            if rank * (o + c) < o * c:
                add(Unit2(0, KIND_POWER, p.index, p.widx, p.off, 0, rows=o, cols=c, K=-(-c // PW_COL_BLOCK),
                          rcap=int(rank), budget=float(rank), numel=p.numel, group=p.group, ps_rows=PW_PS_ROWS))
                continue
        if entry:
            s_atoms = entry_atoms(float(entry_budget), p.numel)
            if code == "topk":
                s_atoms = float(topk_atoms(float(entry_budget), p.numel))
            add(Unit2(0, KIND_ENTRY, p.index, p.widx, p.off, 0, budget=s_atoms,
                      numel=p.numel, group=p.group, ps_rows=ENTRY_TILE_ELEMS))
            continue
        coded = code == "svd" and p.numel >= min_coded_numel
        if coded and len(s) == 4 and s[2] * s[3] > 1:
            o, i, kh, kw = s
            k = kh * kw
            if i % 16 == 0 and 2 * k <= MAX_COLS and o * i // 2 >= 2 * k and k * i <= PS_TILE_ELEMS:
                add(Unit2(0, KIND_SLAB, p.index, p.widx, p.off, 0, rows=o * i // 2, cols=2 * k, K=k, I=i,
                          rcap=slot_capacity(2 * k, rank, systematic), budget=float(rank), numel=p.numel,
                          group=p.group))
                continue
            coded = False
        if coded:
            # 2-D physical matrix [O][I] (Linear, 1x1 conv in channels_last): tall orientation, column blocks
            o = s[0]
            i = p.numel // o
            if o >= i:
                rows, cols, rs, cs = o, i, i, 1
            else:
                rows, cols, rs, cs = i, o, 1, i
            # a trailing 1-column block (cols % block_cols == 1) has no eigenproblem to solve: such tensors (none in
            # the model zoo) travel dense instead of exercising a degenerate unit in the kernels
            if cols >= 2 and cols % block_cols != 1:
                nb = (cols + block_cols - 1) // block_cols
                bud = float(rank) if nb == 1 else float(max(1, -(-rank // nb)))
                for b in range(nb):
                    c0 = b * block_cols
                    bc = min(block_cols, cols - c0)
                    add(Unit2(0, KIND_MAT, p.index, p.widx, p.off + c0 * cs, c0 * cs, rows=rows, cols=bc, rs=rs,
                              cs=cs, rcap=slot_capacity(bc, int(bud), systematic), budget=bud, numel=rows * bc,
                              group=p.group))
                continue
        u = Unit2(0, KIND_DENSE16, p.index, p.widx, p.off, 0, numel=p.numel, group=p.group)
        u.rs = stage_off                      # offset of the staging copy (bf16 elements)
        stage_off += _round_up(p.numel, W_ALIGN)
        add(u)

    # ---- tiles, slots ---------------------------------------------------------------------------------
    enc_tiles: List[Tuple[int, int, int, int]] = []
    ps_by_group: List[List[Tuple[int, int, int]]] = [[] for _ in range(n_groups)]
    enc_range, group_units = [], [[] for _ in range(n_groups)]
    pw_tiles: List[Tuple[int, int, int, int]] = []
    pw_range: List[Tuple[int, int]] = []
    slot_off = gpart_off = 0
    n_coded = 0
    for g in range(n_groups):
        first, pw_first = len(enc_tiles), len(pw_tiles)
        pw_load = [0] * n_owners            # PowerSGD elements of this group per owner
        for u in units:
            if u.group != g:
                continue
            group_units[g].append(u.index)
            u.enc_tile0 = len(enc_tiles)
            if u.kind == KIND_SLAB:
                slab_bytes = u.K * u.I * 2
                ns = max(1, ENC_TILE_BYTES // slab_bytes)
                nslabs = u.rows // (u.I // 2)
                for s0 in range(0, nslabs, ns):
                    enc_tiles.append((u.index, s0, min(ns, nslabs - s0), s0 // ns))
                spt = max(1, min(PS_TILE_ELEMS // (u.K * u.I), PS_MAX_ROWS // (u.I // 2)))
                u.ps_rows = spt * (u.I // 2)
            elif u.kind == KIND_MAT:
                npad = (u.cols + 3) // 4 * 4
                er = max(64, min(1024, 8192 // npad) // 64 * 64)      # fp32 staging tile <= 32 KB
                for r0 in range(0, u.rows, er):
                    enc_tiles.append((u.index, r0, min(er, u.rows - r0), r0 // er))
                nc4 = (u.cols + 3) // 4
                u.ps_rows = max(8, min(PS_MAX_ROWS, PS_TILE_ELEMS // u.cols) & ~7)
            elif u.kind == KIND_DENSE16:
                for e0 in range(0, u.numel, 8192):     # staging copy tiles
                    enc_tiles.append((u.index, e0, min(8192, u.numel - e0), 0))
            elif u.kind in (KIND_QSGD, KIND_ENTRY, KIND_SIGN, KIND_FP8):   # encode tiles = PS tiles (one owner per CTA)
                for j, e0 in enumerate(range(0, u.numel, u.ps_rows)):
                    enc_tiles.append((u.index, e0, min(u.ps_rows, u.numel - e0), j))
            elif u.kind == KIND_POWER:
                for j, r0 in enumerate(range(0, u.rows, PW_ENC_ROWS)):
                    enc_tiles.append((u.index, r0, min(PW_ENC_ROWS, u.rows - r0), j))
                for j, c0 in enumerate(range(0, u.cols, PW_COL_BLOCK)):
                    pw_tiles.append((u.index, c0, min(PW_COL_BLOCK, u.cols - c0), j))
            u.n_enc = len(enc_tiles) - u.enc_tile0
            if u.kind in (KIND_QSGD, KIND_ENTRY, KIND_SIGN, KIND_FP8):
                u.ts_index = n_coded
                n_coded += 1
                u.ps_tile0 = len(ps_by_group[g])
                for e0 in range(0, u.numel, u.ps_rows):
                    ps_by_group[g].append((u.index, e0, min(u.ps_rows, u.numel - e0)))
                u.n_ps = len(ps_by_group[g]) - u.ps_tile0
                u.own0 = u.ps_tile0 % n_owners
                u.slot_off = slot_off
                if u.kind in (KIND_QSGD, KIND_SIGN, KIND_FP8):
                    slot_off += qsgd_slot_floats(u.n_ps, u.rows, u.cols)
                else:
                    slot_off += entry_slot_floats(u.numel, u.n_ps, u.ps_rows)
            elif u.kind == KIND_POWER:
                u.ts_index = n_coded
                n_coded += 1
                u.ps_tile0 = len(ps_by_group[g])
                for r0 in range(0, u.rows, u.ps_rows):
                    ps_by_group[g].append((u.index, r0, min(u.ps_rows, u.rows - r0)))
                u.n_ps = len(ps_by_group[g]) - u.ps_tile0
                u.own0 = min(range(n_owners), key=lambda o: (pw_load[o], o))
                pw_load[u.own0] += u.numel
                u.slot_off = slot_off
                slot_off += pw_slot_floats(u.n_ps, u.rows, u.cols, u.rcap)
                u.gpart_off = gpart_off
                gpart_off += pw_scratch_floats(u.rows, u.cols, u.rcap)
            elif u.coded:
                u.ts_index = n_coded
                n_coded += 1
                u.ubits = ubits
                u.slot_off = slot_off
                slot_off += slot_floats(u.rows, u.cols, u.rcap, ubits)
                u.gpart_off = gpart_off
                gpart_off += u.n_enc * u.cols * u.cols
                u.ps_tile0 = len(ps_by_group[g])
                for r0 in range(0, u.rows, u.ps_rows):
                    ps_by_group[g].append((u.index, r0, min(u.ps_rows, u.rows - r0)))
                u.n_ps = len(ps_by_group[g]) - u.ps_tile0
                u.own0 = u.ps_tile0 % n_owners
            else:
                u.ps_tile0 = len(ps_by_group[g])
                for e0 in range(0, u.numel, DENSE_TILE_ELEMS):
                    ps_by_group[g].append((u.index, e0, min(DENSE_TILE_ELEMS, u.numel - e0)))
                u.n_ps = len(ps_by_group[g]) - u.ps_tile0
                u.own0 = u.ps_tile0 % n_owners
        enc_range.append((first, len(enc_tiles) - first))
        pw_range.append((pw_first, len(pw_tiles) - pw_first))

    ps_tiles: List[Tuple[int, int, int, int]] = []
    ps_range: List[List[Tuple[int, int]]] = []
    for g in range(n_groups):
        row = []
        for o in range(n_owners):
            first = len(ps_tiles)
            for j, (ui, a, b) in enumerate(ps_by_group[g]):
                own = units[ui].own0 if units[ui].kind == KIND_POWER else j % n_owners
                if own == o:
                    ps_tiles.append((ui, a, b, o))
            row.append((first, len(ps_tiles) - first))
        ps_range.append(row)
    return Plan2(params, units, enc_tiles, ps_tiles, enc_range, ps_range, group_units, n_groups, n_owners,
                 max(w_off, W_ALIGN), max(v_off, V_ALIGN), max(stage_off, W_ALIGN), max(slot_off, 32),
                 max(gpart_off, 1), n_coded, rank, code, pw_tiles, pw_range)


def owner_of_row(u: Unit2, row: int, n_owners: int) -> int:
    """Owner of the PS tile that holds tall row ``row`` of a coded unit (what project_push computes)."""
    return (u.own0 + row // u.ps_rows) % n_owners


# error feedback (csrc/v2_feedback.cu): the apply pass runs over the weight tensors of a group in chunks of
# EF_CHUNK_ELEMS elements, one CTA each; EfChunk = {residual offset of the tensor, pointer-table index, first element,
# element count, pad}
EF_CHUNK_ELEMS = 8192
EF_CHUNK_FMT = "<qiiii"


def ef_chunks(plan: "Plan2") -> Tuple[bytes, List[Tuple[int, int]]]:
    """Packed apply chunks of every weight tensor, grouped by backward group, and (first chunk, chunk count) per
    group.  1-D vectors travel exactly in fp32 and have no residual."""
    rows: List[Tuple[int, int, int, int]] = []
    ranges: List[Tuple[int, int]] = []
    for g in range(plan.n_groups):
        first = len(rows)
        for q in plan.params:
            if q.is_w and q.group == g:
                rows.extend((q.off, q.widx, s, min(EF_CHUNK_ELEMS, q.numel - s))
                            for s in range(0, q.numel, EF_CHUNK_ELEMS))
        ranges.append((first, len(rows) - first))
    return b"".join(struct.pack(EF_CHUNK_FMT, o, w, s, c, 0) for o, w, s, c in rows), ranges


OPT_SGD, OPT_ADAM, OPT_AMSGRAD = 0, 1, 2


def pack_ctrl2(step: int = 1, lr: float = 0.01, momentum: float = 0.0, dampening: float = 0.0,
               weight_decay: float = 0.0, nesterov: bool = False, first_step: int = 1, seed: int = 1,
               beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-8, opt: int = OPT_SGD,
               num_aggregate: int = 0) -> bytes:
    return struct.pack(CTRL2_FMT, step, 0, lr, momentum, dampening, weight_decay, int(nesterov), first_step,
                       seed & 0xFFFFFFFFFFFFFFFF, beta1, beta2, eps, 0.0, int(opt), int(num_aggregate), 0, 0)
