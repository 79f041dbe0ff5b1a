"""Byte-exact checks of every data-movement and point-to-point kernel, with guard bands.

Moving data must reproduce bytes exactly, so inputs are seeded random bytes (viewed as floats they
include NaN and -0.0 patterns) and results are compared as raw bytes, never as values. The expected
output is plain CPU slicing and concatenation of every rank's input: each rank draws every rank's
input from CPU generators seeded by (case, rank) and computes the whole expectation itself.

Every output lies inside a region `guard + shift + nbytes + guard` whose bytes are first filled
with a seeded pattern (not a constant: a kernel that writes zeros would match one). After each call
the whole region is compared: the output must hold the payload and everything else, the guards and
the output of a rank that is not a destination, must be byte-identical to the pattern. Registered
and symmetric outputs are views inside one registration with their guards in the same
registration, so a peer's stray store lands in a guard too. Inputs are checked unchanged.

Ranks are threads sharing cuda:0, as in the other GPU tests. The 1 MiB pool (bulk region 512 KiB)
makes the pipelined kernels run at small sizes. Mismatches are collected per rank and reported
together, so the ranks stay in step and one run lists every failing path.
"""
import os
import zlib

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.ops import cuda as gcu

U8 = torch.uint8
STAGE = 1 << 20
GUARD = 64
SHIFTS = (0, 1, 2, 4, 8, 12)
REG_OFFSETS = (0, 16, 4, 1)  # 0 and 16 take the vector paths, 4 and 1 do not
BCAST_DIRECT_MAX = 256 * 1024  # tuning default bcastDirectMaxBytes: mode 0 up to it
VIEW = {1: torch.uint8, 2: torch.int16, 4: torch.float32, 8: torch.float64}  # element-counting APIs


# ---- seeded bytes and the expected layouts (no GPU needed) --------------------------------------

def _gen(key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


_SRC = {}
_SRC_BYTES = 4 << 20


def _seeded(key, n):
    """`n` seeded random bytes for `key`: a slice of a per-key-family source where that is long
    enough (cheap), else a fresh draw."""
    if n + 65536 > _SRC_BYTES:
        return torch.randint(0, 256, (n,), generator=_gen(key), dtype=U8)
    fam = key[0] if isinstance(key, tuple) else key
    src = _SRC.get(fam)
    if src is None:
        src = _SRC.setdefault(fam, torch.randint(0, 256, (_SRC_BYTES,), generator=_gen(("src", fam)), dtype=U8))
    k = zlib.crc32(repr(key).encode()) % 65536
    return src[k:k + n]


def _input(case, r, n):
    """Rank r's input bytes for `case`."""
    return _seeded(("in", case, r), n)


class Region:
    """`guard + shift + nbytes + guard` bytes at `store[start:]`, pre-filled with a seeded pattern;
    `view` is the `nbytes` in the middle. torch views a tensor of `es`-byte elements only at a
    multiple of `es` bytes, so `shift` grows to the next address that allows it."""

    def __init__(self, store, start, shift, nbytes, key, es=1):
        shift += -(store.storage_offset() + start + GUARD + shift) % es
        self.shift, self.lo, self.n = shift, GUARD + shift, nbytes
        self.init = _seeded(("guard", key), 2 * GUARD + shift + nbytes)
        self.mem = store[start:start + self.init.numel()]
        assert self.mem.numel() == self.init.numel(), "region exceeds its store"
        self.mem.copy_(self.init)

    @property
    def view(self):
        return self.mem[self.lo:self.lo + self.n]

    def want(self, payload=None):
        """The region's expected bytes: the pattern, with `payload` in the output if given."""
        w = self.init.clone()
        if payload is not None:
            assert payload.numel() == self.n
            w[self.lo:self.lo + self.n] = payload
        return w


def _plain(nbytes, shift, key, device="cuda", es=1):
    return Region(torch.empty(2 * GUARD + shift + es + nbytes, dtype=U8, device=device), 0, shift, nbytes, key, es)


def _first_diff(got, want, lo, n):
    """None if equal, else where the first differing byte is, relative to the output start."""
    got = got.cpu()
    if got.shape != want.shape:
        return f"shape {tuple(got.shape)} != {tuple(want.shape)}"
    bad = (got != want).nonzero()
    if bad.numel() == 0:
        return None
    i = int(bad[0])
    rel = i - lo
    where = "output" if 0 <= rel < n else ("guard before" if rel < 0 else "guard after")
    return f"{bad.numel()} bytes differ, first at byte {rel} ({where}): got {int(got[i])} want {int(want[i])}"


def _allgatherv_layout(inputs, nbytes):
    """What every rank's allgatherv output holds: rank r's first nbytes[r] bytes, in rank order."""
    return torch.cat([inputs[r][:nbytes[r]] for r in range(len(nbytes))])


def _alltoallv_layout(inputs, table, me):
    """Rank me's alltoallv output: table[q][j] bytes go from rank q to rank j; rank q's block for
    j starts after its blocks for ranks < j, and lands after the blocks from ranks < q."""
    parts = []
    for q in range(len(table)):
        s = sum(table[q][:me])
        parts.append(inputs[q][s:s + table[q][me]])
    return torch.cat(parts) if parts else torch.empty(0, dtype=U8)


def _scatter_layout(root_input, nbytes, me):
    return root_input[me * nbytes:(me + 1) * nbytes]


def test_region_guard_helper():
    """The pattern is seeded (same key, same bytes; other key, other bytes), not constant, and
    `want` changes exactly the output bytes."""
    for shift in SHIFTS:
        for n in (0, 1, 17, 1000):
            a = _plain(n, shift, ("t", n, shift), device="cpu")
            b = _plain(n, shift, ("t", n, shift), device="cpu")
            c = _plain(n, shift, ("u", n, shift), device="cpu")
            assert a.mem.numel() == 2 * GUARD + shift + n and a.lo == GUARD + shift
            assert torch.equal(a.init, b.init) and not torch.equal(a.init, c.init)
            assert torch.unique(a.init[:GUARD]).numel() > 8
            assert _first_diff(a.mem, a.want(), a.lo, n) is None
            p = _seeded(("p", n), n)
            w = a.want(p)
            changed = (w != a.init).nonzero().flatten().tolist()
            assert all(a.lo <= i < a.lo + n for i in changed)
            assert torch.equal(w[a.lo:a.lo + n], p)
            a.view.copy_(p)
            assert _first_diff(a.mem, w, a.lo, n) is None
            # one stray byte on either side is reported as a guard hit
            for off, where in ((-1, "guard before"), (n, "guard after")):
                m = w.clone()
                m[a.lo + off] ^= 0x5A
                assert where in _first_diff(m, w, a.lo, n)


def test_layout_builders_match_a_per_byte_loop():
    P = 4
    g = _gen("layout")
    for trial in range(20):
        nb = torch.randint(0, 40, (P,), generator=g).tolist()
        table = torch.randint(0, 30, (P, P), generator=g).tolist()
        table[trial % P][trial % P] = 0
        inputs = [_input(("layout", trial), r, 200) for r in range(P)]
        # allgatherv / gatherv
        want = []
        for r in range(P):
            for i in range(nb[r]):
                want.append(int(inputs[r][i]))
        assert _allgatherv_layout(inputs, nb).tolist() == want
        # alltoallv
        for me in range(P):
            want = []
            for q in range(P):
                pos = 0
                for j in range(P):
                    for i in range(table[q][j]):
                        if j == me:
                            want.append(int(inputs[q][pos + i]))
                    pos += table[q][j]
            assert _alltoallv_layout(inputs, table, me).tolist() == want
        # scatter
        b = nb[0]
        for me in range(P):
            assert _scatter_layout(inputs[1], b, me).tolist() == [int(inputs[1][me * b + i]) for i in range(b)]


def test_lookup_finds_empty_views():
    """An empty view inside a registration resolves like any other view of it (torch gives empty
    tensors data_ptr() 0): a rank that receives nothing must take its peers' registered path."""
    store = torch.empty(256, dtype=U8)

    class Fake:
        _reg = {store.data_ptr(): (object(), 256)}

    for v in (store[64:64], store[64:64].view(torch.float32), store[255:255], store[3:19]):
        buf, off = gcu.CudaContext.lookup(Fake(), v)
        assert buf is not None and off == v.storage_offset() * v.element_size()
    assert gcu.CudaContext.lookup(Fake(), torch.empty(0, dtype=U8))[0] is None


# ---- GPU helpers ----------------------------------------------------------------------------------

def _cc(ctx, stage=STAGE):
    cc = gcu.CudaContext(ctx, 0, stage_bytes=stage)
    cc.set_timeout(60000)
    return cc


def _limits(cc):
    """Byte limits: the LL limit per block without a tuning-table entry (`ll`) and with one that
    picks LL (`ll_pc`, the LL kernel's own limit), and the pool's bulk region (collectives.cc)."""
    t = gb._C.cuda.get_tuning()
    half = min(-(-max(t["one_shot_max_bytes"], 4096) // 4096) * 4096, STAGE // 4)
    return {"ll": min(t["ll_max_bytes"], cc.pc.ll_max_bytes()), "ll_pc": cc.pc.ll_max_bytes(),
            "bulk": STAGE - 2 * half}


class Checker:
    """Collects mismatches of one rank instead of raising, so that the ranks stay in step."""

    def __init__(self, rank):
        self.rank, self.bad, self.n, self.notes = rank, [], 0, []

    def region(self, what, reg, payload=None):
        self.n += 1
        m = _first_diff(reg.mem, reg.want(payload), reg.lo, reg.n)
        if m is not None:
            self.bad.append(f"rank {self.rank} {what}: {m}")

    def same(self, what, got, want):
        self.n += 1
        m = _first_diff(got, want, 0, want.numel())
        if m is not None:
            self.bad.append(f"rank {self.rank} {what}: {m}")

    def result(self):
        return self.bad, self.n, self.notes


def _report(results):
    bad = [b for r in results for b in r[0]]
    assert sum(r[1] for r in results) > 0
    assert not bad, f"{len(bad)} mismatches:\n" + "\n".join(bad[:60])


def _sync(cc):
    cc.synchronize()


def _set_env(cc, key, value):
    """Change a process-wide setting the ranks read per call: every rank is idle and sees it."""
    _sync(cc)
    cc.pc.host_barrier()
    if cc.rank == 0:
        if value is None:
            os.environ.pop("GLB_" + key, None)
        else:
            os.environ["GLB_" + key] = str(value)
    cc.pc.host_barrier()


def _set_tma(cc, on):
    _sync(cc)
    cc.pc.host_barrier()
    if cc.rank == 0:
        gb._C.cuda.set_tuning({"tma_copies": bool(on)})
    cc.pc.host_barrier()


class Stores:
    """One registered store (16-byte aligned base), one registered store at an odd base address
    (vectorOk false for the whole registration) and one symmetric store per rank. Every region
    starts at byte 0 of its store, so a view's offset inside the registration is GUARD + shift, the
    same on every rank."""

    def __init__(self, cc, nbytes):
        nbytes += 16  # room for the element alignment of Region
        self.reg = torch.empty(nbytes, dtype=U8, device="cuda")
        cc.register(self.reg)
        self._odd_raw = torch.empty(nbytes + 16, dtype=U8, device="cuda")
        self.odd = self._odd_raw[1:1 + nbytes]
        cc.register(self.odd)
        self.sym = cc.empty(nbytes, U8)

    def region(self, kind, shift, nbytes, key, es=1):
        if kind == "plain":
            return _plain(nbytes, shift, key, es=es)
        return Region({"reg": self.reg, "odd": self.odd, "sym": self.sym}[kind], 0, shift, nbytes, key, es)


def _kinds(cc, thorough):
    """(kind, shift) of an output: plain at every shift, registered at the vector and non-vector
    offsets, the odd registration, symmetric."""
    out = [("plain", s) for s in (SHIFTS if thorough else (0, 1, 4))]
    out += [("reg", o) for o in REG_OFFSETS] + [("odd", 0), ("sym", 0), ("sym", 4)]
    return out


def _pick(seq, i):
    return seq[i % len(seq)]


# ---- broadcast ------------------------------------------------------------------------------------

def _bcast_sizes(lim, thorough):
    b = lim["bulk"]
    s = [1, 15, 16, 17, 33, lim["ll"] - 1, lim["ll"] + 1, BCAST_DIRECT_MAX - 16, BCAST_DIRECT_MAX + 16,
         b - 1, b + 1, b * 5 // 2 + 3]
    return s if thorough else [1, 17, 33, BCAST_DIRECT_MAX + 16, b + 1, b * 5 // 2 + 3]


def _bcast_worker(ctx, modes, tiles, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    lim = _limits(cc)
    sizes = _bcast_sizes(lim, thorough)
    st = Stores(cc, 2 * GUARD + 16 + max(sizes))
    roots = list(range(P)) if P <= 4 or thorough else [0, P - 1]
    kinds = _kinds(cc, thorough)
    i = 0
    for mode in modes:
        if mode == 2 and not cc.nvls_available():
            chk.notes.append("mode 2 (multimem) skipped: no NVLS on this context")
            continue
        _set_env(cc, "CUDA_BCAST_MODE", None if mode == "auto" else mode)
        for tile in (tiles if mode == 3 else [0]):
            _set_env(cc, "CUDA_BCAST_TILE", tile or None)
            for n in sizes:
                combos = ([(k, r) for k in kinds for r in roots] if thorough else
                          [(_pick(kinds, i + j), _pick(roots, i + j)) for j in range(max(len(roots), 3))])
                for (kind, shift), root in combos:
                    i += 1
                    case = ("bcast", P, mode, tile, n, kind, shift, root)
                    data = _input(case, root, n)
                    reg = st.region(kind, shift, n, (case, me))
                    if me == root:
                        reg.view.copy_(data)
                    cc.broadcast(reg.view, root=root)
                    _sync(cc)
                    chk.region(f"broadcast mode={mode} tile={tile} n={n} {kind}+{shift} root={root}", reg, data)
    _set_env(cc, "CUDA_BCAST_MODE", None)
    _set_env(cc, "CUDA_BCAST_TILE", None)
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_broadcast_exact(size):
    try:
        _report(gb.spawn_threads(size, _bcast_worker, ["auto", 0, 1, 3], [16, 64], False, cuda_device=0))
    finally:
        os.environ.pop("GLB_CUDA_BCAST_MODE", None)
        os.environ.pop("GLB_CUDA_BCAST_TILE", None)


@pytest.mark.gpu
def test_broadcast_multimem_exact():
    res = None
    try:
        res = gb.spawn_threads(4, _bcast_worker, [2], [0], False, cuda_device=0)
    finally:
        os.environ.pop("GLB_CUDA_BCAST_MODE", None)
    if any(r[2] for r in res):
        pytest.skip(res[0][2][0])
    _report(res)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_broadcast_exact_sweep(size):
    try:
        _report(gb.spawn_threads(size, _bcast_worker, ["auto", 0, 1, 3], [16, 64, 0], True, cuda_device=0))
    finally:
        os.environ.pop("GLB_CUDA_BCAST_MODE", None)
        os.environ.pop("GLB_CUDA_BCAST_TILE", None)


# ---- allgather(v) and gather(v) -------------------------------------------------------------------

def _uneven(P, es, base):
    """Element counts with zeros, and offsets that leave later ranks off the 16-byte grid."""
    pat = [3, 17, 0, 1000, 1, 0, 33, 5]
    return [pat[(q + base) % len(pat)] * (1 if es > 1 else 3) for q in range(P)]


def _gather_cases(P, lim, thorough):
    """(name, es, counts-per-rank in elements, kind, out shift, in shift, env-LL-disable)."""
    cases = []
    ll, bulk = lim["ll"], lim["bulk"]
    for es in (1, 2, 4, 8):
        # LL: equal sizes up to the LL limit, on both sides of it (both limits, see _limits)
        for nb in ((1, 15, 16, 17, 33, ll - 1, ll, ll + 1) if es == 1 else (16, ll // es * es)):
            cases.append(("ll", es, [nb // es] * P, "plain", 0, 0, False))
        cases.append(("ll_over", es, [(ll + 16) // es] * P, "plain", 4, 0, False))
        if lim["ll_pc"] * P <= bulk * 2:
            for nb in ((lim["ll_pc"] - 1, lim["ll_pc"] + 1) if es == 1 else (lim["ll_pc"] + es,)):
                cases.append(("ll_pc", es, [nb // es] * P, "plain", _pick(SHIFTS, nb), 0, False))
        if es == 1:
            cases.append(("staged_bulk-1", 1, [(bulk - 1) // P] * P, "plain", 2, 1, False))
        # the same small sizes with LL disabled: the staged push
        for nb in (1, 17, 33) if es == 1 else (16, 48):
            cases.append(("no_ll", es, [nb // es or 1] * P, "plain", 1 if es == 1 else 2, 4, True))
        # staged allgatherv, uneven
        cases.append(("staged_v", es, _uneven(P, es, 0), "plain", 8, 12, False))
        # registered: vector and non-vector offsets, odd base
        for j, (kind, off) in enumerate([("reg", o) for o in REG_OFFSETS] + [("odd", 0), ("sym", 0)]):
            cases.append(("reg", es, _uneven(P, es, j), kind, off, _pick(SHIFTS, j + es), False))
        # pipelined: larger than the bulk region in total, uneven
        per = (bulk // P + 17) // es
        cases.append(("pipelined", es, [per + 7 * q * (q % 2) for q in range(P)], "plain", 4, 1, False))
        cases.append(("pipelined_bulk+1", es, [(bulk + 1) // es // P + (1 if q == 0 else 0) for q in range(P)],
                      "plain", 0, 0, False))
    if thorough:
        for so in SHIFTS:
            for si in SHIFTS:
                cases.append(("shifts", 1, _uneven(P, 1, so + si), "plain", so, si, False))
                cases.append(("shifts_pipelined", 1, [(bulk // P + 33 + q) for q in range(P)], "plain", so, si, False))
    return cases


def _allgather_worker(ctx, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    lim = _limits(cc)
    cases = _gather_cases(P, lim, thorough)
    st = Stores(cc, 2 * GUARD + 16 + max(sum(c[2]) * c[1] for c in cases))
    ll_off = None
    for ci, (name, es, counts, kind, so, si, no_ll) in enumerate(cases):
        if no_ll != ll_off:
            _set_env(cc, "CUDA_LL_DISABLE", 1 if no_ll else None)
            ll_off = no_ll
        dt = VIEW[es]
        nb = [c * es for c in counts]
        case = ("ag", P, ci)
        inputs = [_input(case, r, nb[r]) for r in range(P)]
        want = _allgatherv_layout(inputs, nb)
        for inplace in ((False, True) if kind in ("plain", "reg") else (False,)):
            out = st.region(kind, so, sum(nb), (case, me, inplace), es)
            o = out.view.view(dt)
            if inplace:
                lo = sum(nb[:me])
                out.view[lo:lo + nb[me]].copy_(inputs[me])
                inp, ireg = o[lo // es:lo // es + counts[me]], None
            else:
                ireg = _plain(nb[me], si, (case, "in", me), es=es)
                ireg.view.copy_(inputs[me])
                inp = ireg.view.view(dt)
            uniform = len(set(counts)) == 1
            if uniform:
                cc.allgather(o, inp)
            else:
                cc.allgatherv(o, inp, counts)
            _sync(cc)
            what = f"allgather{'' if uniform else 'v'} {name} es={es} counts={counts} out={kind}+{out.shift} " + \
                   ("in place" if inplace else f"in+{ireg.shift}")
            chk.region(what, out, want)
            if ireg is not None:
                chk.region(what + " (input)", ireg, inputs[me])
    _set_env(cc, "CUDA_LL_DISABLE", None)
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_allgather_exact(size):
    try:
        _report(gb.spawn_threads(size, _allgather_worker, False, cuda_device=0))
    finally:
        os.environ.pop("GLB_CUDA_LL_DISABLE", None)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_allgather_exact_sweep(size):
    try:
        _report(gb.spawn_threads(size, _allgather_worker, True, cuda_device=0))
    finally:
        os.environ.pop("GLB_CUDA_LL_DISABLE", None)


def _gather_worker(ctx, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    lim = _limits(cc)
    cases = [c for c in _gather_cases(P, lim, thorough) if not c[6]]
    st = Stores(cc, 2 * GUARD + 16 + max(sum(c[2]) * c[1] for c in cases))
    roots = list(range(P)) if thorough else sorted({0, P - 1})
    for ci, (name, es, counts, kind, so, si, _) in enumerate(cases):
        dt = VIEW[es]
        nb = [c * es for c in counts]
        for root in roots:
            case = ("ga", P, ci, root)
            inputs = [_input(case, r, nb[r]) for r in range(P)]
            ireg = _plain(nb[me], si, (case, "in", me), es=es)
            ireg.view.copy_(inputs[me])
            # a registered root output: every rank passes its copy of the registered tensor;
            # a plain one: non-roots alternate between None and a plain tensor
            none = kind == "plain" and me != root and ci % 2 == 0
            out = None if none else st.region(kind, so, sum(nb), (case, me), es)
            o = None if none else out.view.view(dt)
            uniform = len(set(counts)) == 1
            if uniform:
                cc.gather(o, ireg.view.view(dt), root=root)
            else:
                cc.gatherv(o, ireg.view.view(dt), counts, root=root)
            _sync(cc)
            what = f"gather{'' if uniform else 'v'} {name} es={es} counts={counts} root={root} out={kind}+{so} in+{ireg.shift}"
            if out is not None:
                chk.region(what, out, _allgatherv_layout(inputs, nb) if me == root else None)
            chk.region(what + " (input)", ireg, inputs[me])
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_gather_exact(size):
    _report(gb.spawn_threads(size, _gather_worker, False, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [3, 8])
def test_gather_exact_sweep(size):
    _report(gb.spawn_threads(size, _gather_worker, True, cuda_device=0))


# ---- alltoall, alltoallv, scatter -----------------------------------------------------------------

def _alltoall_worker(ctx, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    lim = _limits(cc)
    ll, bulk = lim["ll"], lim["bulk"]
    # (name, bytes per block, output kind, out shift, in shift, LL disabled, in place)
    cases = []
    for b in (1, 15, 16, 17, 33, ll - 1, ll, ll + 1, lim["ll_pc"] - 1, lim["ll_pc"] + 1):
        if b * P <= 2 * bulk:
            cases.append(("ll", b, "plain", 0, _pick(SHIFTS, b), False, b in (17, ll)))
    for b in (1, 17, 33, 4096 + 4):
        cases.append(("no_ll", b, "plain", _pick(SHIFTS, b + 1), _pick(SHIFTS, b), True, b == 33))
    for j, b in enumerate((ll + 1, bulk // P - 16, bulk // P)):
        cases.append(("staged", b, "plain", _pick(SHIFTS, j + 2), _pick(SHIFTS, j + 3), False, j == 0))
    for j, (kind, off) in enumerate([("reg", o) for o in REG_OFFSETS] + [("odd", 0), ("sym", 0)]):
        for b in (33, ll + 17, bulk // P + 1):
            cases.append(("reg", b, kind, off, _pick(SHIFTS, j + b), False, False))
    for j, b in enumerate((bulk // P + 1, bulk * 5 // 2 // P + 3)):
        cases.append(("pipelined", b, "plain", _pick(SHIFTS, j + 1), _pick(SHIFTS, j + 4), False, False))
    if thorough:
        for so in SHIFTS:
            for si in SHIFTS:
                for b in (ll + 33, bulk // P + 33):
                    cases.append(("shifts", b, "plain", so, si, False, False))
                cases.append(("shifts_reg", bulk // P - 33, "reg", so, si, False, False))
    st = Stores(cc, 2 * GUARD + 16 + max(c[1] for c in cases) * P)
    ll_off = None
    for ci, (name, b, kind, so, si, no_ll, inplace) in enumerate(cases):
        if no_ll != ll_off:
            _set_env(cc, "CUDA_LL_DISABLE", 1 if no_ll else None)
            ll_off = no_ll
        case = ("a2a", P, ci)
        inputs = [_input(case, r, b * P) for r in range(P)]
        want = _alltoallv_layout(inputs, [[b] * P for _ in range(P)], me)
        out = st.region(kind, so, b * P, (case, me))
        if inplace:
            out.view.copy_(inputs[me])
            inp, ireg = out.view, None
        else:
            ireg = _plain(b * P, si, (case, "in", me))
            ireg.view.copy_(inputs[me])
            inp = ireg.view
        cc.alltoall(out.view, inp)
        _sync(cc)
        what = f"alltoall {name} block={b} out={kind}+{so} " + ("in place" if inplace else f"in+{si}")
        chk.region(what, out, want)
        if ireg is not None:
            chk.region(what + " (input)", ireg, inputs[me])
    _set_env(cc, "CUDA_LL_DISABLE", None)
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_alltoall_exact(size):
    try:
        _report(gb.spawn_threads(size, _alltoall_worker, False, cuda_device=0))
    finally:
        os.environ.pop("GLB_CUDA_LL_DISABLE", None)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_alltoall_exact_sweep(size):
    try:
        _report(gb.spawn_threads(size, _alltoall_worker, True, cuda_device=0))
    finally:
        os.environ.pop("GLB_CUDA_LL_DISABLE", None)


def _a2av_tables(P, bulk):
    """(name, element size, table of element counts [from q][to j])."""
    g = _gen(("a2av", P))
    out = []
    # zero blocks, the diagonal among them
    t = torch.randint(0, 300, (P, P), generator=g).tolist()
    for q in range(P):
        t[q][q] = 0
        t[q][(q + 1) % P] = 0 if q % 2 else t[q][(q + 1) % P]
    out.append(("zeros", 4, t))
    # offsets 4-byte but not 16-byte aligned: the 128-bit-store body from 4-byte-congruent sources
    out.append(("4B_offsets", 4, [[4 * ((q + j) % 5) + 1 + 2 * (q == j) for j in range(P)] for q in range(P)]))
    out.append(("2B", 2, [[int(x) for x in torch.randint(0, 70, (P,), generator=g)] for _ in range(P)]))
    # odd byte offsets
    out.append(("odd", 1, [[2 * ((3 * q + j) % 7) + 1 for j in range(P)] for q in range(P)]))
    out.append(("8B", 8, [[(q * 7 + j * 3) % 11 for j in range(P)] for q in range(P)]))
    # one block larger than the bulk region
    t = [[(q + 2 * j) % 5 * 33 + 1 for j in range(P)] for q in range(P)]
    t[P - 1][0] = (bulk + 1003) // 4
    out.append(("big_block", 4, t))
    return out


def _alltoallv_worker(ctx, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    bulk = _limits(cc)["bulk"]
    tables = _a2av_tables(P, bulk)
    outs = [("plain", s) for s in ((0, 4, 1) if not thorough else SHIFTS)] + \
        [("reg", o) for o in REG_OFFSETS] + [("odd", 0), ("sym", 0)]
    st = Stores(cc, 2 * GUARD + 16 + max(sum(t[q][j] for q in range(P)) * es for _, es, t in tables for j in range(P)))
    i = 0
    for name, es, table in tables:
        dt = VIEW[es]
        tb = [[c * es for c in row] for row in table]
        for kind, so in outs:
            i += 1
            si = _pick(SHIFTS, i)
            case = ("a2av", P, name, kind, so)
            inputs = [_input(case, r, sum(tb[r])) for r in range(P)]
            want = _alltoallv_layout(inputs, tb, me)
            out = st.region(kind, so, want.numel(), (case, me), es)
            ireg = _plain(sum(tb[me]), si, (case, "in", me), es=es)
            ireg.view.copy_(inputs[me])
            cc.alltoallv(out.view.view(dt), [table[q][me] for q in range(P)], ireg.view.view(dt), table[me])
            _sync(cc)
            what = f"alltoallv {name} out={kind}+{out.shift} in+{ireg.shift}"
            chk.region(what, out, want)
            chk.region(what + " (input)", ireg, inputs[me])
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_alltoallv_exact(size):
    _report(gb.spawn_threads(size, _alltoallv_worker, False, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [3, 8])
def test_alltoallv_exact_sweep(size):
    _report(gb.spawn_threads(size, _alltoallv_worker, True, cuda_device=0))


def _inplace_registered_worker(ctx):
    """In-place alltoall(v) into a registered output is rejected on every rank before launch,
    and the context keeps working."""
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    lim = _limits(cc)
    b = lim["ll_pc"] + 64  # above every LL limit, tuning table or not
    st = Stores(cc, 2 * GUARD + 16 + b * P)
    raised = []
    for kind in ("reg", "sym"):
        for v in (False, True):
            reg = st.region(kind, 0, b * P, ("inplace", kind, v, me))
            try:
                if v:
                    cc.alltoallv(reg.view, [b] * P, reg.view, [b] * P)
                else:
                    cc.alltoall(reg.view, reg.view)
                _sync(cc)
            except ValueError as e:
                raised.append("overlap" in str(e))
            else:
                raised.append(False)
            chk.region(f"rejected in-place {'alltoallv' if v else 'alltoall'} {kind} (untouched)", reg)
    if not all(raised):
        chk.bad.append(f"rank {me}: in-place registered alltoall(v) did not raise: {raised}")
    # still usable
    case = ("after", P)
    inputs = [_input(case, r, b * P) for r in range(P)]
    out = st.region("reg", 16, b * P, (case, me))
    src = _plain(b * P, 4, (case, "in", me))
    src.view.copy_(inputs[me])
    cc.alltoall(out.view, src.view)
    _sync(cc)
    chk.region("alltoall after the rejected calls", out, _alltoallv_layout(inputs, [[b] * P] * P, me))
    # LL-sized in place on a registered output stays allowed: the LL kernel reads each unit before
    # it writes it
    small = st.region("reg", 0, 16 * P, ("ll_inplace", me))
    inputs = [_input(("ll_inplace", P), r, 16 * P) for r in range(P)]
    small.view.copy_(inputs[me])
    cc.alltoall(small.view, small.view)
    _sync(cc)
    chk.region("in-place registered alltoall at LL size", small, _alltoallv_layout(inputs, [[16] * P] * P, me))
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_inplace_registered_alltoall_rejected(size):
    _report(gb.spawn_threads(size, _inplace_registered_worker, cuda_device=0))


def _scatter_worker(ctx, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    bulk = _limits(cc)["bulk"]
    sizes = [1, 15, 16, 17, 33, bulk // P, bulk - 1, bulk, bulk + 1, bulk * 5 // 2 // P]
    roots = list(range(P)) if thorough else sorted({0, P - 1})
    kinds = [("plain", s) for s in SHIFTS] + [("reg", o) for o in REG_OFFSETS] + [("odd", 0), ("sym", 0)]
    st = Stores(cc, 2 * GUARD + 16 + max(sizes))
    i = 0
    for n in sizes:
        for root in roots:
            for kind, so in (kinds if thorough else [_pick(kinds, i + k) for k in range(3)]):
                i += 1
                si = _pick(SHIFTS, i)
                case = ("scatter", P, n, root, kind, so)
                rin = _input(case, root, n * P)
                out = st.region(kind, so, n, (case, me))
                ireg = None
                if me == root:
                    ireg = _plain(n * P, si, (case, "in"))
                    ireg.view.copy_(rin)
                cc.scatter(out.view, ireg.view if ireg is not None else None, root=root)
                _sync(cc)
                what = f"scatter n={n} root={root} out={kind}+{so} in+{si}"
                chk.region(what, out, _scatter_layout(rin, n, me))
                if ireg is not None:
                    chk.region(what + " (root input)", ireg, rin)
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_scatter_exact(size):
    _report(gb.spawn_threads(size, _scatter_worker, False, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [3, 8])
def test_scatter_exact_sweep(size):
    _report(gb.spawn_threads(size, _scatter_worker, True, cuda_device=0))


# ---- point to point ---------------------------------------------------------------------------------

SMALL_BOX = {"GLB_CUDA_P2P_SLOT_KB": "16", "GLB_CUDA_P2P_SLOTS": "2", "GLB_CUDA_P2P_LANES": "4"}


def _p2p_sizes(stripe, ring):
    return [1, 15, stripe - 1, stripe, stripe + 1, 3 * ring + 5, 0, 33]


def _p2p_worker(ctx, stripe, ring, thorough):
    """Back-to-back sendrecv calls on one stream (no sync in between) around a ring: each rank
    sends sizes[(k + me) % len] bytes, so the ring's counters carry over between calls of
    different sizes and one direction of some calls is empty."""
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    right, left = (me + 1) % P, (me - 1) % P
    sizes = _p2p_sizes(stripe, ring)
    shifts = (0, 4, 1)
    for rnd, (ss, rs) in enumerate([(a, b) for a in shifts for b in shifts] if thorough else
                                   [(0, 0), (4, 4), (1, 1), (0, 4), (4, 1), (1, 0)]):
        calls = []
        for k in range(len(sizes)):
            ns, nr = sizes[(k + me) % len(sizes)], sizes[(k + left) % len(sizes)]
            case = ("p2p", P, rnd, k)
            data = _input(case, me, ns)
            src = _plain(ns, ss, (case, "s", me))
            src.view.copy_(data)
            dst = _plain(nr, rs, (case, "r", me))
            calls.append((k, ns, nr, src, data, dst, _input(case, left, nr)))
        _sync(cc)
        cc.pc.host_barrier()  # every allocation done before kernels that wait for a peer
        for k, ns, nr, src, _, dst, _ in calls:
            cc.sendrecv(src.view, right, dst.view, left)
        _sync(cc)
        for k, ns, nr, src, data, dst, want in calls:
            what = f"sendrecv call {k} send {ns}B+{ss} recv {nr}B+{rs}"
            chk.region(what, dst, want)
            chk.region(what + " (input)", src, data)
        cc.pc.host_barrier()
    if P == 2:
        # send and recv as separate kernels on separate streams, both directions at once
        s1, s2 = gcu.new_stream(0), gcu.new_stream(0)
        n = 3 * ring + 17
        case = ("p2p_streams", P)
        src = _plain(n, 4, (case, "s", me))
        src.view.copy_(_input(case, me, n))
        dst = _plain(n, 1, (case, "r", me))
        _sync(cc)
        cc.pc.host_barrier()
        cc.send(src.view, 1 - me, stream=s1)
        cc.recv(dst.view, 1 - me, stream=s2)
        s1.synchronize()
        s2.synchronize()
        chk.region("send / recv on two streams", dst, _input(case, 1 - me, n))
        chk.region("send / recv on two streams (input)", src, _input(case, me, n))
    cc.check_health()
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4])
def test_sendrecv_small_mailbox_exact(size, monkeypatch):
    """A 2 x 16 KiB ring cut into 4 stripes of 4 KiB: a few hundred KB wrap it many times."""
    for k, v in SMALL_BOX.items():
        monkeypatch.setenv(k, v)
    _report(gb.spawn_threads(size, _p2p_worker, 4096, 2 * 16 * 1024, False, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4])
def test_sendrecv_small_mailbox_exact_sweep(size, monkeypatch):
    for k, v in SMALL_BOX.items():
        monkeypatch.setenv(k, v)
    _report(gb.spawn_threads(size, _p2p_worker, 4096, 2 * 16 * 1024, True, cuda_device=0))


def _p2p_default_worker(ctx):
    """One transfer larger than the default ring (4 slots of 3 MiB)."""
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    n = (13 << 20) + 3
    case = ("p2p_big", P)
    src = _plain(n, 1, (case, "s", me))
    src.view.copy_(torch.randint(0, 256, (n,), generator=_gen((case, me)), dtype=U8))
    dst = _plain(n, 4, (case, "r", me))
    _sync(cc)
    cc.pc.host_barrier()
    cc.sendrecv(src.view, (me + 1) % P, dst.view, (me - 1) % P)
    _sync(cc)
    chk.region("sendrecv larger than the default ring", dst,
               torch.randint(0, 256, (n,), generator=_gen((case, (me - 1) % P)), dtype=U8))
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3])
def test_sendrecv_default_mailbox_exact(size):
    for k in SMALL_BOX:
        assert k not in os.environ
    _report(gb.spawn_threads(size, _p2p_default_worker, cuda_device=0))


def _exchange_worker(ctx, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    right, left = (me + 1) % P, (me - 1) % P
    sizes = [1, 15, 65535, 65536, 65536 + 17, (2 << 20) + 3]
    sym = cc.empty(2 * GUARD + 16 + max(sizes), U8)
    i = 0
    for tma in (True, False):
        _set_tma(cc, tma)
        for off in (0, 16, 4):
            for k in range(len(sizes) if thorough else 3):
                i += 1
                # a different size per rank: I send n[me] and receive n[left]
                n = [sizes[(k + 2 * r + i) % len(sizes)] for r in range(P)]
                case = ("xchg", P, tma, off, k)
                data = _input(case, me, n[me])
                src = _plain(n[me], off, (case, "s", me))
                src.view.copy_(data)
                dst = Region(sym, 0, off, n[left], (case, "r", me))
                _sync(cc)
                cc.pc.host_barrier()
                cc.exchange(src.view, right, dst.view, left)
                _sync(cc)
                cc.pc.host_barrier()
                what = f"exchange tma={tma} recv {n[left]}B at +{off} send {n[me]}B"
                chk.region(what, dst, _input(case, left, n[left]))
                chk.region(what + " (input)", src, data)
    _set_tma(cc, False)
    cc.pc.host_barrier()
    return chk.result()


def _put_get_worker(ctx, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    right, left = (me + 1) % P, (me - 1) % P
    sizes = [1, 17, 65535, 65536, 65536 + 17, 300_003]
    win = cc.empty(2 * GUARD + 16 + max(sizes), U8)
    i = 0
    for tma in (True, False):
        _set_tma(cc, tma)
        for off in (0, 4, 1):
            for n in (sizes if thorough else sizes[1:5]):
                i += 1
                ls = _pick((0, 4, 1), i)
                case = ("put", P, tma, off, n)
                # put: I write n bytes at window byte GUARD + off of my right neighbour's window
                w = Region(win, 0, 0, max(sizes) + 16, (case, "w", me))
                data = _input(case, me, n)
                src = _plain(n, ls, (case, "s", me))
                src.view.copy_(data)
                _sync(cc)
                cc.pc.host_barrier()
                cc.put(src.view, win, right, remote_offset=GUARD + off)
                _sync(cc)
                cc.pc.host_barrier()
                payload = w.init[w.lo:w.lo + w.n].clone()
                payload[off:off + n] = _input(case, left, n)
                chk.region(f"put tma={tma} n={n} at +{off} local+{ls} (target window)", w, payload)
                # get: I read n bytes at GUARD + off of my left neighbour's (re-filled) window
                case = ("get", P, tma, off, n)
                w = Region(win, 0, 0, max(sizes) + 16, (case, "w", me))
                dst = _plain(n, ls, (case, "d", me))
                _sync(cc)
                cc.pc.host_barrier()
                cc.get(dst.view, win, left, remote_offset=GUARD + off)
                _sync(cc)
                cc.pc.host_barrier()
                theirs = _seeded(("guard", (case, "w", left)), w.init.numel())
                chk.region(f"get tma={tma} n={n} at +{off} local+{ls}", dst, theirs[GUARD + off:GUARD + off + n])
                chk.region(f"get tma={tma} n={n} at +{off} (source window)", w)
    _set_tma(cc, False)
    cc.pc.host_barrier()
    return chk.result()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4])
def test_exchange_exact(size):
    try:
        _report(gb.spawn_threads(size, _exchange_worker, False, cuda_device=0))
    finally:
        gb._C.cuda.set_tuning({"tma_copies": False})


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 4])
def test_put_get_exact(size):
    try:
        _report(gb.spawn_threads(size, _put_get_worker, False, cuda_device=0))
    finally:
        gb._C.cuda.set_tuning({"tma_copies": False})


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 4])
def test_exchange_put_get_exact_sweep(size):
    try:
        _report(gb.spawn_threads(size, _exchange_worker, True, cuda_device=0))
        _report(gb.spawn_threads(size, _put_get_worker, True, cuda_device=0))
    finally:
        gb._C.cuda.set_tuning({"tma_copies": False})


# ---- one rank: the calls that reduce to cudaMemcpyAsync ---------------------------------------------

def _single_worker(ctx):
    cc = _cc(ctx)
    chk = Checker(0)
    st = Stores(cc, 2 * GUARD + 16 + 100_003)
    for n in (1, 17, 100_003):
        for kind, so in (("plain", 1), ("plain", 4), ("reg", 0), ("odd", 0), ("sym", 4)):
            case = ("single", n, kind, so)
            data = _input(case, 0, n)
            src = _plain(n, 2, (case, "in"))
            src.view.copy_(data)
            calls = [("allgather", lambda o, i: cc.allgather(o, i)),
                     ("allgatherv", lambda o, i: cc.allgatherv(o, i, [n])),
                     ("gather", lambda o, i: cc.gather(o, i)),
                     ("alltoall", lambda o, i: cc.alltoall(o, i)),
                     ("alltoallv", lambda o, i: cc.alltoallv(o, [n], i, [n])),
                     ("scatter", lambda o, i: cc.scatter(o, i)),
                     ("broadcast", None)]
            for name, fn in calls:
                out = st.region(kind, so, n, (case, name))
                if fn is None:
                    out.view.copy_(data)
                    cc.broadcast(out.view)
                else:
                    fn(out.view, src.view)
                _sync(cc)
                chk.region(f"P=1 {name} n={n} out={kind}+{so}", out, data)
                chk.region(f"P=1 {name} n={n} (input)", src, data)
    return chk.result()


@pytest.mark.gpu
def test_single_rank_copies_exact():
    _report(gb.spawn_threads(1, _single_worker, cuda_device=0))
