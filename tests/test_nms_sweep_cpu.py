"""A model of the NMS sweep's schedule, written from nms_enqueue and nms_sweep_kernel (csrc/kernels_nms.cu), checked
without a GPU.

The sweep keeps the `removed` bitmap of a set in shared memory and walks its mask slab in steps: a step is a 64-row
block b and a chunk of `chunk` mask words starting at column c0, and the chunks of block b cover the columns [b, nw).
The words of the next step are staged into the other half of a double buffer while the current one is used.  Large
sets (more than 14,400 boxes on an H100) take several chunks per block.  These tests pin the shared-memory plan, the
walk, the staging and the keep / drop decisions of that walk on random masks; tests/test_gpu_nms_edges.py runs the
kernel itself at the same chunk counts."""
import numpy as np
import pytest

H100_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
MAX_WORDS = 25600            # the largest set the 200 KB bitmap check accepts: ceil(n / 64) words
STATIC_SMEM = 16             # nms_sweep_kernel's static shared memory (s_keep), as ptxas reports it for sm_90a
ALL = (1 << 64) - 1


def plan(optin, max_words):
    """nms_enqueue: (chunk, dynamic shared memory in bytes) of the sweep for the largest set's word count."""
    avail_words = (optin - 64) // 8 - max_words
    assert avail_words > 0
    chunk = max(1, min(max_words, avail_words // 128))
    return chunk, 8 * (2 * 64 * chunk + max_words)


def walk(nv, chunk):
    """The steps of nms_sweep_kernel for a set with nv valid rows, as the kernel's loop makes them.  Returns the
    prologue's stage and, per step, (b, c0, cw, buffer read, stage issued or None, wait_prior argument).  A stage is
    (buffer, first row, rows, first word, words)."""
    nw = (nv + 63) // 64
    prologue = (0, 0, min(64, nv), 0, min(chunk, nw)) if nw > 0 else None
    steps = []
    b = c0 = step = 0
    while b < nw:
        nb, nc = b, c0 + chunk
        if nc >= nw:
            nb = b + 1
            nc = nb
        stage = None
        if nb < nw:
            stage = ((step + 1) & 1, nb * 64, min(64, nv - nb * 64), nc, min(chunk, nw - nc))
        steps.append((b, c0, min(chunk, nw - c0), step & 1, stage, 1 if stage else 0))
        b, c0 = nb, nc
        step += 1
    return prologue, steps


def check_walk(nv, chunk):
    nw = (nv + 63) // 64
    prologue, steps = walk(nv, chunk)
    seen = np.zeros((nw, nw), np.int32)
    first = {}
    committed = 1 if prologue else 0    # cp.async commit groups issued so far: the prologue's, then one per stage
    for s, (b, c0, cw, buf, stage, wait) in enumerate(steps):
        assert 1 <= cw <= chunk and c0 >= b
        first.setdefault(b, c0)
        seen[b, c0:c0 + cw] += 1
        # what this step reads is what was staged for it: the prologue for step 0, else the stage of step - 1
        want = (buf, b * 64, min(64, nv - b * 64), c0, cw)
        assert (prologue if s == 0 else steps[s - 1][4]) == want, (nv, chunk, s)
        if stage is not None:
            assert stage[0] != buf      # never stages into the buffer it reads
            assert 1 <= stage[2] <= 64 and 1 <= stage[4] <= chunk
            committed += 1
        # wait_prior(wait) leaves the newest `wait` groups in flight: the group of this step (number s) has landed
        assert committed - wait > s
    want = np.triu(np.ones((nw, nw), np.int32))
    assert np.array_equal(seen, want), (nv, chunk)       # every (b, c >= b, c < nw) exactly once
    assert all(first[b] == b for b in range(nw))         # each block starts with its diagonal word
    return len(steps)


def test_shared_memory_fits_for_every_accepted_set_size():
    w = np.arange(1, MAX_WORDS + 1)
    avail = (H100_OPTIN - 64) // 8 - w
    assert avail.min() > 0
    chunk = np.maximum(1, np.minimum(w, avail // 128))
    smem = 8 * (2 * 64 * chunk + w)
    assert np.all(smem + 64 <= H100_OPTIN)                 # nms_enqueue leaves 64 bytes for the static part
    assert STATIC_SMEM <= 64
    assert np.all(chunk >= 1) and np.all(chunk <= w)
    # one chunk per block up to 225 words (14,400 boxes); several from 226 on
    assert np.array_equal(chunk == w, w <= 225)
    for mw in (1, 225, 226, 394, 525, 938, MAX_WORDS):
        assert plan(H100_OPTIN, mw) == (chunk[mw - 1], smem[mw - 1])


def chunk_groups():
    """(chunk, smallest max_words, largest max_words) for every chunk the H100 plan produces."""
    groups = {}
    for mw in range(1, MAX_WORDS + 1):
        c = plan(H100_OPTIN, mw)[0]
        lo, hi = groups.get(c, (mw, mw))
        groups[c] = (min(lo, mw), max(hi, mw))
    return sorted((c, lo, hi) for c, (lo, hi) in groups.items())


def test_walk_covers_every_word_once_for_every_max_words():
    """The walk depends on the valid words nw and the chunk alone, and chunk is set by max_words >= nw.  For every chunk
    the H100 plan produces, the walk is checked at nw = 4 chunk + 1 (capped at the largest max_words with that chunk),
    whose blocks b have every remaining length nw - b from 1 to 4 chunk + 1: every length mod chunk, and one to five
    chunks per block; and at the small and one-past-a-chunk word counts."""
    groups = chunk_groups()
    assert [c for c, _, _ in groups] == list(range(1, 226))
    assert min(c for c, _, hi in groups if hi > 225) == 26     # the narrowest chunk, at the largest sets
    total = 0
    for c, lo, hi in groups:
        for nw in sorted({w for w in (1, 2, c, c + 1, 2 * c + 1, 4 * c + 1, hi) if w <= min(hi, 4 * c + 1)}):
            for nv in {64 * nw, 64 * nw - 63}:     # a full last block, a last block of one row
                total += check_walk(nv, c)
    assert total > 0


@pytest.mark.parametrize("n,chunks", [(10000, 1), (14400, 1), (14401, 2), (25200, 2), (33600, 3), (60000, 5)])
def test_chunks_of_block_0_at_the_detector_sizes(n, chunks):
    w = (n + 63) // 64
    chunk = plan(H100_OPTIN, w)[0]
    _, steps = walk(n, chunk)
    got = [(c0, cw) for b, c0, cw, *_ in steps if b == 0]
    assert len(got) == chunks
    if n == 14401:
        assert got == [(0, 225), (225, 1)]   # the second chunk is one word wide
    if n <= 14401:
        check_walk(n, chunk)


# --------------------------------------------------------------------------- the sweep on random masks
def greedy(sup):
    """Plain greedy NMS on a suppression matrix in rank order (sup[i, j]: i removes j, read for j > i only)."""
    nv = len(sup)
    removed = np.zeros(nv, bool)
    kept = []
    for i in range(nv):
        if removed[i]:
            continue
        kept.append(i)
        removed[i + 1:] |= sup[i, i + 1:]
    return kept


def slab_of(sup, n, rng):
    """The mask slab of a set of n boxes with nv = len(sup) valid rows, as nms_mask_kernel leaves it: word (i, jb) for
    i < nv and jb >= i / 64 holds the bits of columns jb * 64 + t in (i, nv); every other word is never written, so it
    holds whatever the pool's memory held (random here)."""
    nv = len(sup)
    words = (n + 63) // 64
    slab = rng.integers(0, 1 << 63, (n, words), dtype=np.int64).astype(np.uint64) * np.uint64(2)
    for i in range(nv):
        for jb in range(i // 64, (nv + 63) // 64):
            bits = 0
            for t in range(64):
                j = jb * 64 + t
                if i < j < nv and sup[i, j]:
                    bits |= 1 << t
            slab[i, jb] = bits
    return slab


def sweep(slab, nv, chunk, rng):
    """nms_sweep_kernel on one set, step for step: staging into the double buffer (which starts as garbage), the
    diagonal walk of the alive rows, and the OR of the kept rows into `removed`.  Returns the kept rows."""
    words = slab.shape[1]
    nw = (nv + 63) // 64
    sm = [[int(x) for x in row] for row in rng.integers(0, 1 << 62, (2 * 64, chunk))]   # [2][64][chunk]
    removed = [0] * nw
    kept = []

    def stage(buf, r0, rows, c0, cw):
        for r in range(rows):
            for c in range(cw):
                sm[buf * 64 + r][c] = int(slab[r0 + r, c0 + c])

    prologue, steps = walk(nv, chunk)
    if prologue:
        stage(*prologue)
    keep = 0
    for b, c0, cw, buf, st, _ in steps:
        if st:
            stage(*st)      # the other buffer: the model has no overlap, so it may be filled at once
        cur = sm[buf * 64: buf * 64 + 64]
        if c0 == b:
            lim = min(64, nv - b * 64)
            alive = (ALL if lim == 64 else (1 << lim) - 1) & ~removed[b]
            kp = 0
            while alive:
                r = (alive & -alive).bit_length() - 1
                kp |= 1 << r
                alive &= alive - 1
                alive &= ~cur[r][0]
            keep = kp
            kept += [b * 64 + r for r in range(64) if (keep >> r) & 1]
        if keep:
            for c in range(cw):
                if c0 + c <= b:
                    continue
                acc = 0
                m = keep
                while m:
                    acc |= cur[(m & -m).bit_length() - 1][c]
                    m &= m - 1
                removed[c0 + c] |= acc
    return kept


def chains(nv, rng, length=3, stride=97):
    """Suppression matrix made of chains i -> i + stride -> i + 2 stride: each link's head removes its tail, so greedy
    keeps every other box of a chain.  A stride past 64 * chunk makes the links cross chunks."""
    sup = np.zeros((nv, nv), bool)
    for i in rng.permutation(nv)[: nv // (2 * length)]:
        for k in range(length - 1):
            a, b = i + k * stride, i + (k + 1) * stride
            if b < nv:
                sup[a, b] = True
    return sup


@pytest.mark.parametrize("nv,extra", [(1, 0), (63, 5), (64, 0), (65, 70), (130, 0), (700, 1), (1000, 300)])
@pytest.mark.parametrize("chunk", [1, 2, 3, 5, None])
@pytest.mark.parametrize("kind", ["sparse", "dense", "chains"])
def test_sweep_equals_greedy(nv, extra, chunk, kind):
    rng = np.random.default_rng(nv * 31 + (chunk or 0) * 7 + len(kind))
    n = nv + extra          # the set's size: its slab pitch is ceil(n / 64) words, however many rows pass the filters
    nw = (nv + 63) // 64
    c = (n + 63) // 64 if chunk is None else chunk
    if kind == "sparse":
        sup = rng.random((nv, nv)) < 3.0 / max(nv, 1)
    elif kind == "dense":
        sup = rng.random((nv, nv)) < 0.3
    else:
        sup = chains(nv, rng, stride=64 * c + 7 if nv > 64 * c + 7 else 33)
    slab = slab_of(sup, n, rng)
    got = sweep(slab, nv, c, rng)
    assert got == greedy(sup), (nv, n, c, nw)
