"""The host side of the RD-loop batch API (tb_rdo_batch_*, include/thor_b200.h) as a server drives it: slots reused for other frames and other
geometries, launches over a prefix of the slots, a second round enqueued before the first has run, tb_rdo_encode_frames growing and shrinking its
internal batch, and argument errors on a live batch.

Every launch's decisions are checked against the reference's (RJ.HostFrame.check: reconstruction, block state, RD cost per super block), and where it
is cheap the leaf lists and coefficients against oracle/librdo_hostcheck.so (RJ.leaf_differences).  The committed golden jobs (tests/golden, all
128x136: 8-bit qp 32, 10-bit hard content at qp 4, 12-bit qp 51) need no compiled reference; the geometry cases capture three cases of
tests/test_rdo_matrix.py and are skipped like the matrix where oracle/_ref is absent.  Host buffers are pinned (tb_malloc_host), so the copies are
asynchronous and the host runs ahead of the stream."""
import contextlib
import ctypes as C
import multiprocessing
import os
from concurrent.futures import ProcessPoolExecutor, ThreadPoolExecutor

import numpy as np
import pytest

from test_rdo_jobs import golden_jobs
from test_rdo_matrix import BY_NAME, CONTENT, needs_capture

pytestmark = pytest.mark.gpu

TB_ERR_ARG = -2
NSTATS = 68
# tb_rdo_batch_stats: the work the RD loop executed ([11..22], [22] = super blocks) and the overlapped B-frame decisions by where their joint search
# ran ([66..67]).  Both depend only on the decisions, not on which warp or CTA drew which candidate or super block.  The other entries count cycles.
WORK = list(range(11, 23)) + [66, 67]
ST_SB = 22
TRACE = np.dtype([(k, np.int32) for k in ("frame", "row", "col", "cta")] + [("t_start", np.uint64), ("t_end", np.uint64)])


@pytest.fixture(scope="module")
def lib():
    import thor_b200 as tb
    L = tb.lib
    L.tb_rdo_batch_create.restype = C.c_void_p
    L.tb_rdo_batch_create.argtypes = [C.c_int, C.c_int]
    L.tb_rdo_batch_upload.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.tb_rdo_batch_run.argtypes = [C.c_void_p, C.c_int]
    L.tb_rdo_batch_download.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.tb_rdo_batch_sync.argtypes = [C.c_void_p]
    L.tb_rdo_batch_grid.argtypes = [C.c_void_p]
    L.tb_rdo_batch_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.tb_rdo_batch_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.tb_rdo_batch_destroy.argtypes = [C.c_void_p]
    L.tb_rdo_last_error.restype = C.c_char_p
    tb.init(0)
    return L


@pytest.fixture
def pinned(lib):
    """alloc(nbytes) -> address of pinned host memory, freed after the test once the library's stream is idle"""
    ptrs = []

    def alloc(nbytes):
        p = lib.tb_malloc_host(max(nbytes, 16))
        assert p, "tb_malloc_host"
        ptrs.append(p)
        return p
    yield alloc
    lib.tb_sync()
    for p in ptrs:
        lib.tb_free_host(p)


@pytest.fixture(scope="module")
def golden(tmp_path_factory):
    """golden(case) -> the committed jobs of one golden case"""
    from thor_b200 import rdo_jobs as RJ
    done = {}

    def get(case):
        if case not in done:
            d = str(tmp_path_factory.mktemp(case))
            golden_jobs(d, case)
            done[case] = RJ.load_jobs(d)
        return done[case]
    return get


@pytest.fixture(scope="module")
def host_leaves(golden):
    """host_leaves(job) -> oracle/librdo_hostcheck.so's decisions on a golden job (an RJ.HostFrame), computed once per golden case"""
    from _libs import host_decisions
    keep, by_job = [], {}

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data

    def get(job):
        if id(job) not in by_job:
            for case in ("hdb_128x136", "hdb_hard_q4_10bit", "hdb_q51_12bit"):
                jobs = golden(case)
                if any(j is job for j in jobs):
                    for j, hf in zip(jobs, host_decisions(jobs, alloc)):
                        assert hf.check() == {"rec": True, "blk": True, "sb_cost": True}, (case, j.frame_num, "host decisions differ from the reference's")
                        by_job[id(j)] = hf
        return by_job[id(job)]
    return get


@pytest.fixture(scope="module")
def captured(tmp_path_factory):
    """the jobs of three cases of tests/test_rdo_matrix.py, captured with the reference encoder: {name: jobs}"""
    from test_rdo_jobs import capture
    from thor_b200 import rdo_jobs as RJ

    def one(name):
        _, flags, w, h, n, qp, bd, content = BY_NAME[name]
        return name, RJ.load_jobs(capture(str(tmp_path_factory.mktemp(name)), flags, w, h, n, bd, qp, CONTENT[content]))
    tmp_path_factory.getbasetemp()
    with ThreadPoolExecutor(3) as ex:
        return dict(ex.map(one, ["hdb_pan_neg", "hdb_sb64_rect", "ldb_bipred4"]))


class Batch:
    """one tb_rdo_batch_t; every call must return TB_OK"""

    def __init__(self, L, nslots, sample_bytes):
        self.L = L
        self.b = L.tb_rdo_batch_create(nslots, sample_bytes)
        assert self.b, L.tb_rdo_last_error()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.L.tb_rdo_batch_destroy(self.b)

    def ok(self, rc, what):
        assert rc == 0, (what, rc, self.L.tb_rdo_last_error())

    def upload(self, slot, hf):
        self.ok(self.L.tb_rdo_batch_upload(self.b, slot, C.byref(hf.desc)), "upload %d" % slot)

    def run(self, n):
        self.ok(self.L.tb_rdo_batch_run(self.b, n), "run %d" % n)

    def download(self, slot, hf):
        self.ok(self.L.tb_rdo_batch_download(self.b, slot, C.byref(hf.desc)), "download %d" % slot)

    def sync(self):
        self.ok(self.L.tb_rdo_batch_sync(self.b), "sync")

    def round(self, hosts):
        """hosts[s] into slot s, one launch over them all, their decisions back, one sync"""
        for s, hf in enumerate(hosts):
            self.upload(s, hf)
        self.run(len(hosts))
        for s, hf in enumerate(hosts):
            self.download(s, hf)
        self.sync()

    def stats(self):
        out = (C.c_uint64 * NSTATS)()
        assert self.L.tb_rdo_batch_stats(self.b, out, NSTATS) == NSTATS
        return np.array(out, np.uint64)

    def trace(self):
        n = self.L.tb_rdo_batch_trace(self.b, None, 0)
        rec = np.zeros(n, TRACE)
        assert n == 0 or self.L.tb_rdo_batch_trace(self.b, rec.ctypes.data, n) == n
        return rec

    def grid(self):
        return int(self.L.tb_rdo_batch_grid(self.b))


def geometry(job):
    """(super-block columns, rows) of a job"""
    sb = 1 << job.hdr.log2_sb_size
    return -(-job.hdr.width // sb), -(-job.hdr.height // sb)


def assert_reference(hosts, what):
    bad = [(k, hf.job.frame_num, r) for k, hf in enumerate(hosts) for r in [hf.check()] if not all(r.values())]
    assert not bad, ("%s: %d of %d frames differ from the reference's decisions" % (what, len(bad), len(hosts)), bad[:6])


def assert_host_leaves(hosts, host_leaves, what):
    for k, hf in enumerate(hosts):
        d = hf.leaf_differences(host_leaves(hf.job))
        assert not d, (what, "slot", k, "frame", hf.job.frame_num, d)


def assert_last_launch(batch, hosts, what):
    """tb_rdo_batch_trace holds every super block of the launch over `hosts` (slot s = hosts[s]) exactly once and no other, and the work counters
    of tb_rdo_batch_stats count that launch's super blocks"""
    tr = batch.trace()
    want = {(s, r, c) for s, hf in enumerate(hosts) for r in range(geometry(hf.job)[1]) for c in range(geometry(hf.job)[0])}
    got = [(int(f), int(r), int(c)) for f, r, c in zip(tr["frame"], tr["row"], tr["col"])]
    assert len(got) == len(want) and set(got) == want, (what, "trace", len(got), len(set(got)), len(want), sorted(set(got) ^ want)[:8])
    assert ((tr["cta"] >= 0) & (tr["cta"] < batch.grid())).all(), what
    assert int(batch.stats()[ST_SB]) == len(want), (what, "super blocks counted", int(batch.stats()[ST_SB]), len(want))


def differing(a, b):
    """(share of 4x4 block-state entries, share of reconstructed samples) in which the reference's decisions on two jobs of one geometry differ"""
    blk = (a.blk.view(np.uint8).reshape(a.blk.size, -1) != b.blk.view(np.uint8).reshape(b.blk.size, -1)).any(axis=1).mean()
    rec = np.concatenate([(a.rec[p] != b.rec[p]).ravel() for p in range(3)]).mean()
    return float(blk), float(rec)


def frames(jobs, alloc):
    from thor_b200 import rdo_jobs as RJ
    return [RJ.HostFrame(j, alloc) for j in jobs]


# -------------------------------------------------------------------------------------------------------------------------------------------------
# slots reused for other frames of the same geometry
# -------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sample_bytes", [1, 2], ids=["8bit", "16bit"])
def test_reused_slot_returns_the_new_frames_decisions(lib, golden, host_leaves, pinned, sample_bytes):
    """A slot keeps its device buffers for a frame of the same geometry: what the kernel failed to write would still hold the previous frame's
    decisions.  16 bits: the 10-bit qp 4 hard frames in slots 0..4, then the 12-bit qp 51 frames in slots 0..2, and the reverse in a new batch.
    8 bits: the nine frames in slots 0..8, then frame (s + 1) % 9 in slot s.  The two frames of a reused slot differ in most block-state entries and
    reconstructed samples, so a part of the outputs left unwritten shows up."""
    if sample_bytes == 2:
        hard, q51 = golden("hdb_hard_q4_10bit"), golden("hdb_q51_12bit")
        orders = [[hard, q51], [q51, hard]]
    else:
        g = golden("hdb_128x136")
        orders = [[g, [g[(s + 1) % 9] for s in range(9)]]]
    for order in orders:
        with Batch(lib, max(len(r) for r in order), sample_bytes) as batch:
            in_slot = {}
            for k, jobs in enumerate(order):
                what = "round %d (%s)" % (k, ", ".join("%d-bit frame %d" % (j.hdr.bitdepth, j.frame_num) for j in jobs))
                for s, j in enumerate(jobs):
                    if s in in_slot:
                        blk, rec = differing(in_slot[s], j)
                        assert blk > 0.5 and rec > 0.5, ("slot %d: the frames before and after share most decisions" % s, blk, rec)
                    in_slot[s] = j
                hosts = frames(jobs, pinned)
                batch.round(hosts)
                assert_reference(hosts, what)
                assert_host_leaves(hosts, host_leaves, what)
                assert_last_launch(batch, hosts, what)


# -------------------------------------------------------------------------------------------------------------------------------------------------
# launches without a new upload, over a prefix of the slots, and the work counters
# -------------------------------------------------------------------------------------------------------------------------------------------------
def test_rerun_without_upload_repeats_decisions_and_work(lib, golden, pinned):
    """the same batch launched twice: the second launch's decisions, downloaded into zeroed host buffers, are those of the first, and so is its work"""
    from thor_b200 import rdo_jobs as RJ
    g = golden("hdb_128x136")
    hosts = frames(g, pinned)
    with Batch(lib, len(g), 1) as batch:
        batch.round(hosts)
        assert_reference(hosts, "first launch")
        first = [(hf.rec[0].copy(), hf.rec[1].copy(), hf.rec[2].copy(), hf.blk.copy(), hf.leaf_count.copy(), hf.leaves.copy(), hf.coeffs.copy()) for hf in hosts]
        s1 = batch.stats()
        for hf in hosts:
            hf.clear_outputs()
            hf.leaves.view(np.uint8)[...] = 0
            hf.coeffs[...] = 0
        batch.run(len(hosts))
        for s, hf in enumerate(hosts):
            batch.download(s, hf)
        batch.sync()
        s2 = batch.stats()
        assert_last_launch(batch, hosts, "second launch")
    assert_reference(hosts, "second launch")
    for hf, f in zip(hosts, first):
        for name, a, b in zip(("rec y", "rec u", "rec v", "blk", "leaf_count"), f, (hf.rec[0], hf.rec[1], hf.rec[2], hf.blk, hf.leaf_count)):
            assert np.array_equal(a, b), ("frame", hf.job.frame_num, name)
        # what the bit writer reads; the other leaf fields hold whichever candidate the deciding warp saw last (RJ.LEAF_FIELD_MODES)
        d = RJ.leaf_differences(hf.leaves, hf.leaf_count, hf.coeffs, f[5], f[4], f[6])
        assert not d, ("frame", hf.job.frame_num, d)
    assert (s1[11:23] > 0).all(), s1[11:23]
    assert np.array_equal(s1[WORK], s2[WORK]), dict(zip(WORK, zip(s1[WORK].tolist(), s2[WORK].tolist())))
    assert int(s2[ST_SB]) == sum(j.nsb for j in g)


def test_work_of_a_two_frame_launch_is_the_sum_of_its_frames(lib, golden, pinned):
    """the work counters of one launch over a B frame and the P frame equal the sums of the two one-frame launches"""
    g = golden("hdb_128x136")
    a, b = g[1], g[8]
    assert (a.hdr.frame_type, b.hdr.frame_type) == (2, 1)
    with Batch(lib, 2, 1) as batch:
        both = frames([a, b], pinned)
        batch.round(both)
        assert_reference(both, "two frames")
        s_ab = batch.stats()
        only_a = frames([a], pinned)
        batch.run(1)
        batch.download(0, only_a[0])
        batch.sync()
        assert_reference(only_a, "first frame alone")
        s_a = batch.stats()
        only_b = frames([b], pinned)
        batch.round(only_b)
        assert_reference(only_b, "second frame alone")
        s_b = batch.stats()
    assert s_ab[66] + s_ab[67] > 0, "the B frame makes overlapped decisions with a joint bi-prediction search"
    assert np.array_equal(s_ab[WORK], s_a[WORK] + s_b[WORK]), dict(zip(WORK, zip(s_ab[WORK].tolist(), s_a[WORK].tolist(), s_b[WORK].tolist())))


def test_prefix_run_leaves_the_other_slots_as_their_last_launch_left_them(lib, golden, pinned):
    """tb_rdo_batch_run(b, k) after a launch over all nine slots, with new frames in slots 0..k-1: those return the new frames' decisions, slots k..8
    still return the decisions of the first launch"""
    g = golden("hdb_128x136")
    k = 4
    with Batch(lib, len(g), 1) as batch:
        first = frames(g, pinned)
        batch.round(first)
        assert_reference(first, "full launch")
        new = frames([g[(s + 1) % 9] for s in range(k)], pinned)
        for s, hf in enumerate(new):
            batch.upload(s, hf)
        batch.run(k)
        again = new + frames(g[k:], pinned)
        for s, hf in enumerate(again):
            batch.download(s, hf)
        batch.sync()
        assert_last_launch(batch, new, "prefix launch")
    assert_reference(again, "prefix launch: slots below %d new, the others from the full launch" % k)


# -------------------------------------------------------------------------------------------------------------------------------------------------
# geometry changes in one slot
# -------------------------------------------------------------------------------------------------------------------------------------------------
@needs_capture
def test_geometry_changes_in_one_slot(lib, golden, captured, pinned):
    """one slot takes, in turn: a 128x136 B frame, a 384x256 one, 128x136 again, a frame with two references and one with four (the same geometry),
    a frame of 64-sample super blocks, and the I frame of the first clip after one of its B frames.  The row table, the grid and the trace of the
    batch grow along the way; after every launch the trace holds that launch's super blocks and no other"""
    g = golden("hdb_128x136")
    pan = [j for j in captured["hdb_pan_neg"] if j.hdr.frame_type == 2][0]
    ldb = captured["ldb_bipred4"]
    ldb2, ldb4 = [j for j in ldb if j.hdr.num_ref == 2][0], [j for j in ldb if j.hdr.num_ref >= 4][0]
    sb64 = [j for j in captured["hdb_sb64_rect"] if j.hdr.frame_type == 2][0]
    steps = [g[1], pan, g[2], ldb2, ldb4, sb64, g[3], g[0]]
    assert (pan.hdr.width, pan.hdr.height) == (384, 256) and sb64.hdr.log2_sb_size == 6 and g[0].hdr.frame_type == 0 and g[0].hdr.num_ref == 0
    seen = []
    with Batch(lib, 1, 1) as batch:
        for k, j in enumerate(steps):
            what = "step %d: %dx%d, %d-sample super blocks, frame type %d, %d references" % (k, j.hdr.width, j.hdr.height, 1 << j.hdr.log2_sb_size,
                                                                                           j.hdr.frame_type, j.hdr.num_ref)
            hosts = frames([j], pinned)
            batch.round(hosts)
            assert_reference(hosts, what)
            assert_last_launch(batch, hosts, what)
            nsbx, nsby = geometry(j)
            seen.append((nsby, batch.grid(), nsbx * nsby))
    for i, name in enumerate(("rows", "grid", "trace")):
        v = [s[i] for s in seen]
        assert any(v[t] > max(v[:t]) for t in range(1, len(v))), ("the %s never grew" % name, v)


# -------------------------------------------------------------------------------------------------------------------------------------------------
# a second round enqueued while the first is still queued
# -------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["one_batch", "two_batches", pytest.param("reallocating", marks=needs_capture)])
def test_uploads_while_a_launch_is_queued(lib, golden, host_leaves, pinned, request, variant):
    """upload A, run, download A, upload B into the same slots, run, download B, and only then synchronise.  A is four copies of the nine golden
    frames, so the host is still ahead of A's launch when B's uploads return (measured with events behind every call of round A); B puts frame
    (s + 1) % 9 into slot s.  two_batches: B goes to a second batch on the same stream.  reallocating: B's first frame has another geometry, so its
    upload frees buffers round A reads and must wait for it."""
    import torch
    g = golden("hdb_128x136")
    a_jobs = g * 4
    b_jobs = [g[(s + 1) % 9] for s in range(9)]
    if variant == "reallocating":
        b_jobs[0] = [j for j in request.getfixturevalue("captured")["hdb_pan_neg"] if j.hdr.frame_type == 2][0]
    a_hosts, b_hosts = frames(a_jobs, pinned), frames(b_jobs, pinned)
    stream = torch.cuda.ExternalStream(int(lib.tb_stream()))
    marks = []

    def mark():
        e = torch.cuda.Event()
        e.record(stream)
        marks.append(e)
    with contextlib.ExitStack() as stack:
        x = stack.enter_context(Batch(lib, len(a_jobs), 1))
        y = stack.enter_context(Batch(lib, len(b_jobs), 1)) if variant == "two_batches" else x
        for s, hf in enumerate(a_hosts):
            x.upload(s, hf)
            mark()
        x.run(len(a_hosts))
        mark()
        launch_a = marks[-1]
        for s, hf in enumerate(a_hosts):
            x.download(s, hf)
            mark()
        for s, hf in enumerate(b_hosts):
            y.upload(s, hf)
        depth = sum(not e.query() for e in marks)
        a_running = not launch_a.query()
        y.run(len(b_hosts))
        for s, hf in enumerate(b_hosts):
            y.download(s, hf)
        y.sync()
        if y is not x:
            x.sync()
        assert_last_launch(y, b_hosts, "round B")
        if y is not x:
            assert_last_launch(x, a_hosts, "round A")
    print("%s: %d of the %d calls of round A still queued when round B's uploads returned (A's launch %s)" % (variant, depth, len(marks),
          "not finished" if a_running else "finished"))
    assert_reference(a_hosts, "round A")
    assert_reference(b_hosts, "round B")
    assert_host_leaves([hf for hf in b_hosts if hf.job in g], host_leaves, "round B")
    if variant != "reallocating":
        assert a_running and depth > len(a_hosts), ("the host did not run ahead of round A", depth, len(marks))


# -------------------------------------------------------------------------------------------------------------------------------------------------
# tb_rdo_encode_frames' internal batch
# -------------------------------------------------------------------------------------------------------------------------------------------------
def encode_frames_sequence(job_dirs, calls):
    """(in a fresh process, so that tb_rdo_encode_frames' internal batches start empty) tb_rdo_encode_frames on the first n jobs of a golden case,
    call after call; returns each call's return code and every frame's check()"""
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    import thor_b200 as tb
    from thor_b200 import rdo_jobs as RJ
    L = tb.lib
    L.tb_rdo_encode_frames.argtypes = [C.c_void_p, C.c_int]
    L.tb_rdo_last_error.restype = C.c_char_p
    jobs = {case: RJ.load_jobs(d) for case, d in job_dirs.items()}
    keep, out = [], []

    def alloc(nbytes):
        a = np.zeros(max(nbytes, 16), np.uint8); keep.append(a)
        return a.ctypes.data
    for case, n in calls:
        hosts = [RJ.HostFrame(j, alloc) for j in jobs[case][:n]]
        descs = (RJ.RdoFrame * n)(*[hf.desc for hf in hosts])
        rc = L.tb_rdo_encode_frames(descs, n)
        out.append((case, n, rc, L.tb_rdo_last_error().decode() if rc else "", [hf.check() for hf in hosts]))
    return out


def test_encode_frames_grows_and_shrinks_its_internal_batch(tmp_path):
    """n = 1, then 9 (the 8-bit batch is recreated), then 3 (reused), with 16-bit calls in between that grow and reuse the other batch"""
    dirs = {}
    for case in ("hdb_128x136", "hdb_hard_q4_10bit", "hdb_q51_12bit"):
        d = tmp_path / case
        d.mkdir()
        golden_jobs(str(d), case)
        dirs[case] = str(d)
    calls = [("hdb_128x136", 1), ("hdb_q51_12bit", 1), ("hdb_128x136", 9), ("hdb_hard_q4_10bit", 5), ("hdb_128x136", 3), ("hdb_q51_12bit", 3),
             ("hdb_hard_q4_10bit", 2)]
    with ProcessPoolExecutor(1, mp_context=multiprocessing.get_context("spawn")) as ex:
        results = ex.submit(encode_frames_sequence, dirs, calls).result()
    assert len(results) == len(calls)
    for case, n, rc, err, checks in results:
        assert rc == 0, (case, n, err)
        assert len(checks) == n and all(c == {"rec": True, "blk": True, "sb_cost": True} for c in checks), (case, n, checks)


# -------------------------------------------------------------------------------------------------------------------------------------------------
# argument errors on a live batch
# -------------------------------------------------------------------------------------------------------------------------------------------------
def test_argument_errors_leave_the_batch_working(lib, golden, pinned):
    from thor_b200 import rdo_jobs as RJ
    g = golden("hdb_128x136")
    hosts = frames(g[:3], pinned)
    other_size = frames(golden("hdb_q51_12bit")[:1], pinned)[0]
    with Batch(lib, 3, 1) as batch:
        assert lib.tb_rdo_batch_download(batch.b, 0, C.byref(hosts[0].desc)) == TB_ERR_ARG, "download of a slot never uploaded"
        batch.upload(0, hosts[0])
        batch.upload(1, hosts[1])
        assert lib.tb_rdo_batch_run(batch.b, 0) == TB_ERR_ARG, "n_active = 0"
        assert lib.tb_rdo_batch_run(batch.b, 4) == TB_ERR_ARG, "n_active > slots"
        assert lib.tb_rdo_batch_run(batch.b, 3) == TB_ERR_ARG, "slot 2 never uploaded"
        assert lib.tb_rdo_batch_upload(batch.b, 2, C.byref(other_size.desc)) == TB_ERR_ARG, "upload of 16-bit samples into an 8-bit batch"
        assert lib.tb_rdo_batch_run(batch.b, 3) == TB_ERR_ARG, "slot 2 still never uploaded"
        batch.run(2)
        batch.download(0, hosts[0])
        narrow = RJ.RdoFrame.from_buffer_copy(bytes(hosts[1].desc))
        narrow.width = 64
        assert lib.tb_rdo_batch_download(batch.b, 1, C.byref(narrow)) == TB_ERR_ARG, "download into a frame of another geometry"
        batch.download(1, hosts[1])
        batch.sync()
        assert_reference(hosts[:2], "after the errors")
        batch.upload(2, hosts[2])
        batch.round(hosts)
        assert_last_launch(batch, hosts, "after the errors")
    assert_reference(hosts, "after the errors, all three slots")


@pytest.mark.parametrize("width", [120, 88, 8])
def test_16bit_frame_widths_off_the_multiple_of_16_are_refused(lib, golden, pinned, width):
    """16-bit frames whose width is 8 mod 16: chroma widths of 4 mod 8, which the reference's SIMD chroma interpolation predicts unlike its C code in
    rectangular frame-edge blocks.  tb_rdo_batch_upload and tb_rdo_encode_frames refuse them with TB_ERR_ARG and a message, and the batch still
    decides the frames it holds afterwards.  The width is narrowed in a copy of the descriptor of a 128-wide frame (the other checks on it still
    pass): nothing of that frame reaches the device."""
    from thor_b200 import rdo_jobs as RJ
    hosts = frames(golden("hdb_hard_q4_10bit")[:2], pinned)
    odd = RJ.RdoFrame.from_buffer_copy(bytes(hosts[1].desc))
    odd.width = width
    lib.tb_rdo_encode_frames.argtypes = [C.c_void_p, C.c_int]
    with Batch(lib, 2, 2) as batch:
        batch.upload(0, hosts[0])
        assert lib.tb_rdo_batch_upload(batch.b, 1, C.byref(odd)) == TB_ERR_ARG
        assert b"multiples of 16" in lib.tb_rdo_last_error(), lib.tb_rdo_last_error()
        assert lib.tb_rdo_batch_run(batch.b, 2) == TB_ERR_ARG, "slot 1 was never uploaded"
        descs = (RJ.RdoFrame * 2)(hosts[0].desc, odd)
        assert lib.tb_rdo_encode_frames(descs, 2) == TB_ERR_ARG
        assert b"multiples of 16" in lib.tb_rdo_last_error(), lib.tb_rdo_last_error()
        batch.upload(1, hosts[1])
        batch.run(2)
        for s, hf in enumerate(hosts):
            batch.download(s, hf)
        batch.sync()
        assert_last_launch(batch, hosts, "after the refused uploads")
    assert_reference(hosts, "after the refused uploads")
