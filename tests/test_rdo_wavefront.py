"""The RD loop's wavefront at the widths of the benchmark's frames (GPU).  tests/test_rdo_matrix.py's strips of a 1080p HDB and a 2160p RA encode
(15 and 30 super-block columns), three copies of every frame in one launch of the batch API with the per-super-block trace: every frame must
return the reference's decisions, every super block must start after its left and up-right neighbours have ended, and the rows of a frame must
overlap: a row starts once the row above is two super blocks ahead, not once it has finished.  Frames three super blocks wide or less, as in the
rest of the suite, leave no room for that overlap."""
import numpy as np
import pytest

from test_rdo_batch_api import Batch, frames, geometry, lib, pinned  # noqa: F401  (fixtures)
from test_rdo_matrix import captured_cases, needs_capture  # noqa: F401  (fixture)
from test_rdo_sched import check_dependencies

pytestmark = pytest.mark.gpu

STRIPS = ["hdb_1080_strip", "ra_2160_strip"]
COPIES = 3


@needs_capture
def test_wavefront_at_1080p_and_2160p_widths(lib, pinned, captured_cases):
    jobs = [j for name, (_, js) in captured_cases(STRIPS).items() for j in js]
    assert {geometry(j)[0] for j in jobs} == {15, 30}
    from thor_b200 import rdo_jobs as RJ
    first = frames(jobs, pinned)
    hosts = first + [RJ.HostFrame(hf.job, pinned, share_inputs=hf) for _ in range(COPIES - 1) for hf in first]   # copies upload from the same inputs
    with Batch(lib, len(hosts), 1) as batch:
        batch.round(hosts)
        rec = batch.trace()
        grid = batch.grid()
    bad = [(k, hf.job.hdr.width, hf.job.frame_num, r) for k, hf in enumerate(hosts) for r in [hf.check()] if not all(r.values())]
    assert not bad, ("%d of %d frames differ from the reference's decisions" % (len(bad), len(hosts)), bad[:6])
    tr = {k: rec[k] for k in rec.dtype.names}
    tr["nsbx"] = np.array([geometry(hf.job)[0] for hf in hosts])
    tr["nsby"] = np.array([geometry(hf.job)[1] for hf in hosts])
    assert ((tr["cta"] >= 0) & (tr["cta"] < grid)).all()
    assert (tr["t_end"] >= tr["t_start"]).all()
    check_dependencies(tr)
    serial = []
    for f, hf in enumerate(hosts):
        nsbx = int(tr["nsbx"][f])
        m = tr["frame"] == f
        row, col = tr["row"][m], tr["col"][m]
        last_of_row0 = tr["t_start"][m][(row == 0) & (col == nsbx - 1)]
        row1_ends = tr["t_end"][m][row == 1]
        if not (row1_ends.min() < last_of_row0[0]):
            serial.append((f, hf.job.hdr.width, hf.job.frame_num))
    assert not serial, ("frames whose row 1 ran after row 0 had finished (no wavefront)", serial[:8])
