"""GPU tests of the device -> host copy of the computeAlignments and LowHash0 results under every state of the host blocks.

The results are copied out while the later batches still run: by direct DMA into page-locked blocks (the library's large
result blocks once recycled), through a pinned staging ring and copier threads into pageable ones (a fresh block, or one
whose first owner still holds it), and the compressed bytes' block grows when the previous call's bytes per candidate fall
short. What a call returns must not depend on which of these paths it took. The host pool is per process, so the calls run
in a fresh subprocess (this file run as a script) in a fixed order, and the test compares what it wrote. The candidate sets
are tiled so that the result blocks exceed the pool's 8 MiB threshold for recycled blocks, and SHB_ALIGN_BATCH cuts them
into many batches."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _path in (HERE, ROOT):                      # run as the subprocess
    if _path not in sys.path:
        sys.path.insert(0, _path)

from oracle import bindings as B  # noqa: E402
from shasta_b200 import synth  # noqa: E402
from support import candidate_set, oracle_options  # noqa: E402

OPTS = dict(alignMethod=3, k=14, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10, minAlignedFraction=0.1,
            downsamplingFactor=0.05, bandExtend=10, maxBand=1000)
TILES = 60                                      # 60 x 3000 candidates: 11.5 MB of AlignmentData records at most
BATCH = 4096
# LowHash0 on 3000 reads of a 4000-marker genome: every read overlaps hundreds of others, about 2 M candidates (24 MB).
LOWHASH_SET = dict(reads=3000, k=14, genome_markers=4000, n50_bases=12000, min_bases=8000, seed=11)
LOWHASH = dict(m=4, hashFraction=0.01, minHashIterationCount=20, minBucketSize=2, maxBucketSize=1000, minFrequency=2)


def align_inputs():
    """The markers, the base candidates, and which of them the GPU keeps (from the oracle, so without the GPU)."""
    d, cand = candidate_set(500, 14, 77, genome_markers=30000)
    base = np.ascontiguousarray(cand[:3000])
    orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], base, oracle_options(OPTS), threads=8)
    return d, base, orec, otoc, odata


def tiled(rec, toc, data, tiles):
    """The result of a candidate set repeated `tiles` times: the records and bytes repeat, the toc is rebased."""
    n, nb = len(rec), int(toc[-1])
    rtoc = np.concatenate([toc[:-1].astype(np.uint64) + np.uint64(t * nb) for t in range(tiles)] + [np.array([tiles * nb], np.uint64)])
    return np.tile(rec, (tiles, 1)).reshape(tiles * n, 16), rtoc, np.tile(data, tiles)


def kept_mask(base, orec):
    """Which base candidates have a stored alignment (a record starts with the candidate's read ids and isSameStrand)."""
    kept = {(int(r[0]), int(r[1]), int(r[2])) for r in orec}
    return np.array([(int(c[0]), int(c[1]), int(c[2])) in kept for c in base])


# ---- the subprocess ----------------------------------------------------------------------------------------------------
def worker(out_dir):
    from shasta_b200 import capi
    d, base, orec, otoc, odata = align_inputs()
    keep = kept_mask(base, orec)
    full = np.ascontiguousarray(np.tile(base, (TILES, 1)))
    longer = np.ascontiguousarray(np.tile(base[keep], (TILES, 1)))         # only kept candidates: more bytes per candidate
    none = np.ascontiguousarray(np.tile(base[~keep], (TILES, 1)))          # no stored alignment at all
    ctx = capi.Context(0)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    opts = capi.make_align_options(**OPTS)

    def align(name, cand):
        rec, ctoc, cdata, res = capi.compute_alignments(ctx, cand, opts)
        np.savez(os.path.join(out_dir, name + ".npz"), rec=rec, ctoc=ctoc, cdata=cdata,
                 digests=np.array([res.alignmentDataDigest, res.compressedDigest], np.uint64))
        return rec, ctoc, cdata

    first = align("first", full)                       # first call of the process: fresh, pageable blocks
    held = align("held", full)                         # the first call's blocks are still held: fresh blocks again
    del first, held
    gc.collect()
    align("recycled", full)                            # recycled, page-locked blocks (those the first two calls freed)
    gc.collect()
    align("recycled2", full)
    gc.collect()
    align("longer", longer)                            # the data block outgrows the previous call's estimate
    gc.collect()
    align("longer_again", longer)
    gc.collect()
    align("no_alignments", none)
    align("no_candidates", np.zeros((0, 3), np.uint32))
    ctx.close()

    # LowHash0 on its own context
    d = synth.generate(synth.SynthParams(**LOWHASH_SET))
    ctx = capi.Context(0)
    lp = capi.make_lowhash_params(**LOWHASH)

    def lowhash(name):
        cand, _, res = ctx.find_alignment_candidates_lowhash0(d["toc"], d["data"], d["flags"], lp)
        np.savez(os.path.join(out_dir, "lowhash_" + name + ".npz"), cand=cand, digest=np.array([res.candidateDigest], np.uint64))
        return cand

    first = lowhash("first")
    held = lowhash("held")
    del first, held
    gc.collect()
    lowhash("recycled")
    gc.collect()
    lowhash("recycled2")
    ctx.close()


# ---- the test ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def outputs(tmp_path_factory):
    out = tmp_path_factory.mktemp("result_copy")
    flags = [f for f, on in (("-I", sys.flags.isolated), ("-E", sys.flags.ignore_environment), ("-s", sys.flags.no_user_site)) if on]
    env = dict(os.environ, SHB_ALIGN_BATCH=str(BATCH))
    proc = subprocess.run([sys.executable, *flags, os.path.abspath(__file__), str(out)], cwd=ROOT, env=env,
                          capture_output=True, text=True, timeout=1200)
    assert proc.returncode == 0, f"worker failed:\n{proc.stdout[-3000:]}\n{proc.stderr[-3000:]}"
    return out


def _load(out, name):
    return np.load(os.path.join(out, name + ".npz"))


def _same(got, want):
    return all(np.array_equal(got[k], want[k]) for k in ("rec", "ctoc", "cdata", "digests"))


@pytest.fixture(scope="module")
def expected():
    _, base, orec, otoc, odata = align_inputs()
    # the kept candidates alone store the same alignments as the whole set
    return dict(full=tiled(orec, otoc, odata, TILES), keep=kept_mask(base, orec), base=base)


@pytest.mark.gpu
def test_first_call_matches_oracle(outputs, expected):
    got = _load(outputs, "first")
    rec, toc, data = expected["full"]
    assert len(got["rec"]) == len(rec) and 64 * len(rec) >= 8 << 20
    assert np.array_equal(got["rec"], rec) and np.array_equal(got["ctoc"], toc) and np.array_equal(got["cdata"], data)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["held", "recycled", "recycled2"])
def test_calls_on_other_blocks_match_first(outputs, name):
    assert _same(_load(outputs, name), _load(outputs, "first"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["longer", "longer_again"])
def test_data_block_growth(outputs, expected, name):
    got = _load(outputs, name)
    rec, toc, data = expected["full"]
    assert np.array_equal(got["rec"], rec) and np.array_equal(got["ctoc"], toc) and np.array_equal(got["cdata"], data)
    # the call before "longer" sized its data block from a smaller number of bytes per candidate
    full_rate = int(_load(outputs, "recycled2")["ctoc"][-1]) / (TILES * len(expected["base"]))
    candidates = TILES * int(expected["keep"].sum())
    assert len(data) > full_rate * candidates * 1.03 + (1 << 20)
    assert _same(got, _load(outputs, "longer"))


@pytest.mark.gpu
def test_no_alignments_and_no_candidates(outputs):
    for name in ("no_alignments", "no_candidates"):
        got = _load(outputs, name)
        assert len(got["rec"]) == 0 and len(got["cdata"]) == 0 and list(got["ctoc"]) == [0], name
        assert list(got["digests"]) == list(_load(outputs, "no_candidates")["digests"]), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["held", "recycled", "recycled2"])
def test_lowhash_candidates_match_first(outputs, name):
    first, got = _load(outputs, "lowhash_first"), _load(outputs, "lowhash_" + name)
    assert 12 * len(first["cand"]) >= 8 << 20
    assert np.array_equal(got["cand"], first["cand"]) and np.array_equal(got["digest"], first["digest"])


if __name__ == "__main__":
    worker(sys.argv[1])
