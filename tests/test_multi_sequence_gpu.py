"""GPU tests of one context tracking several sequences per batch (plf_set_max_sequences / plf_batch_run_sequences).

The oracle is the library itself: every pair of a mixed batch must give, bit for bit, what a single-sequence context gives
when that sequence's frames are fed to it alone and in the same order - every plf_frame_result field (DT included),
get_frame(k) and get_matches(k)."""
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import synth

pytestmark = pytest.mark.gpu

CAM = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
PRM = dict(orb_nfeatures=700, lsd_nfeatures=150)
LENGTHS = (8, 12, 10, 9)

_FRAMES = {}


def sequences():
    """Four sequences of LENGTHS pairs, each through its own synth.World."""
    if "seqs" not in _FRAMES:
        seqs = []
        for s, n in enumerate(LENGTHS):
            world = synth.World(seed=40 + s, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
            seqs.append([(L, R) for L, R, _ in synth.stream(CAM, n, world=world, seed=50 + s, step=0.15)])
        _FRAMES["seqs"] = seqs
    return _FRAMES["seqs"]


def limits(B):
    lim = plf.default_limits()
    lim.max_batch = B
    return lim


def collect(fe, keys, res, out):
    for k, key in enumerate(keys):
        out[key] = (res[k], fe.get_frame(k), fe.get_matches(k))


def alone(seqs, prm, restarts=(), cam=CAM):
    """Each sequence on its own through one single-sequence context: reset_sequence() before it and before every pair
    (s, i) in `restarts`.  Returns {(s, i): (result, frame, matches)}."""
    out = {}
    with plf.Frontend(camera=cam, limits=limits(max(len(f) for f in seqs)), **prm) as fe:
        for s, frames in enumerate(seqs):
            cuts = sorted({0, len(frames)} | {i for q, i in restarts if q == s})
            for a, b in zip(cuts, cuts[1:]):
                fe.reset_sequence()
                fe.batch_upload(np.stack([f[0] for f in frames[a:b]]), np.stack([f[1] for f in frames[a:b]]))
                fe.batch_run(b - a)
                collect(fe, [(s, i) for i in range(a, b)], fe.batch_download_array(b - a), out)
    return out


def batch_args(seqs, batch, restarts):
    L = np.stack([seqs[s][i][0] for s, i in batch])
    R = np.stack([seqs[s][i][1] for s, i in batch])
    seq = np.array([s for s, _ in batch], np.int32)
    rst = np.array([(s, i) in restarts for s, i in batch]) if restarts else None
    return L, R, seq, rst


def mixed(seqs, batches, prm, restarts=(), nseq=4, cam=CAM):
    """The batches (lists of (s, i)) one after the other through one context with max_sequences = nseq; restart flags on
    the pairs in `restarts`.  Returns {(s, i): (result, frame, matches)}."""
    out = {}
    with plf.Frontend(camera=cam, limits=limits(max(map(len, batches))), max_sequences=nseq, **prm) as fe:
        for batch in batches:
            L, R, seq, rst = batch_args(seqs, batch, restarts)
            fe.batch_upload(L, R)
            fe.batch_run(len(batch), seq=seq, restart=rst)
            collect(fe, batch, fe.batch_download_array(len(batch)), out)
    return out


def assert_same(ref, got):
    assert ref.keys() == got.keys()
    for key in ref:
        (ra, fa, ma), (rb, fb, mb) = ref[key], got[key]
        for f in ra.dtype.names:   # field for field, bit for bit (DT included)
            assert ra[f].tobytes() == rb[f].tobytes(), (key, f)
        for da, db in ((fa, fb), (ma, mb)):
            assert da.keys() == db.keys()
            for k in da:
                assert da[k].shape == db[k].shape and da[k].tobytes() == db[k].tobytes(), (key, k)


def chunks(order, B):
    return [order[i:i + B] for i in range(0, len(order), B)]


def interleavings(lengths=LENGTHS):
    """contiguous blocks: the sequences one after the other in batches of 7 (so batches hold blocks of unequal size);
    round robin: one pair of every sequence per batch (B = 4); random: a seeded merge in batches of 6; absent: sequences
    0, 1 for two batches, then 2, 3 for two batches, ..., two pairs of each present sequence per batch, so each carried
    frame waits through runs without its sequence and sequences 2 and 3 first appear in the third batch."""
    n = len(lengths)
    blocks = chunks([(s, i) for s in range(n) for i in range(lengths[s])], 7)
    rr = [[(s, i) for s in range(n) if i < lengths[s]] for i in range(max(lengths))]
    rng = np.random.default_rng(0)
    pos, order = [0] * n, []
    while len(order) < sum(lengths):
        s = int(rng.choice([q for q in range(n) if pos[q] < lengths[q]]))
        order.append((s, pos[s]))
        pos[s] += 1
    absent, pos, t = [], [0] * n, 0
    while any(pos[q] < lengths[q] for q in range(n)):
        group = (0, 1) if (t // 2) % 2 == 0 else (2, 3)
        batch = []
        for s in group:
            take = min(2, lengths[s] - pos[s])
            batch += [(s, pos[s] + j) for j in range(take)]
            pos[s] += take
        if batch:
            absent.append(batch)
        t += 1
    return {"blocks": blocks, "round_robin": rr, "random": chunks(order, 6), "absent": absent}


def test_interleavings_are_what_they_claim():
    runs = interleavings()
    for name, batches in runs.items():
        flat = [key for b in batches for key in b]
        assert sorted(flat) == sorted((s, i) for s in range(4) for i in range(LENGTHS[s])), name
        for s in range(4):   # temporal order within each sequence
            assert [i for q, i in flat if q == s] == list(range(LENGTHS[s])), name
    assert all(len(b) == 4 for b in runs["round_robin"][:8])
    first = {s: next(j for j, b in enumerate(runs["absent"]) if any(q == s for q, _ in b)) for s in range(4)}
    assert first[2] == first[3] == 2
    assert any(len({q for q, _ in b}) < 4 for b in runs["random"])


@pytest.mark.parametrize("variant", ["default", "matching_strategy_3", "no_points", "no_lines"])
def test_mixed_batches_equal_each_sequence_alone(built, variant):
    """Four sequences of 8-12 pairs in four interleavings (contiguous blocks of unequal size, round robin with B = 4, a
    seeded random merge, batches that leave sequences out for two runs): every pair equals the sequence run alone.
    matching_strategy = 3 takes the windowed frame-to-frame path (per-problem query slots of the batched matchGrid)."""
    prm = dict(PRM, **{"default": {}, "matching_strategy_3": dict(matching_strategy=3),
                       "no_points": dict(has_points=0), "no_lines": dict(has_lines=0)}[variant])
    seqs = sequences()
    ref = alone(seqs, prm)
    tracked = sum(r["status"] == 0 for r, _, _ in ref.values())
    assert tracked >= sum(LENGTHS) // 2, tracked   # the sequences do track
    for name, batches in interleavings().items():
        got = mixed(seqs, batches, prm)
        assert_same(ref, got)
        for s in range(4):
            assert got[(s, 0)][0]["status"] == 2, (name, s)


RESTARTS = ((1, 5), (2, 3), (0, 6), (3, 1))


@pytest.mark.parametrize("name", ["blocks", "round_robin", "absent"])
def test_restart_flags(built, name):
    """restart[k] makes pair k a first frame (status 2) and the sequence's next pair tracks against it; a sequence's first
    pair in a later batch is a first frame too.  Equal to a single-sequence context with reset_sequence() at the same
    points."""
    seqs = sequences()
    ref = alone(seqs, PRM, restarts=RESTARTS)
    got = mixed(seqs, interleavings()[name], PRM, restarts=RESTARTS)
    assert_same(ref, got)
    for s, i in RESTARTS + tuple((s, 0) for s in range(4)):
        assert got[(s, i)][0]["status"] == 2, (s, i)
    for s, i in RESTARTS:
        assert got[(s, i + 1)][0]["status"] == 0 and got[(s, i + 1)][0]["n_matched_pt"] > 0, (s, i)


def test_three_batches_in_flight(built):
    """Up to three batches in flight, each with its own sequence table and restart flags: the pinned ring of tables and the
    per-batch device table are not overwritten while a batch waits.  Results equal the batches run one at a time; the
    frames and matches of the last batch (get_frame / get_matches refer to the batch most recently run) too."""
    seqs = sequences()
    batches = interleavings()["random"]
    restarts = ((1, 5), (2, 3))
    ref = mixed(seqs, batches, PRM, restarts=restarts)
    got = {}
    with plf.Frontend(camera=CAM, limits=limits(6), max_sequences=4, **PRM) as fe:
        pending = []
        for j, batch in enumerate(batches):
            L, R, seq, rst = batch_args(seqs, batch, restarts)
            fe.batch_upload(L, R)
            fe.batch_run(len(batch), seq=seq, restart=rst)
            pending.append(batch)
            if len(pending) == 3 or j == len(batches) - 1:
                while pending:
                    b = pending.pop(0)
                    res = fe.batch_download_array(len(b))
                    for k, key in enumerate(b):
                        got[key] = res[k]
        last = batches[-1]
        frames = {key: (fe.get_frame(k), fe.get_matches(k)) for k, key in enumerate(last)}
    assert got.keys() == ref.keys()
    for key in ref:
        for f in got[key].dtype.names:
            assert got[key][f].tobytes() == ref[key][0][f].tobytes(), (key, f)
    for key, (fr, ma) in frames.items():
        for a, b in ((fr, ref[key][1]), (ma, ref[key][2])):
            for k in a:
                assert a[k].tobytes() == b[k].tobytes(), (key, k)


def test_default_sequence_is_the_single_sequence_path(built):
    """batch_run(B) equals batch_run(B, seq=zeros) bit for bit, and a context sized for three sequences that only uses
    sequence 0 equals a max_sequences = 1 context."""
    frames = sequences()[1]
    batches = chunks([(0, i) for i in range(len(frames))], 5)
    seqs = [frames]

    def run(nseq, explicit):
        out = {}
        with plf.Frontend(camera=CAM, limits=limits(5), max_sequences=nseq, **PRM) as fe:
            for batch in batches:
                L, R, seq, _ = batch_args(seqs, batch, ())
                fe.batch_upload(L, R)
                fe.batch_run(len(batch), seq=seq if explicit else None)
                collect(fe, batch, fe.batch_download_array(len(batch)), out)
        return out
    base = run(1, False)
    assert_same(base, run(1, True))
    assert_same(base, run(3, True))
    assert_same(base, alone(seqs, PRM))


def test_errors_leave_the_sequences_unchanged(built):
    """seq out of range or negative: PLF_ERR_INVALID before anything is enqueued; the next valid batch, on the same upload,
    gives the results of an uninterrupted run.  plf_set_max_sequences after the first upload: PLF_ERR_STATE; n < 1:
    PLF_ERR_INVALID."""
    seqs = sequences()[:2]
    batches = [[(0, 0), (1, 0), (0, 1), (1, 1)], [(1, 2), (0, 2), (1, 3), (0, 3)]]
    ref = alone([s[:4] for s in seqs], PRM)
    got = {}
    with plf.Frontend(camera=CAM, limits=limits(4), max_sequences=2, **PRM) as fe:
        for batch in batches:
            L, R, seq, _ = batch_args(seqs, batch, ())
            fe.batch_upload(L, R)
            for bad in ([0, 2, 0, 1], [1, 0, -1, 0]):
                with pytest.raises(plf.PlfError, match=r"plf_batch_run_sequences failed \(-1\).*outside \[0, 2\)"):
                    fe.batch_run(4, seq=np.array(bad, np.int32), restart=np.ones(4, bool))
            fe.batch_run(4, seq=seq)
            collect(fe, batch, fe.batch_download_array(4), got)
            with pytest.raises(plf.PlfError, match="no batch in flight"):
                fe.batch_download(4)
        with pytest.raises(plf.PlfError, match=r"plf_set_max_sequences failed \(-5\)"):
            fe._check(fe.lib.plf_set_max_sequences(fe._ctx, 3), "plf_set_max_sequences")
    assert_same(ref, got)
    for n in (0, -2):
        with pytest.raises(plf.PlfError, match=r"plf_set_max_sequences failed \(-1\)"):
            plf.Frontend(camera=CAM, limits=limits(1), max_sequences=n)
    with plf.Frontend(camera=CAM, limits=limits(1)) as fe:   # before the first upload the count may still change
        fe._check(fe.lib.plf_set_max_sequences(fe._ctx, 5), "plf_set_max_sequences")
        with pytest.raises(plf.PlfError, match="seq must be a 1-D integer array of 1 entries"):
            fe.batch_run(1, seq=np.zeros(2, np.int32))


def test_live_cameras_at_kitti_shape(built):
    """32 live cameras at KITTI shape: one batch of B = 32 per step holds one pair of every sequence, for 4 steps.  Each
    sequence equals itself run alone through a single-sequence context (reset_sequence() between sequences)."""
    n, steps = 32, 4
    cam = plf.KITTI_CAMERA
    world = synth.World(seed=7)
    seqs = [[(L, R) for L, R, _ in synth.stream(cam, steps, world=world, seed=100 + s)] for s in range(n)]
    prm = dict(orb_nfeatures=1500, lsd_nfeatures=200)
    ref = alone(seqs, prm, cam=cam)
    got = mixed(seqs, [[(s, i) for s in range(n)] for i in range(steps)], prm, nseq=n, cam=cam)
    assert_same(ref, got)
    assert sum(got[(s, i)][0]["status"] == 0 for s in range(n) for i in range(1, steps)) >= 0.75 * n * (steps - 1)
