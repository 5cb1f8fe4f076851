"""CPU: the host rules of offline jobs in a stream group (StreamGroup.submit): codec tiles at the steady slice lengths,
the rule by which jobs take the filler slots of a tick's planned calls, and the argument checks of submit()."""
import random
from types import SimpleNamespace

import pytest
import torch

from sam_audio_b200.stream import SeparationJob, StreamGroup
from sam_audio_b200.windows import (stream_bucket, stream_drain_bucket, stream_group_capacity, stream_hop,
                                    stream_job_admit, stream_job_min_frames, stream_job_slots, stream_steady_slices,
                                    stream_tiles)

HOP, HALO_ENC, HALO_DEC = 1920, 6, 8          # the standard codec rates (sab_codec_tiling reports these halos)


def _check_tiles(n, L, h, tiles):
    assert tiles[0][0] == 0 and tiles[0][1] == 0
    assert tiles[-1][0] + L == n and tiles[-1][2] == n
    covered = [0] * n
    for start, k0, k1 in tiles:
        assert 0 <= start and start + L <= n                     # every tile has the steady length, inside [0, n)
        assert start <= k0 < k1 <= start + L
        if start > 0:                                            # an interior cut on the left
            assert k0 >= start + h
        if start + L < n:                                        # an interior cut on the right
            assert k1 <= start + L - h
        for t in range(k0, k1):
            covered[t] += 1
    assert covered == [1] * n                                    # the kept rows cover [0, n) exactly once
    assert [k0 for _, k0, _ in tiles[1:]] == [k1 for _, _, k1 in tiles[:-1]]   # in order
    assert [s for s, _, _ in tiles] == sorted(s for s, _, _ in tiles)


@pytest.mark.parametrize("W", [8, 9, 16, 50, 250])
@pytest.mark.parametrize("halo", [HALO_ENC, HALO_DEC, 1, 3])
def test_tiles_at_the_steady_length(W, halo):
    """For every n from the job's minimum length up to many tiles: tiles of exactly H + 2 * halo frames, the first at
    0, the last ending at n, kept rows at least a halo away from every interior cut and covering [0, n) once."""
    L = stream_hop(W) + 2 * halo
    for n in list(range(L, L + 3 * stream_hop(W) + 5)) + [L * 17 + 3, 15_000, 15_001]:
        _check_tiles(n, L, halo, stream_tiles(n, L, halo))


def test_tiles_brute_force_random():
    rng = random.Random(0)
    for _ in range(2000):
        h = rng.randint(0, 12)
        L = rng.randint(2 * h + 1, 2 * h + 60)
        n = rng.randint(L, L * 8)
        _check_tiles(n, L, h, stream_tiles(n, L, h))


def test_tiles_refuse_what_they_cannot_cut():
    with pytest.raises(ValueError, match="n >= L > 2"):
        stream_tiles(10, 11, 2)
    with pytest.raises(ValueError, match="n >= L > 2"):
        stream_tiles(100, 12, 6)
    assert stream_tiles(12, 12, 3) == [(0, 0, 12)]


def test_steady_slices_and_minimum():
    for W in (8, 50, 250, 10000):
        H = stream_hop(W)
        assert stream_steady_slices(W, HALO_ENC, HALO_DEC) == (H + 2 * HALO_ENC, H + 2 * HALO_DEC)
        assert stream_job_min_frames(W, HALO_ENC, HALO_DEC) == H + 2 * HALO_DEC


def test_admission_fifo():
    assert stream_job_admit([3, 5, 2], 4) == [3, 1, 0]
    assert stream_job_admit([0, 5, 2], 4) == [0, 4, 0]
    assert stream_job_admit([1, 0, 2], 9) == [1, 0, 2]
    assert stream_job_admit([4, 4], 0) == [0, 0]
    assert stream_job_admit([], 3) == []


@pytest.mark.parametrize("capacity", [1, 3, 8, 400])
def test_slots_with_jobs_keep_the_call(capacity):
    """Job items only take filler slots: the call keeps its size (the bucket of its live items), live items keep their
    slots, job items follow them in order, and without job items the slots are stream_bucket's."""
    for n_live in range(1, capacity + 1):
        base = stream_bucket(n_live, capacity)
        assert stream_job_slots(n_live, len(base), 0) == base
        for n_jobs in range(0, len(base) - n_live + 1):
            slots = stream_job_slots(n_live, len(base), n_jobs)
            assert len(slots) == len(base)
            assert slots[:n_live + n_jobs] == list(range(n_live + n_jobs))
            assert all(0 <= x < n_live for x in slots[n_live + n_jobs:])
        with pytest.raises(ValueError):
            stream_job_slots(n_live, len(base), len(base) - n_live + 1)


def test_drain_uses_resident_buckets():
    assert stream_drain_bucket(1, set()) == 1 and stream_drain_bucket(7, set()) == 1
    assert stream_drain_bucket(3, {1, 4, 8}) == 4
    assert stream_drain_bucket(8, {1, 4, 8}) == 8
    assert stream_drain_bucket(30, {1, 4, 8}) == 8
    assert stream_drain_bucket(1, {2, 16}) == 2


class _JobSim:
    """A host-only SeparationJob (its tile plans and counters, no device state) advanced as StreamGroup advances it.
    The items it offers come from the job's own _encode_offer / _solve_offer / _decode_offer; taking them checks them
    against brute force: a window's features [k * H, min(k * H + W, n_final)) are encoded, a decode tile's latent frames
    are all final, and windows and tiles go in order."""

    def __init__(self, n_final, W):
        job = SeparationJob.__new__(SeparationJob)
        job.W, job.H = W, stream_hop(W)
        job._init_schedule(n_final, HALO_ENC, HALO_DEC)
        self.job, self.solve_log, self.dec_log = job, [], []
        self.offers = {"encode": job._encode_offer, "solve": job._solve_offer, "decode": job._decode_offer}

    def offer(self, step):
        return self.offers[step]()

    def take(self, step, t):
        j = self.job
        assert 0 <= t <= self.offer(step)
        if step == "encode":
            for _, k0, k1 in j._enc_tiles[j._enc_next:j._enc_next + t]:
                assert k0 == j._enc_end
                j._enc_end = k1
            j._enc_next += t
        elif step == "solve":
            for k in range(j.windows_solved, j.windows_solved + t):
                assert min(k * j.H + j.W, j.n_final) <= j._enc_end
            self.solve_log += list(range(j.windows_solved, j.windows_solved + t))
            j.windows_solved += t
            j.final_frames = j.n_final if j._ends_at(j.windows_solved) else j.windows_solved * j.H
        else:
            for start, _, _ in j._dec_tiles[j._dec_next:j._dec_next + t]:
                assert start + j._dec_len <= j.final_frames
            self.dec_log += list(range(j._dec_next, j._dec_next + t))
            j._dec_next += t

    @property
    def done(self):
        return self.job._dec_next == len(self.job._dec_tiles)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_jobs_fill_only_filler_slots_in_order(seed):
    """Push ticks with random live item counts per call: every call keeps its live bucket, job items never exceed its
    filler slots, a later job takes slots only when the earlier ones have nothing ready, and every job's windows and
    decode tiles go in order.  Ticks that hold only jobs then finish them at resident buckets."""
    rng = random.Random(seed)
    W = rng.choice([50, 250])
    cap = stream_group_capacity(W, 100_000)
    jobs = [_JobSim(rng.randint(stream_job_min_frames(W, HALO_ENC, HALO_DEC), 40 * W), W) for _ in range(3)]
    resident = set()
    for tick in range(60):
        queue = [j for j in jobs[:1 + tick // 20] if not j.done]
        for step in ("encode", "solve", "decode"):
            if rng.random() < 0.2:
                continue                                         # no live call of the steady length in this tick
            n_live = rng.randint(1, 12)
            size = len(stream_bucket(n_live, cap))
            if step == "solve":
                resident.add(size)
            offers = [j.offer(step) for j in queue]
            taken = stream_job_admit(offers, size - n_live)
            assert sum(taken) <= size - n_live
            for i, (o, t) in enumerate(zip(offers, taken)):
                assert t <= o
                if t < o:
                    assert not any(taken[i + 1:])                # first in, first out
            slots = stream_job_slots(n_live, size, sum(taken))
            assert len(slots) == size and slots[:n_live] == list(range(n_live))
            for j, t in zip(queue, taken):
                j.take(step, t)
    for _ in range(10_000):                                      # drain: ticks that hold only jobs
        queue = [j for j in jobs if not j.done]
        if not queue:
            break
        for step in ("encode", "solve", "decode"):
            offers = [j.offer(step) for j in queue]
            if not any(offers):
                continue
            size = stream_drain_bucket(sum(offers), resident)
            assert size in (resident or {1})
            for j, t in zip(queue, stream_job_admit(offers, size)):
                j.take(step, t)
    for j in jobs:
        assert j.done and j.solve_log == list(range(j.job.windows_total))
        assert j.dec_log == list(range(len(j.job._dec_tiles)))


def _fake_group(closed=False, W=50):
    model = SimpleNamespace(sample_rate=48000)
    return SimpleNamespace(closed=closed, model=model, W=W, hop=HOP, halo_enc=HALO_ENC, halo_dec=HALO_DEC)


def test_submit_argument_checks():
    g = _fake_group()
    long = torch.zeros(48000 * 30)
    with pytest.raises(RuntimeError, match="closed"):
        StreamGroup.submit(_fake_group(closed=True), long, "rain")
    with pytest.raises(TypeError, match="one string"):
        StreamGroup.submit(g, long, ["rain", "dog"])
    with pytest.raises(TypeError, match="submit\\(\\) takes a tensor"):
        StreamGroup.submit(g, long.numpy(), "rain")
    for bad in (torch.zeros(2, 3, 48000), torch.zeros(0), torch.zeros(2, 0), torch.zeros(9, 48000 * 30)):
        with pytest.raises(ValueError, match="1 <= C <= 8"):
            StreamGroup.submit(g, bad, "rain")
    for rate in (7999, 192001, 16000.5, True):
        with pytest.raises(ValueError, match="rates are integers"):
            StreamGroup.submit(g, long, "rain", sample_rate=rate)
    # W = 50: H = 44, so a job needs 44 + 2 * 8 = 60 frames (2.4 s); 59 frames of samples are too short
    need = stream_job_min_frames(50, HALO_ENC, HALO_DEC)
    with pytest.raises(ValueError, match="too short.*separate\\(\\) or stream\\(\\)"):
        StreamGroup.submit(g, torch.zeros((need - 1) * HOP), "rain")
    # the length counts at the codec's rate: 2.4 s at 16 kHz minus one sample resamples to 59 frames and a bit
    with pytest.raises(ValueError, match="too short"):
        StreamGroup.submit(g, torch.zeros(2, need * HOP // 3 - 1 - HOP // 3), "rain", sample_rate=16000)


def test_result_before_done_raises():
    """result() refuses a job that is not done (or was cancelled); cancel() works on a job whose group is gone."""
    job = SeparationJob.__new__(SeparationJob)
    job.done = job.cancelled = False
    job.windows_solved, job.windows_total = 3, 9
    job._group = lambda: None
    with pytest.raises(RuntimeError, match="not done \\(3 of 9 windows"):
        job.result()
    job.cancel()
    with pytest.raises(RuntimeError, match="cancelled"):
        job.result()
