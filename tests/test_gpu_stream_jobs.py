"""GPU (H100) tests of offline jobs in stream groups (StreamGroup.submit, sam_audio_b200/stream.py): a job's result equals
SAMAudio.stream() with the whole recording pushed once and flushed, bit for bit; live streams are bit-identical with and
without jobs in their group; jobs add no planned call, change no item count and build no plan in push ticks; cancel()
frees a job's memory."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SR = 48000
PROMPTS = ["man speaking", "dog barking loudly", "a piano", "rain on the roof", "a crowd cheering at night"]


@pytest.fixture(scope="module")
def small_model():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.model import build_synthetic_model
    return build_synthetic_model("sam-audio-small", seed=0, device="cuda:0", weights_device="cuda:0")


def _recording(seconds, seed, rate=SR, channels=1):
    from sam_audio_b200.synthetic import synthetic_clip
    n = int(rate * seconds)
    x = torch.stack([synthetic_clip(seed + 100 * c, n).reshape(-1) for c in range(channels)]).cuda()
    return x[0] if channels == 1 else x


def _cat(outs):
    return torch.cat([o.target for o in outs]), torch.cat([o.residual for o in outs])


def _stream_whole(model, wav, prompt, seed, window_seconds, rate=None):
    """The stream a job equals: the whole recording pushed once, then flushed."""
    s = model.stream(prompt, window_seconds=window_seconds, seed=seed, sample_rate=rate)
    outs = [s.push(wav), s.flush()]
    torch.cuda.synchronize()
    return _cat(outs)


def _assert_job_equals_stream(model, job, wav, prompt, seed, window_seconds, rate=None):
    assert job.done and job.windows_solved == job.windows_total
    out = job.result()
    ref_t, ref_r = _stream_whole(model, wav, prompt, seed, window_seconds, rate)
    assert out.target.shape == ref_t.shape and out.residual.shape == ref_r.shape
    assert torch.equal(out.target, ref_t) and torch.equal(out.residual, ref_r)


@pytest.mark.parametrize("which", ["tiny", "small"])
@pytest.mark.parametrize("seconds,window_seconds,rate,channels", [(75, 10.0, None, 1), (20, 2.0, None, 1),
                                                                   (20, 2.0, 16000, 2)],
                         ids=["75s-W250", "20s-W50", "16k-stereo"])
def test_job_equals_the_stream_pushed_whole(request, which, seconds, window_seconds, rate, channels):
    """A job drained in a group that has never ticked (bucket 1) returns the bits of model.stream() with the whole
    recording pushed once and flushed: 75 s mono at W = 250, 20 s at W = 50, 16 kHz stereo."""
    model = request.getfixturevalue("tiny_model" if which == "tiny" else "small_model")
    wav = _recording(seconds, 3, rate or SR, channels)
    g = model.stream_group(window_seconds=window_seconds)
    job = g.submit(wav, PROMPTS[1], seed=5, sample_rate=rate)
    with pytest.raises(RuntimeError, match="not done"):
        job.result()
    g.drain()
    g.close()
    _assert_job_equals_stream(model, job, wav, PROMPTS[1], 5, window_seconds, rate)


def _run_group(model, plan, ticks, window_seconds, jobs=(), drain_at=None):
    """plan: per live stream (prompt, seed, recording, open tick, close tick or None, chunk sizes cycled, skip period);
    jobs: (tick, recording, prompt, seed, rate) submitted before that tick's push.  drain_at: (tick, job index) drained
    after that tick's push.  Returns the live streams' concatenated (target, residual), the jobs, and the job windows
    solved in push ticks."""
    g = model.stream_group(window_seconds=window_seconds)
    state = [dict(s=None, pos=0, n=0, outs=[]) for _ in plan]
    submitted = []
    for t in range(ticks):
        for st, (prompt, seed, wav, t_open, _, _, _) in zip(state, plan):
            if t == t_open:
                st["s"] = g.open(prompt, seed=seed)
        for t_job, wav, prompt, seed, rate in jobs:
            if t == t_job:
                submitted.append(g.submit(wav, prompt, seed=seed, sample_rate=rate))
        push = {}
        for st, (_, _, wav, _, _, sizes, skip) in zip(state, plan):
            s = st["s"]
            if s is None or s.closed or st["pos"] >= wav.numel() or (skip and t % skip == 0):
                continue
            n = sizes[st["n"] % len(sizes)]
            push[s] = wav[st["pos"]:st["pos"] + n]
            st["pos"] += push[s].numel()
            st["n"] += 1
        if push:
            outs = g.push(push)
            for st in state:
                if st["s"] in outs:
                    st["outs"].append(outs[st["s"]])
        for st, (_, _, _, _, t_close, _, _) in zip(state, plan):
            if t_close == t and st["s"] is not None and not st["s"].closed:
                st["outs"].append(st["s"].flush())
        if drain_at is not None and drain_at[0] == t:
            in_push_ticks = [j.windows_solved for j in submitted]
            g.drain([submitted[drain_at[1]]])
    tails = g.close()
    for st in state:
        if st["s"] in tails:
            st["outs"].append(tails[st["s"]])
    torch.cuda.synchronize()
    return [_cat(st["outs"]) for st in state], submitted, (in_push_ticks if drain_at else None)


@pytest.mark.parametrize("which", ["tiny", "small"])
def test_live_streams_do_not_notice_jobs(request, which):
    """Five live streams (different prompts, seeds, starts and chunkings, one joining late, one leaving early) and two
    jobs submitted at different ticks: every live stream is bit-identical to the same ticks without jobs, the jobs
    take filler slots of the push ticks, and they finish (one through drain(), one through close()) with the bits of
    model.stream() pushed whole."""
    model = request.getfixturevalue("tiny_model" if which == "tiny" else "small_model")
    ws = 2.0
    h = 84480                      # 1.76 s: the hop of W = 50, so streams pushed this much solve one window per tick
    plan = [
        (PROMPTS[0], 0, _recording(24, 1), 0, None, [h], 0),
        (PROMPTS[1], 7, _recording(20, 2), 1, None, [SR // 2 + 1, 1, 3 * SR - 7], 0),
        (PROMPTS[2], 3, _recording(22, 3), 0, 13, [h, h + 1921], 0),          # closes early
        (PROMPTS[3], 11, _recording(14, 4), 6, None, [h + 5], 0),            # opens mid-way
        (PROMPTS[4], 5, _recording(24, 5), 0, None, [4801, h, 2 * h, 1], 0),
    ]
    jobs = [(1, _recording(20, 30), PROMPTS[3], 9, None),
            (5, _recording(11, 31, 16000, 2), PROMPTS[2], 4, 16000)]
    without, _, _ = _run_group(model, plan, 20, ws)
    with_jobs, submitted, in_push_ticks = _run_group(model, plan, 20, ws, jobs, drain_at=(8, 0))
    for (t1, r1), (t2, r2), p in zip(without, with_jobs, plan):
        assert t1.numel() > 0 and torch.equal(t1, t2) and torch.equal(r1, r2), p[0]
    assert sum(in_push_ticks) > 0, in_push_ticks                              # jobs ran in filler slots
    for job, (_, wav, prompt, seed, rate) in zip(submitted, jobs):
        _assert_job_equals_stream(model, job, wav, prompt, seed, ws, rate)


def _record_calls(eng, monkeypatch, log):
    """Wrap the engine's planned calls to log (call, items)."""
    for name, items in (("encode", lambda a: a[0].shape[0]), ("prepare", lambda a: a[0]),
                        ("solve", lambda a: a[0].shape[0]), ("decode", lambda a: a[1])):
        fn = getattr(eng, name)

        def wrapped(*a, _fn=fn, _name=name, _items=items, **k):
            log.append((_name, int(_items(a))))
            return _fn(*a, **k)
        monkeypatch.setattr(eng, name, wrapped)


def test_steady_ticks_with_jobs_plan_nothing_and_keep_item_counts(tiny_model, monkeypatch):
    """Five staggered live streams pushed 1 s per tick at W = 50 (as in test_gpu_stream_group), once without and once
    with a long job queued before the warm-up ends.  Over 25 steady ticks with the job progressing: no DiT plan build,
    no graph capture, no codec plan build, a constant workspace, and the same planned calls with the same item counts
    as without the job."""
    eng = tiny_model._ensure_engine()
    wavs = [_recording(130, 40 + i) for i in range(5)]
    job_wav = _recording(300, 50)

    def run(with_job):
        log = []
        with tiny_model.stream_group(window_seconds=2.0) as g:
            streams = [g.open(PROMPTS[i], seed=i) for i in range(5)]
            pos = [int(i * 0.35 * SR) for i in range(5)]
            for s, w, p in zip(streams, wavs, pos):
                if p:
                    s.push(w[:p])
            job = None

            def tick():
                g.push({s: wavs[i][pos[i]:pos[i] + SR] for i, s in enumerate(streams)})
                for i in range(5):
                    pos[i] += SR
            for t in range(100):
                if with_job and t == 80:
                    job = g.submit(job_wav, PROMPTS[0], seed=3)
                tick()
            torch.cuda.synchronize()
            stats, ws = eng.plan_stats(), eng.workspace_bytes()
            solved0 = job.windows_solved if job else 0
            with monkeypatch.context() as mp:
                _record_calls(eng, mp, log)
                for _ in range(25):
                    tick()
                    assert eng.workspace_bytes() == ws
            torch.cuda.synchronize()
            after = eng.plan_stats()
            for k in ("dit_plan_builds", "graph_captures", "codec_plan_builds"):
                assert after[k] == stats[k], (k, stats, after)
            progressed = (job.windows_solved - solved0) if job else 0
            if job:
                assert not job.done
                job.cancel()
        return log, progressed

    base, _ = run(False)
    with_job, progressed = run(True)
    assert progressed > 0
    assert with_job == base


def test_cancel_frees_the_job_memory(tiny_model):
    """A job that has progressed through push ticks and is then cancelled leaves the allocator where it was before it was
    submitted, once the live streams have ended too.  Three live streams in lockstep make three windows ready per tick
    at W = 50, a bucket of 4 with one filler slot per call for the job."""
    g = tiny_model.stream_group(window_seconds=2.0)
    live = [g.open(PROMPTS[i], seed=i) for i in range(3)]
    wavs = [_recording(12, 70 + i) for i in range(3)]
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    job = g.submit(_recording(30, 75), PROMPTS[1], seed=1)
    for t in range(10):
        g.push({s: w[t * SR:(t + 1) * SR] for s, w in zip(live, wavs)})
    assert job.windows_solved > 0 and not job.done
    job.cancel()
    g.flush(live)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before
    with pytest.raises(RuntimeError, match="cancelled"):
        job.result()
    g.close()


def test_submit_copies_the_recording(tiny_model):
    """A 48 kHz mono recording whose length is a multiple of the hop (20 s) is read by the job's tiles over later ticks;
    submit() copies it, so a caller that reuses its buffer for the next recording right away leaves the job unchanged."""
    g = tiny_model.stream_group(window_seconds=2.0)
    wav = _recording(20, 80)
    assert wav.numel() % tiny_model.cfg.audio_codec.hop_length == 0
    buf = wav.clone()
    job = g.submit(buf, PROMPTS[0], seed=2)
    buf.copy_(_recording(20, 81))                         # the next recording arrives in the same buffer
    g.drain()
    g.close()
    _assert_job_equals_stream(tiny_model, job, wav, PROMPTS[0], 2, 2.0)
