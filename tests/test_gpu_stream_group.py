"""GPU (H100) tests of stream groups (SAMAudio.stream_group, sam_audio_b200/stream.py): each stream's output is
bit-identical to the same stream run alone through SAMAudio.stream(), filler items change no bit, steady ticks plan
nothing, and the default plan residency is unchanged outside groups."""
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


def _recording(seconds, seed):
    from sam_audio_b200.synthetic import synthetic_clip
    return synthetic_clip(seed, int(SR * seconds)).reshape(-1).cuda()


def _cat(outs):
    return torch.cat([o.target for o in outs]), torch.cat([o.residual for o in outs])


def _alone(model, prompt, seed, chunks, window_seconds):
    s = model.stream(prompt, window_seconds=window_seconds, seed=seed)
    outs = [s.push(c) for c in chunks] + [s.flush()]
    torch.cuda.synchronize()
    return _cat(outs)


def _run_group(model, plan, ticks, window_seconds):
    """plan: per stream (prompt, seed, recording, open tick, close tick or None, chunk sizes cycled, skip period).
    Returns, per stream, its chunks in push order and its concatenated (target, residual)."""
    g = model.stream_group(window_seconds=window_seconds)
    state = [dict(s=None, pos=0, chunks=[], outs=[]) for _ in plan]
    for t in range(ticks):
        for st, (prompt, seed, wav, t_open, _, _, _) in zip(state, plan):
            if t == t_open:
                st["s"] = g.open(prompt, seed=seed)
        push = {}
        for i, (st, (_, _, wav, t_open, t_close, sizes, skip)) in enumerate(zip(state, plan)):
            s = st["s"]
            if s is None or s.closed or st["pos"] >= wav.numel() or (skip and t % skip == 0):
                continue
            n = sizes[len(st["chunks"]) % len(sizes)]
            c = wav[st["pos"]:st["pos"] + n]
            st["pos"] += c.numel()
            st["chunks"].append(c)
            push[s] = c
        if push:
            outs = g.push(push)
            for st in state:
                if st["s"] in outs:
                    st["outs"].append(outs[st["s"]])
        for st, (_, _, _, _, t_close, _, _) in zip(state, plan):
            if t_close == t and st["s"] is not None and not st["s"].closed:
                st["outs"].append(st["s"].flush())               # one stream leaves on its own
    tails = g.close()
    for st in state:
        if st["s"] in tails:
            st["outs"].append(tails[st["s"]])
    torch.cuda.synchronize()
    return [(st["chunks"], _cat(st["outs"])) for st in state]


@pytest.mark.parametrize("which,group_windows", [("tiny", None), ("small", None), ("tiny", 3)])
def test_each_stream_equals_the_stream_alone(request, monkeypatch, which, group_windows):
    """Five streams with different prompts (<= 8 tokens), seeds, start ticks and chunkings, one opening mid-way and one
    closing early, ticks that push a subset: every stream's output equals model.stream() on the same pushes, bit for
    bit.  With grouped solves of three windows (SAB_WINDOW_ROWS), ticks are split into several solves, and a stream's
    windows straddle two of them next to other streams' windows."""
    model = request.getfixturevalue("tiny_model" if which == "tiny" else "small_model")
    if group_windows:
        monkeypatch.setenv("SAB_WINDOW_ROWS", str(group_windows * 50))
    ws = 2.0
    plan = [
        (PROMPTS[0], 0, _recording(14, 1), 0, None, [SR], 0),
        (PROMPTS[1], 7, _recording(12, 2), 1, None, [SR // 2 + 1, 1, 3 * SR - 7], 0),
        (PROMPTS[2], 3, _recording(13, 3), 2, 9, [SR, 1921], 4),              # closes early
        (PROMPTS[3], 11, _recording(9, 4), 6, None, [2 * SR + 5], 0),          # opens mid-way
        (PROMPTS[4], 5, _recording(15, 5), 0, None, [4801, SR, 96_001, 1], 3),
    ]
    got = _run_group(model, plan, 18, ws)
    for (prompt, seed, *_), (chunks, (tgt, res)) in zip(plan, got):
        assert chunks and tgt.numel() == res.numel() > 0
        ref_t, ref_r = _alone(model, prompt, seed, chunks, ws)
        assert torch.equal(tgt, ref_t) and torch.equal(res, ref_r), prompt


def test_filler_items_change_no_bit(tiny_model, monkeypatch):
    """Three streams in lockstep make three windows ready per tick: a bucket of 4 with one filler item.  With the group
    size set to three windows (SAB_WINDOW_ROWS), the same windows are solved with no filler: the same bits."""
    from sam_audio_b200.windows import stream_bucket, stream_group_capacity, window_rows_budget
    W = 50
    assert len(stream_bucket(3, stream_group_capacity(W, window_rows_budget()))) == 4
    plan = [(PROMPTS[i], i, _recording(8, 20 + i), 0, None, [SR], 0) for i in range(3)]
    with_filler = _run_group(tiny_model, plan, 9, 2.0)
    monkeypatch.setenv("SAB_WINDOW_ROWS", str(3 * W))
    assert len(stream_bucket(3, stream_group_capacity(W, window_rows_budget()))) == 3
    without = _run_group(tiny_model, plan, 9, 2.0)
    for (_, (t1, r1)), (_, (t2, r2)) in zip(with_filler, without):
        assert torch.equal(t1, t2) and torch.equal(r1, r2)


def test_steady_ticks_plan_nothing(tiny_model):
    """Five streams with staggered starts pushed 1 s per tick at W = 50 (H = 44 frames, so the windows per tick vary and
    repeat every 44 ticks).  After a warm-up of two such periods, in which every bucket the later ticks use has been
    solved at least twice (the second solve of a plan captures its graph), 25 further ticks build no DiT plan, capture
    no graph and build no codec plan, and the engine's workspace stays the same."""
    eng = tiny_model._ensure_engine()
    wavs = [_recording(130, 40 + i) for i in range(5)]
    with tiny_model.stream_group(window_seconds=2.0) as g:
        streams = [g.open(PROMPTS[i], seed=i) for i in range(5)]
        pos = [int(i * 0.35 * SR) for i in range(5)]
        for s, w, p in zip(streams, wavs, pos):
            if p:
                s.push(w[:p])

        def tick():
            out = {}
            before = [s.windows_solved for s in streams]
            for i, s in enumerate(streams):
                out[s] = wavs[i][pos[i]:pos[i] + SR]
                pos[i] += SR
            g.push(out)
            return sum(s.windows_solved - b for s, b in zip(streams, before))

        for _ in range(100):
            tick()
        torch.cuda.synchronize()
        stats, ws = eng.plan_stats(), eng.workspace_bytes()
        counts = []
        for _ in range(25):
            counts.append(tick())
            assert eng.workspace_bytes() == ws
        torch.cuda.synchronize()
        after = eng.plan_stats()
        assert len(set(counts)) > 1, counts
        for k in ("dit_plan_builds", "graph_captures", "codec_plan_builds"):
            assert after[k] == stats[k], (k, stats, after)
        assert after["dit_plans_resident"] > 1
        tails = g.close()                                                # flushes all five streams in one tick
    assert set(tails) == set(streams) and all(t.target.numel() > 0 for t in tails.values())
    end = eng.plan_stats()
    assert end["dit_plan_builds"] == after["dit_plan_builds"]            # the flush reused the resident buckets
    assert end["dit_plans_resident"] == 1                                # close() gave back the default residency


def test_a_failed_flush_ends_its_streams_and_close_restores_residency(tiny_model, monkeypatch):
    """A flush whose tick raises still ends its streams and leaves the group consistent: close() flushes the rest and
    gives the engine back its default residency."""
    from sam_audio_b200.stream import StreamGroup
    eng = tiny_model._ensure_engine()
    g = tiny_model.stream_group(window_seconds=2.0)
    a, b, c = (g.open(PROMPTS[i], seed=i) for i in range(3))
    g.push({a: _recording(4, 60), b: _recording(3, 61), c: _recording(4, 62)})   # 5 windows: bucket 8
    g.push({a: _recording(2, 63)})                                                # 1 window: bucket 1
    assert eng.plan_stats()["dit_plans_resident"] > 1

    def fail(self, due, flushed):
        raise RuntimeError("tick failed")
    with monkeypatch.context() as mp:
        mp.setattr(StreamGroup, "_tick", fail)
        with pytest.raises(RuntimeError, match="tick failed"):
            g.flush([a, b])
    assert a.closed and b.closed and g.streams == [c]
    with pytest.raises(RuntimeError, match="closed"):
        a.push(_recording(1, 66))
    tails = g.close()
    assert set(tails) == {c} and tails[c].target.numel() > 0
    torch.cuda.synchronize()
    assert eng.plan_stats()["dit_plans_resident"] == 1


def test_a_dropped_group_gives_back_the_residency(tiny_model):
    """A group that is dropped without close() restores the default residency when it is collected."""
    import gc
    eng = tiny_model._ensure_engine()
    g = tiny_model.stream_group(window_seconds=2.0)
    streams = [g.open(PROMPTS[i], seed=i) for i in range(3)]
    g.push({s: _recording(3 + i, 70 + i) for i, s in enumerate(streams)})        # 5 windows: bucket 8
    g.push({streams[0]: _recording(2, 80)})                                       # 1 window: bucket 1
    assert eng.plan_stats()["dit_plans_resident"] > 1
    del g, streams
    gc.collect()
    torch.cuda.synchronize()
    assert eng.plan_stats()["dit_plans_resident"] == 1


def test_default_limits_keep_one_dit_plan(tiny_model):
    """Outside a group the engine keeps today's residency: separate() of two shapes and a stream that solves one and
    then several windows per push leave one DiT plan and at most three codec plans per direction."""
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_descriptions
    eng = tiny_model._ensure_engine()
    cc = tiny_model.cfg.audio_codec
    proc = SAMAudioProcessor(cc.hop_length, cc.sample_rate)
    for lens in ([9600, 5000], [20000]):
        batch = proc(descriptions=synthetic_descriptions(len(lens)),
                     audios=[synthetic_clip(i, n) for i, n in enumerate(lens)]).to("cuda:0")
        tiny_model.separate(batch)
        assert eng.plan_stats()["dit_plans_resident"] == 1
    wav = _recording(30, 9)
    s = tiny_model.stream(PROMPTS[0], window_seconds=2.0)
    s.push(wav[:SR * 3])
    s.push(wav[SR * 3:SR * 20])                                            # several windows in one push
    s.flush()
    torch.cuda.synchronize()
    st = eng.plan_stats()
    assert st["dit_plans_resident"] == 1 and st["codec_plans_resident"] <= 6
