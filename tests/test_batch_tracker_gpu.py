"""Several sequences per GPU in lock-step (pytracking_b200/batch.py, b200trk_dimp_batch_*), on the GPU:
  * capacity 1 reproduces the solo DiMPTracker bit for bit (boxes, flags, score maps, filters), DiMP-50 and PrDiMP-50;
  * a sequence's bits do not depend on its batch-mates, its slot or when they started (capacity 4, a mate released and replaced);
  * against solo trackers: filter-synchronised scores within 1e-4 relative with the same arg-max cell, closed-loop boxes within
    0.5 px (stock schedule), mean IoU within 0.01 (bench schedule);
  * track_sequences keeps the slots busy and every sequence equals it tracked alone at the same capacity;
  * run-to-run determinism, one forward / classify / localisation per step, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# bench.py's TRACKER_PARAMS (the bench schedule: 10 iterations every frame)
BENCH = dict(image_sample_size=288, search_area_scale=5, sample_memory_size=50, learning_rate=0.01, init_samples_minimum_weight=0.25,
             train_skipping=1, update_classifier=True, net_opt_iter=10, net_opt_update_iter=10, net_opt_hn_iter=1, advanced_localization=True,
             target_not_found_threshold=-1e9, distractor_threshold=0.8, hard_negative_threshold=0.5, target_neighborhood_scale=2.2,
             dispalcement_scale=0.8, hard_negative_learning_rate=0.02, augmentation_expansion_factor=2, use_iou_net=False)
STOCK = dict(BENCH, train_skipping=20, net_opt_update_iter=2)
PRDIMP = dict(BENCH, image_sample_size=352, search_area_scale=6, border_mode="inside_major", patch_max_scale_change=1.5,
              score_preprocess="softmax")


def _sd():
    from pytracking_b200 import synth
    return synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)


def _seq(q, n):
    from pytracking_b200 import synth
    frames, bb = synth.make_sequence(q, num_frames=n)
    return frames, bb


def _batch(capacity, cfg=BENCH, newton=None):
    from pytracking_b200.batch import DiMPBatchTracker
    from pytracking_b200.tracker import make_params
    return DiMPBatchTracker(_sd(), make_params(**cfg), capacity, newton=newton)


def _solo(cfg=BENCH, newton=None):
    from pytracking_b200.tracker import DiMPTracker, make_params
    return DiMPTracker(_sd(), make_params(**cfg), newton=newton)


def _bits(t):
    return t.detach().float().cpu().numpy().view(np.uint32).copy()


def _run_solo(cfg, newton, frames, bb):
    trk = _solo(cfg, newton)
    trk.initialize(frames[0], {"init_bbox": bb})
    rec = [(list(bb), 0, None, _bits(trk.engine.filter))]
    for f in frames[1:]:
        box = trk.track(f)["target_bbox"]
        rec.append((box, int(trk.info.flag), _bits(trk.engine.scores[0]), _bits(trk.engine.filter)))
    trk.close()
    return rec


@pytest.mark.parametrize("kind", ["dimp", "prdimp"])
def test_capacity_one_equals_solo_tracker_bitwise(kind):
    cfg, newton = (BENCH, None) if kind == "dimp" else (PRDIMP, {})
    frames, bb = _seq(0, 60)
    solo = _run_solo(cfg, newton, frames, bb)
    bt = _batch(1, cfg, newton)
    out = bt.step({0: (frames[0], {"init_bbox": bb})})
    assert out[0]["target_bbox"] == [float(np.float32(v)) for v in bb]
    assert np.array_equal(_bits(bt.filter(0)), solo[0][3])
    for t in range(1, len(frames)):
        out = bt.step({0: (frames[t], None)})
        box, flag, scores, filt = solo[t]
        assert out[0]["target_bbox"] == box, (kind, t)
        assert int(bt.last_info[0].flag) == flag, (kind, t)
        assert np.array_equal(_bits(bt.scores(0)), scores), (kind, t)
        assert np.array_equal(_bits(bt.filter(0)), filt), (kind, t)
    bt.close()


def _mates_run(layout, n_frames, release_at, replacement, cfg=BENCH, newton=None):
    """layout: {slot: (sequence, first step)}; at step release_at the slot of the mate `replacement[0]` gets sequence replacement[1].
    Returns per slot the list of (box, score bits, filter bits) of every frame of its first sequence (capacity 4, configuration
    cfg / newton as for _batch)."""
    bt = _batch(4, cfg, newton)
    seqs = {slot: _seq(q, n_frames) for slot, (q, _) in layout.items()}
    pos = {slot: 0 for slot in layout}
    rec = {slot: [] for slot in layout}
    total = max(s0 for _, s0 in layout.values()) + n_frames + 1
    for step in range(total):
        if step == release_at:
            slot, q = replacement
            bt.release(slot)
            seqs[slot] = _seq(q, n_frames)
            pos[slot] = 0
            layout = {**layout, slot: (q, step)}
            rec[slot] = None                                   # the replaced mate is not compared
        batch = {}
        for slot, (q, s0) in layout.items():
            frames, bb = seqs[slot]
            if step >= s0 and pos[slot] < len(frames):
                batch[slot] = (frames[pos[slot]], {"init_bbox": bb} if pos[slot] == 0 else None)
                pos[slot] += 1
        if not batch:
            continue
        out = bt.step(batch)
        for slot in out:
            if rec[slot] is not None:
                rec[slot].append((out[slot]["target_bbox"], _bits(bt.scores(slot)), _bits(bt.filter(slot))))
    bt.close()
    return rec


def check_batch_mates_do_not_change_a_sequence(cfg=BENCH, newton=None):
    n = 40
    a = _mates_run({0: (0, 0), 1: (1, 0), 2: (2, 0), 3: (3, 0)}, n, release_at=20, replacement=(2, 7), cfg=cfg, newton=newton)
    b = _mates_run({3: (0, 2), 0: (4, 0), 1: (5, 0), 2: (6, 0)}, n, release_at=25, replacement=(1, 8), cfg=cfg, newton=newton)
    qa, qb = a[0], b[3]
    assert len(qa) == len(qb) == n + 1
    for t in range(1, n + 1):                                  # frame 0 is the init step (its scores belong to no filter of the sequence)
        assert qa[t][0] == qb[t][0], t
        assert np.array_equal(qa[t][1], qb[t][1]), t
        assert np.array_equal(qa[t][2], qb[t][2]), t
    assert np.array_equal(qa[0][2], qb[0][2])


def test_batch_mates_do_not_change_a_sequence():
    check_batch_mates_do_not_change_a_sequence()


def test_run_to_run_determinism():
    layout = {0: (0, 0), 1: (1, 0), 2: (2, 1), 3: (3, 3)}
    a = _mates_run(layout, 25, release_at=10, replacement=(1, 9))
    b = _mates_run(layout, 25, release_at=10, replacement=(1, 9))
    for slot in (0, 2, 3):
        for x, y in zip(a[slot], b[slot]):
            assert x[0] == y[0] and np.array_equal(x[1], y[1]) and np.array_equal(x[2], y[2])


def test_scores_match_solo_with_synchronised_filters():
    """Each slot's scores at capacity 4 against a solo engine (forward at batch 1) given the same crop and the same filter."""
    bt = _batch(4, STOCK)
    solo = _solo(STOCK)
    eng = solo.engine
    seqs = [_seq(q, 20) for q in range(4)]
    bt.step({s: (seqs[s][0][0], {"init_bbox": seqs[s][1]}) for s in range(4)})
    worst = 0.0
    for t in range(1, 21):
        before = [bt.filter(s).clone() for s in range(4)]
        bt.step({s: (seqs[s][0][t], None) for s in range(4)})
        for s in range(4):
            eng.filter.copy_(before[s])
            eng.localize_device(bt.crop(s)[None].contiguous())
            ref, mine = eng.scores[0].float().cpu(), bt.scores(s).float().cpu()
            err = float((mine - ref).abs().max() / ref.abs().max())
            worst = max(worst, err)
            assert err <= 1e-4, (t, s, err)
            assert int(mine.argmax()) == int(ref.argmax()), (t, s)
    solo.close()
    bt.close()
    print("worst relative score difference batch(4) vs solo: %.3g" % worst)


def _closed_loop(cfg, n, newton=None):
    from pytracking_b200 import shard, synth
    seqs = [_seq(q, n) for q in range(4)]
    bt = _batch(4, cfg, newton)
    boxes_b = {s: [] for s in range(4)}
    bt.step({s: (seqs[s][0][0], {"init_bbox": seqs[s][1]}) for s in range(4)})
    for t in range(1, n + 1):
        out = bt.step({s: (seqs[s][0][t], None) for s in range(4)})
        for s in range(4):
            boxes_b[s].append(out[s]["target_bbox"])
    bt.close()
    boxes_s = {}
    for s in range(4):
        trk = _solo(cfg, newton)
        trk.initialize(seqs[s][0][0], {"init_bbox": seqs[s][1]})
        boxes_s[s] = [trk.track(f)["target_bbox"] for f in seqs[s][0][1:]]
        trk.close()
    iou = {}
    for s in range(4):
        gt = torch.tensor(synth.sequence_ground_truth(s, n)[1:], dtype=torch.float32)
        iou[s] = (float(shard.iou_overlap(torch.tensor(boxes_b[s]), gt).mean()), float(shard.iou_overlap(torch.tensor(boxes_s[s]), gt).mean()))
    return boxes_b, boxes_s, iou


def check_closed_loop_within_half_a_pixel_of_solo(cfg=STOCK, newton=None):
    boxes_b, boxes_s, _ = _closed_loop(cfg, 100, newton)
    worst = 0.0
    for s in range(4):
        d = np.abs(np.array(boxes_b[s]) - np.array(boxes_s[s])).max()
        worst = max(worst, float(d))
        assert d <= 0.5, (s, d)
    return worst


def test_closed_loop_stock_schedule_within_half_a_pixel_of_solo():
    check_closed_loop_within_half_a_pixel_of_solo()


def test_bench_schedule_iou_matches_solo():
    _, _, iou = _closed_loop(BENCH, 100)
    for s, (b, so) in iou.items():
        assert abs(b - so) <= 0.01, (s, b, so)


def test_track_sequences_equals_each_sequence_alone():
    from pytracking_b200.batch import track_sequences
    lengths = [12, 25, 7, 18, 30, 9, 15]
    seqs = [_seq(q, n) for q, n in enumerate(lengths)]
    bt = _batch(3)
    res = track_sequences(bt, [(frames, bb) for frames, bb in seqs])
    assert [len(r["target_bbox"]) for r in res] == [n + 1 for n in lengths]
    assert all(len(r["time"]) == len(r["target_bbox"]) for r in res)
    for q, (frames, bb) in enumerate(seqs):
        alone = track_sequences(bt, [(frames, bb)])[0]
        assert alone["target_bbox"] == res[q]["target_bbox"], q
    bt.close()


def test_steady_step_runs_one_forward_classify_and_localisation():
    """Capacity 4 with one busy slot launches exactly what one solo frame launches: one crop, one forward (the cached graph: the same
    pointers and batch size every step), one classify, one localisation and the slot's optimiser."""
    from pytracking_b200 import _lib
    L = _lib.lib()
    frames, bb = _seq(0, 12)
    solo = _solo()
    solo.initialize(frames[0], {"init_bbox": bb})
    bt = _batch(4)
    bt.step({0: (frames[0], {"init_bbox": bb})})
    ds, db = [], []
    for t in range(1, 12):
        c0 = L.b200trk_launch_count(); solo.track(frames[t]); c1 = L.b200trk_launch_count()
        bt.step({0: (frames[t], None)}); c2 = L.b200trk_launch_count()
        ds.append(c1 - c0); db.append(c2 - c1)
    assert ds[-5:] == db[-5:], (ds, db)
    assert len(set(db[-5:])) == 1, db
    solo.close()
    bt.close()


def test_refusals():
    from pytracking_b200 import _lib
    from pytracking_b200.batch import DiMPBatchTracker
    from pytracking_b200.tracker import make_params
    with pytest.raises(RuntimeError, match="use_iou_net"):
        DiMPBatchTracker(_sd(), make_params(**dict(BENCH, use_iou_net=True)), 2)
    for cap in (0, 17):
        with pytest.raises(RuntimeError, match="capacity"):
            DiMPBatchTracker(_sd(), make_params(**BENCH), cap)
    bt = _batch(2)
    frames, bb = _seq(0, 3)
    with pytest.raises(RuntimeError, match="not tracking a sequence"):
        bt.step({0: (frames[0], None)})                                    # never initialised
    bt.step({0: (frames[0], {"init_bbox": bb})})
    with pytest.raises(RuntimeError, match="frame is 240x320"):
        bt.step({0: (np.ascontiguousarray(frames[1][:240, :320]), None)})  # frame size changes mid-sequence
    with pytest.raises(RuntimeError, match="slot 2 outside"):
        bt.step({2: (frames[1], None)})
    items = (_lib.BatchItem * 2)()
    keep = [np.ascontiguousarray(frames[1]) for _ in range(2)]
    for k in range(2):
        items[k].slot, items[k].image, items[k].H, items[k].W, items[k].init = 0, keep[k].ctypes.data, 480, 640, 0
    infos = (_lib.FrameInfo * 2)()
    with pytest.raises(RuntimeError, match="appears twice"):
        _lib.check(_lib.lib().b200trk_dimp_batch_step_host(bt.handle, items, 2, infos, C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                   "dimp_batch_step")
    bt.step({0: (frames[1], None)})                                        # nothing was changed by the refused steps
    bt.release(0)
    with pytest.raises(RuntimeError, match="not tracking a sequence"):
        bt.step({0: (frames[2], None)})                                    # released
    bt.close()
