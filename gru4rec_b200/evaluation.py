"""evaluate_gpu with the reference's signature and return value (hidasib/GRU4Rec evaluation.py:15-147)."""
import os

import numpy as np
import pandas as pd

from . import _lib
from .baselines import Baseline

_MODES = {'standard': 0, 'conservative': 1, 'median': 2, 'tiebreaking': 3}


def _prepare(gru, test_data, session_key, item_key, time_key):
    """evaluate_gpu's test data (evaluation.py:84-89): merged with the item map (unknown items dropped) and sorted by session,
    time and item; returns (frame, item indices, session offsets)"""
    test_data = pd.merge(test_data, pd.DataFrame({'ItemIdx': gru.itemidmap.values, item_key: gru.itemidmap.index}), on=item_key, how='inner')
    test_data.sort_values([session_key, time_key, item_key], inplace=True)
    offset_sessions = np.zeros(test_data[session_key].nunique() + 1, dtype=np.int32)
    offset_sessions[1:] = test_data.groupby(session_key).size().cumsum()
    return test_data, test_data.ItemIdx.values, offset_sessions


def _prepare_history(gru, test_data, history, session_key, item_key, time_key):
    """the test data prepared by _prepare; with a history frame (prepared by the same rules, restricted to the test sessions),
    each test session becomes its history rows followed by its test rows, whatever their times.  Returns (frame, item indices,
    session offsets, n_history): n_history (per session, its leading history events) is None when no history row is left, and
    the evaluation is then exactly the plain one"""
    test_data, items, offs = _prepare(gru, test_data, session_key, item_key, time_key)
    if history is None or len(history) == 0:
        return test_data, items, offs, None
    hist = _prepare(gru, history, session_key, item_key, time_key)[0]
    hist = hist[hist[session_key].isin(pd.unique(test_data[session_key]))]
    if len(hist) == 0:
        return test_data, items, offs, None
    sids = test_data[session_key].values[offs[:-1]]
    n_hist = hist.groupby(session_key).size().reindex(sids, fill_value=0).values.astype(np.int32)
    both = pd.concat([hist.assign(_g4r_part=0), test_data.assign(_g4r_part=1)], ignore_index=True)
    both = both.sort_values([session_key, '_g4r_part'], kind='stable').drop(columns='_g4r_part')
    offs = np.zeros(len(sids) + 1, dtype=np.int32)
    offs[1:] = both.groupby(session_key).size().reindex(sids).values.cumsum()
    return both, both.ItemIdx.values, offs, n_hist


class _ExcludeSeen(object):
    """exclude_seen on the engine for the duration of one evaluation (reset whatever happens, like the candidate items).  The
    library refuses seen lists over its budget (lanes x (longest session - 1) int32); the same test on the whole test set is made
    here first, so that every rank of a torch.distributed job refuses together (a rank's shard never needs more) with a
    ValueError that names the longest session"""

    def __init__(self, eng, on, test_data, session_key, offset_sessions, lanes):
        self.eng, self.on = eng, on
        if on:
            lens = np.diff(offset_sessions)
            j = int(np.argmax(lens)) if len(lens) else 0
            need = int(lanes) * max(1, int(lens[j]) - 1 if len(lens) else 1) * 4
            if need > _lib.seen_budget():
                sid = test_data[session_key].values[offset_sessions[j]]
                sid = sid.item() if isinstance(sid, np.generic) else sid
                raise ValueError('exclude_seen: session %r has %d events; its seen lists for %d lanes take %d bytes, over the %d-byte '
                                 'budget' % (sid, int(lens[j]), int(lanes), need, _lib.seen_budget()))

    def __enter__(self):
        if self.on:
            self.eng.set_eval_exclude_seen(True)
        return self

    def __exit__(self, typ, err, tb):
        if self.on:
            self.eng.set_eval_exclude_seen(False)
        return False


def _cuts(cut_off):
    multi_cut_off = (type(cut_off) == list) or (type(cut_off) == tuple)
    return list(cut_off) if multi_cut_off else [cut_off]


def evaluate_gpu(gru, test_data, items=None, session_key='SessionId', item_key='ItemId', time_key='Time', cut_off=[20], batch_size=100, mode='standard',
                 exclude_seen=False, history=None):
    '''
    Recall@N and MRR@N of next-item prediction, session-parallel (evaluation.py:15-147).
    Returns (recall_list, mrr_list), one entry per cut-off.  `mode` as in the reference; 'tiebreaking' adds U(0,1)*1e-10 to
    every score before the standard ranking (evaluation.py:55,65) -- it only matters where scores saturate at (near) zero; the
    noise is a counter hash on the device (the reference's comes from Theano's MRG stream).  `items`: the targets are ranked against these item ids only (evaluation.py:52-56,84-100); as in the
    reference the target's own score competes only if the target is listed, so 'conservative' can give rank 0 (MRR = inf).
    Under a torch.distributed job (torchrun, one process per GPU) every rank calls this with the same test data and scores
    every world-th session; all ranks return the same (summed) result.  G4R_EVAL_SHARD=0 switches the sharding off.
    `exclude_seen` (an addition to the reference's signature): evaluate what recommend_next_batch(exclude_seen=True) serves.
    Each event is ranked without the items its session has input so far, the current input included (with `items`, every
    occurrence of such an item leaves the list); an event whose target is among them is a miss (rank inf: it adds nothing to
    Recall or MRR but still counts as an event).  The seen lists live on the device, (batch_size x longest session - 1) int32
    within 256 MiB: a longer longest session raises ValueError naming it (on every rank of a torch.distributed job).
    `history` (an addition to the reference's signature): a DataFrame with the test data's key columns, each session's events
    before its test events.  It is prepared like the test data (unknown items dropped, sorted by session, time and item) and
    only its sessions that are also in the test data are used.  The evaluation is then that of the concatenated data (every
    test session's history followed by its test events, whatever their times), counting only the events whose target is a test
    event: a session with h >= 1 history events and t test events contributes t events, the first one with the last history
    item as input and the state after the history before it; a session without history contributes t - 1 as before.  With
    exclude_seen the history's items count as seen, and the seen-list budget applies to the longest concatenated session.
    Only the counted events are ranked on the device.  history=None or an empty frame: exactly the evaluation without it.
    '''
    if isinstance(gru, Baseline):
        return _evaluate_baseline(gru, test_data, items, session_key, item_key, time_key, cut_off, mode, 0, exclude_seen, history, True)
    if gru.error_during_train: raise Exception
    if mode not in _MODES:
        raise NotImplementedError
    cuts = _cuts(cut_off)
    print('Measuring Recall@{} and MRR@{}'.format(','.join([str(c) for c in cuts]), ','.join([str(c) for c in cuts])))
    test_data, test_data_items, offset_sessions, n_hist = _prepare_history(gru, test_data, history, session_key, item_key, time_key)
    n_sessions = len(offset_sessions) - 1
    world, rank = gru._world()
    if world > 1 and os.environ.get('G4R_EVAL_SHARD', '1') == '0':
        world, rank = 1, 0                                     # every rank scores the whole test set on its own replica
    if world > 1 and n_sessions < batch_size:
        # the reference indexes offset_sessions[arange(batch_size) + 1] (evaluation.py:93-94): same error, whatever the shard sizes
        raise IndexError('index out of bounds: fewer sessions than batch_size (reference: IndexError at evaluation.py:94)')
    eng = gru._ensure_engine(batch_size)
    if items is not None:
        eng.set_eval_items(gru.itemidmap[items].values)       # KeyError for unknown ids, as the reference's gru.itemidmap[items]
    try:
        with _ExcludeSeen(eng, exclude_seen, test_data, session_key, offset_sessions, batch_size):
            if world == 1:
                sched = _lib.Schedule(test_data_items, offset_sessions, None, batch_size, 0, mode=1, n_history=n_hist)
                rec, mrr, n = eng.eval_schedule(sched, cuts, _MODES[mode])
            else:
                # one process per GPU: rank r scores every world-th session on its full replica of the model; the hit and
                # reciprocal-rank sums (double) and the event count are summed over the ranks -- no exchange on the data path
                from .parallel import shard_eval_sessions, allreduce_sum
                import torch.distributed as dist
                mine = shard_eval_sessions(n_sessions, rank, world)
                rec, mrr, n = np.zeros(len(cuts)), np.zeros(len(cuts)), 0
                if len(mine):
                    sched = _lib.Schedule(test_data_items, offset_sessions, mine, min(batch_size, len(mine)), 0, mode=1, n_history=n_hist)
                    rec, mrr, n = eng.eval_schedule(sched, cuts, _MODES[mode])
                tot = allreduce_sum(np.concatenate([rec, mrr, [float(n)]]), dist)
                rec, mrr, n = tot[:len(cuts)], tot[len(cuts):2 * len(cuts)], int(round(tot[-1]))
    finally:
        if items is not None:
            eng.set_eval_items(None)
    # the scoring hidden state is shared with predict_next_batch (gru4rec.py:696-697 keeps separate buffers): force its reset
    gru.predict = None
    recall = [float(r) / n for r in rec]
    mrrs = [float(m) / n for m in mrr]
    return recall, mrrs


def _ranks(counts, mode):
    """rank of every event from its (#greater, #equal) counts, by the formula of `mode` (evaluation.py:60-63); the counts
    (-1, -1) of an exclude_seen miss give inf"""
    gt, eq = counts[:, 0].astype(np.float64), counts[:, 1].astype(np.float64)
    if mode == 'conservative':
        r = gt + eq
    elif mode == 'median':
        r = gt + 0.5 * (eq - 1.0) + 1.0
    else:
        r = gt + 1.0
    miss = counts[:, 0] < 0
    if miss.any():
        r[miss] = np.inf
    return r


def evaluate_events(gru, test_data, items=None, session_key='SessionId', item_key='ItemId', time_key='Time', cut_off=[20], batch_size=100, mode='standard', k=0,
                    exclude_seen=False, history=None):
    '''
    evaluate_gpu with per-event outputs, from one evaluation pass on the device.  The test data is prepared, batched and ranked
    exactly as evaluate_gpu does it (same arguments, modes and `items` semantics).  Returns a dict:

    - 'events': DataFrame with one row per scored event (every event but the first of its session), in the order of the sorted
      test data: session id, time, input item id (column 'input_item'), target item id (column `item_key`) and 'rank' (float64,
      by the formula of `mode`, so 'median' gives halves).
    - 'recall', 'mrr': lists, one entry per cut-off, equal to evaluate_gpu's for the same arguments.
    - 'ndcg': NDCG@N per cut-off, mean(1 / log2(rank + 1) if rank <= N else 0) over the events.  With `items` in
      'conservative' mode a target outside the items can get rank 0 (as in evaluate_gpu, where MRR is then inf): its
      1 / log2(1) makes NDCG inf too.
    - k > 0: 'topk_items' [n_events, k] (original item ids, best first), 'topk_scores' [n_events, k] float32 and 'coverage'
      (distinct recommended items / n_items): the list recommend_next_batch would return for the event's session after its input
      (ranking key, the smaller item index first on equal keys, predict_next_batch's scores; with `items`, only those items
      compete and the softmax normaliser runs over them).  The lists do not tie-break like 'rank' does: the rank of a target
      that ties other items depends on `mode`, its place in the list on the item index.

    `exclude_seen` as in evaluate_gpu: every rank, sum and list leaves out the items the session has input so far, the current
    input included.  'rank' is inf exactly for the events whose target is among them (NDCG 0), and each list is what
    recommend_next_batch(..., exclude_seen=True) returns after that input; a list with fewer than k eligible items is padded
    with item None (the item array is then of object dtype) and score NaN, and 'coverage' ignores the padding.

    `history` as in evaluate_gpu: 'events' has one row per counted event, in the order of the concatenated data (sessions
    sorted, each session's history before its test events); the first row of a warm-started session has the session's last
    history item as 'input_item'.

    Single process only: under a torch.distributed job it raises NotImplementedError.
    '''
    if isinstance(gru, Baseline):
        return _evaluate_baseline(gru, test_data, items, session_key, item_key, time_key, cut_off, mode, k, exclude_seen, history, False)
    if gru.error_during_train: raise Exception
    if mode not in _MODES:
        raise NotImplementedError
    if k != 0:
        k = _lib.check_topk(k, gru.n_items if items is None else len(set(gru.itemidmap[items].values)))
    if gru._world()[0] > 1:
        raise NotImplementedError('evaluate_events runs in a single process (evaluate_gpu shards sessions over the ranks)')
    cuts = _cuts(cut_off)
    test_data, test_data_items, offset_sessions, n_hist = _prepare_history(gru, test_data, history, session_key, item_key, time_key)
    eng = gru._ensure_engine(batch_size)
    if items is not None:
        eng.set_eval_items(gru.itemidmap[items].values)
    try:
        with _ExcludeSeen(eng, exclude_seen, test_data, session_key, offset_sessions, batch_size):
            sched = _lib.Schedule(test_data_items, offset_sessions, None, batch_size, 0, mode=1 | _lib.SCHED_POSITIONS, n_history=n_hist)
            rec, mrr, n, counts, top_i, top_s = eng.eval_events(sched, cuts, _MODES[mode], k)
        pos = sched.positions()
    finally:
        if items is not None:
            eng.set_eval_items(None)
    gru.predict = None                                     # the scoring hidden state is shared with predict_next_batch
    # events in schedule order -> rows of the sorted frame (the target's row), then frame order
    if n_hist is None:
        M = sched.batch_sizes()
        row = (pos[np.arange(pos.shape[1])[None, :] < M[:, None]] + 1).astype(np.int64)
    else:
        row = (pos[sched.counted()] + 1).astype(np.int64)
    order = np.argsort(row, kind='stable')
    return _events_result(gru, test_data, row[order], counts[order], rec, mrr, n, cuts, mode, k, top_i[order] if k else None,
                          top_s[order] if k else None, session_key, item_key, time_key)


def _relevant(test_data_items, offset_sessions, n_hist):
    """the counted events in frame order and their relevant sets: for the input at row p, the distinct items of rows p+1 ..
    end of its session, first occurrence first.  Returns (input rows, items, offsets (row of first occurrence - p), CSR
    pointer [n_events + 1])"""
    rows, items, offs, ptr = [], [], [], [0]
    for s in range(len(offset_sessions) - 1):
        a, b = int(offset_sessions[s]), int(offset_sessions[s + 1])
        for t in range(a + max(int(n_hist[s]) if n_hist is not None else 0, 1), b):
            seen = set()
            for q in range(t, b):
                it = test_data_items[q]
                if it not in seen:
                    seen.add(it)
                    items.append(it)
                    offs.append(q - t + 1)
            rows.append(t - 1)
            ptr.append(len(items))
    return np.array(rows, np.int64), np.array(items, np.int64), np.array(offs, np.int64), np.array(ptr, np.int64)


def _rest_budget(test_data, session_key, offset_sessions, lanes):
    """the library's limit on the relevant lists (lanes x (longest session - 1) int32 within the seen-list budget), checked
    here first for a ValueError that names the longest session"""
    lens = np.diff(offset_sessions)
    if not len(lens):
        return
    j = int(np.argmax(lens))
    need = int(lanes) * max(1, int(lens[j]) - 1) * 4
    if need > _lib.seen_budget():
        sid = test_data[session_key].values[offset_sessions[j]]
        sid = sid.item() if isinstance(sid, np.generic) else sid
        raise ValueError('evaluate_rest: session %r has %d events; its relevant lists for %d lanes take %d bytes, over the %d-byte '
                         'budget' % (sid, int(lens[j]), int(lanes), need, _lib.seen_budget()))


_REST_METRICS = ('hitrate', 'precision', 'recall', 'mrr', 'ndcg', 'map')


def evaluate_rest(gru, test_data, items=None, session_key='SessionId', item_key='ItemId', time_key='Time', cut_off=[20], batch_size=100,
                  mode='standard', exclude_seen=False, history=None):
    '''
    Rest-of-session evaluation: every event evaluate_gpu counts (same arguments, including `history`) is scored once against
    the catalogue, and each DISTINCT item of the rest of its session (the items after the input, first occurrence first, the
    next item first) is ranked as if it were the event's target, among the same competitors and by the formula of `mode`.
    Two relevant items compete with each other like any other items, so a rank is a list position.  In 'tiebreaking' a
    relevant item's score carries the noise of its own column, so it never beats itself.

    - `exclude_seen`: competitors leave out the session's inputs so far, as in evaluate_gpu; a relevant item the session has
      already input is a miss (rank inf) and still counts in |R|.
    - `items`: only these items compete, as in evaluate_gpu.  A relevant item that is NOT listed can never be recommended: it
      is a miss (rank inf) and still counts in |R|.  This differs from evaluate_gpu, where an unlisted target still gets a rank.

    Per event, with R the relevant set, r_j the rank of j and hits = |{j in R: r_j <= N}| (misses never hit), averaged over the
    events: HitRate@N = [hits > 0], Precision@N = hits / N, Recall@N = hits / |R|, MRR@N = 1 / min r_j if that is <= N,
    NDCG@N = sum_{r_j <= N} 1 / log2(r_j + 1) over sum_{i <= min(|R|, N)} 1 / log2(i + 1), MAP@N = sum_{r_j <= N}
    (|{i in R: r_i <= r_j}| / r_j) / min(|R|, N).  With |R| = 1 they are evaluate_gpu's Recall (HitRate, Recall) and MRR
    (MRR, MAP), evaluate_events' NDCG, and Precision = Recall / N.

    Returns a dict: 'hitrate', 'precision', 'recall', 'mrr', 'ndcg', 'map' (lists, one entry per cut-off, from sums kept in
    double on the device), 'n_events', 'n_pairs' and 'pairs': a DataFrame with one row per (event, relevant item) in frame order:
    session id, the event's time (that of its next item, as in evaluate_events), 'input_item', the relevant item (`item_key`),
    'offset' (events after the input where the item first occurs; 1 = the next item) and 'rank' (float64, inf for a miss).
    The relevant lists take batch_size x (longest session - 1) int32 on the device within 256 MiB; over that it raises
    ValueError naming the session.  They take the tile kind of the next-item ranking.  Single process only (NotImplementedError
    under torch.distributed); the baselines are not covered yet (NotImplementedError).
    '''
    if isinstance(gru, Baseline):
        raise NotImplementedError('evaluate_rest does not cover the baselines yet')
    if gru.error_during_train: raise Exception
    if mode not in _MODES:
        raise NotImplementedError
    if gru._world()[0] > 1:
        raise NotImplementedError('evaluate_rest runs in a single process')
    cuts = _cuts(cut_off)
    test_data, test_data_items, offset_sessions, n_hist = _prepare_history(gru, test_data, history, session_key, item_key, time_key)
    _rest_budget(test_data, session_key, offset_sessions, batch_size)
    rows, rel, off, ptr = _relevant(test_data_items, offset_sessions, n_hist)
    eng = gru._ensure_engine(batch_size)
    if items is not None:
        eng.set_eval_items(gru.itemidmap[items].values)
    try:
        with _ExcludeSeen(eng, exclude_seen, test_data, session_key, offset_sessions, batch_size):
            sched = _lib.Schedule(test_data_items, offset_sessions, None, batch_size, 0, mode=1 | _lib.SCHED_POSITIONS, n_history=n_hist)
            sums, n, n_pairs, counts, offsets = eng.eval_rest(sched, cuts, _MODES[mode])
        pos = sched.positions()
    finally:
        if items is not None:
            eng.set_eval_items(None)
    gru.predict = None                                     # the scoring hidden state is shared with predict_next_batch
    # events in schedule order -> frame order (by input row); each event's pairs keep their first-occurrence order
    if n_hist is None:
        M = sched.batch_sizes()
        inp = pos[np.arange(pos.shape[1])[None, :] < M[:, None]].astype(np.int64)
    else:
        inp = pos[sched.counted()].astype(np.int64)
    order = np.argsort(inp, kind='stable')
    lens = np.diff(offsets)[order]
    if n != len(rows) or n_pairs != len(rel) or not np.array_equal(inp[order], rows) or not np.array_equal(lens, np.diff(ptr)):
        raise RuntimeError('evaluate_rest: the device ranked other events than the test data holds')
    idx = np.repeat(offsets[:-1][order] - ptr[:-1], lens) + np.arange(len(rel))
    rank = _ranks(counts[idx], mode) if len(rel) else np.zeros(0)
    ev = np.repeat(np.arange(len(rows)), lens)
    inp_rows, tgt_rows = rows[ev], rows[ev] + 1
    pairs = pd.DataFrame({session_key: test_data[session_key].values[inp_rows], time_key: test_data[time_key].values[tgt_rows],
                          'input_item': test_data[item_key].values[inp_rows], item_key: gru.itemidmap.index.values[rel],
                          'offset': off, 'rank': rank})
    out = {m: [float(v) / n if n else float('nan') for v in sums[i]] for i, m in enumerate(_REST_METRICS)}
    out.update(n_events=int(n), n_pairs=int(n_pairs), pairs=pairs)
    return out


def _events_result(gru, test_data, row, counts, rec, mrr, n, cuts, mode, k, top_i, top_s, session_key, item_key, time_key):
    """evaluate_events' result from the counted events in frame order: `row` the frame rows of their targets, their counts,
    the device sums and (k > 0) their lists of item indices"""
    rank = _ranks(counts, mode)
    tgt, inp = test_data.iloc[row], test_data.iloc[row - 1]
    events = pd.DataFrame({session_key: tgt[session_key].values, time_key: tgt[time_key].values, 'input_item': inp[item_key].values,
                           item_key: tgt[item_key].values, 'rank': rank})
    with np.errstate(divide='ignore'):
        ndcg = [float(np.where(rank <= c, 1.0 / np.log2(rank + 1.0), 0.0).mean()) if n else float('nan') for c in cuts]
    out = {'events': events, 'recall': [float(r) / n for r in rec], 'mrr': [float(m) / n for m in mrr], 'ndcg': ndcg}
    if k:
        ids = gru.itemidmap.index.values
        pad = top_i < 0                                    # exclude_seen: fewer than k eligible items
        if pad.any():
            out['topk_items'] = ids[np.where(pad, 0, top_i)].astype(object)
            out['topk_items'][pad] = None
        else:
            out['topk_items'] = ids[top_i]
        out['topk_scores'] = top_s
        out['coverage'] = len(np.unique(top_i[~pad])) / gru.n_items
    return out


def _evaluate_baseline(model, test_data, items, session_key, item_key, time_key, cut_off, mode, k, exclude_seen, history, sums_only):
    """evaluate_gpu (sums_only) / evaluate_events of a baseline (DESIGN §3j): the same preparation, `items` lookup, rank rules
    and result layout as for a GRU4Rec model; every counted event is ranked on the device on its own (a baseline has no
    recurrent state), so batch_size has no effect.  Single process only."""
    if mode not in _MODES:
        raise NotImplementedError
    if model._world()[0] > 1:
        raise NotImplementedError('the baselines are evaluated in a single process')
    cand = None if items is None else model.itemidmap[items].values      # KeyError for unknown ids
    if k != 0:
        k = _lib.check_topk(k, model.n_items if cand is None else len(set(cand)))
    cuts = _cuts(cut_off)
    if sums_only:
        print('Measuring Recall@{} and MRR@{}'.format(','.join([str(c) for c in cuts]), ','.join([str(c) for c in cuts])))
    test_data, test_data_items, offset_sessions, n_hist = _prepare_history(model, test_data, history, session_key, item_key, time_key)
    model._cover(int(np.diff(offset_sessions).max(initial=0)))
    rec, mrr, n, counts, top_i, top_s = model._device().evaluate(test_data_items, offset_sessions, n_hist, cuts, _MODES[mode], cand,
                                                                 exclude_seen, k, counts=not sums_only)
    if sums_only:
        return [float(r) / n for r in rec], [float(m) / n for m in mrr]
    # the counted events' targets: every row past the first max(n_history, 1) of its session, in frame order
    lens = np.diff(offset_sessions)
    first = np.repeat(np.maximum(n_hist if n_hist is not None else np.zeros(len(lens), np.int32), 1), lens)
    row = np.flatnonzero(np.arange(len(test_data)) - np.repeat(offset_sessions[:-1], lens) >= first)
    return _events_result(model, test_data, row, counts, rec, mrr, n, cuts, mode, k, top_i, top_s, session_key, item_key, time_key)
