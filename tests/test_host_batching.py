"""-m "not gpu": the product's host-side batching (renet_b200.utils / graph / synthetic) against the
oracle restatement of reference utils.py:68-93,115-181,209-244 and get_history_graph.py:142-190."""
import numpy as np
import torch

from helpers import load_npz
from oracle import restate
from renet_b200 import synthetic, utils
from renet_b200.graph import get_big_graph


def _tiny():
    quads, num_e, num_r = synthetic.make_quads('tiny', seed=3)
    return quads, num_e, num_r


def test_get_big_graph_matches_reference_golden():
    b = load_npz('graph_kats.npz')
    quads, R = b['quads'].astype(np.int64), int(b['R'])
    for tt in np.unique(quads[:, 3]):
        g = get_big_graph(quads[quads[:, 3] == tt][:, :3], R)
        src, dst = g.edges()
        np.testing.assert_array_equal(g.ndata['id'].view(-1).numpy(), b['g%d/id' % tt])
        np.testing.assert_array_equal(src.numpy(), b['g%d/src' % tt])
        np.testing.assert_array_equal(dst.numpy(), b['g%d/dst' % tt])
        np.testing.assert_array_equal(g.edata['type_s'].numpy(), b['g%d/type_s' % tt])
        np.testing.assert_array_equal(g.edata['type_o'].numpy(), b['g%d/type_o' % tt])
        np.testing.assert_array_equal(g.ndata['norm'].view(-1).numpy(), b['g%d/norm' % tt])
        assert g.ids == {int(e): i for i, e in enumerate(b['g%d/id' % tt])}
        assert np.all(np.diff(g.dst) >= 0)      # destination-sorted copy


def test_build_history_matches_oracle():
    quads, num_e, _ = _tiny()
    a = synthetic.build_history(quads)
    b = restate.build_history(quads, num_e)
    for x, y in zip(a, b):
        assert len(x) == len(y)
        for hx, hy in zip(x, y):
            assert len(hx) == len(hy)
            for ex, ey in zip(hx, hy):
                np.testing.assert_array_equal(np.asarray(ex), np.asarray(ey))
    assert max(len(h) for h in a[0]) == 10     # rolling window of 10 (get_history_graph.py:118)


def _check_batch(quads, num_r, sel, col, hist, hist_t):
    gd_p = synthetic.build_graph_dict(quads, num_r)
    gd_o = restate.build_graph_dict(quads, num_r)
    H, HT = [hist[i] for i in sel], [hist_t[i] for i in sel]
    hb = utils.assemble_history_batch_host(H, HT, quads[sel][:, col], gd_p, sort=True)
    bo = restate.assemble_batch(H, HT, quads[sel][:, col], sort=True)
    go = restate.batch_graphs(bo, gd_o)
    g = hb.graph
    np.testing.assert_array_equal(hb.seq_len, bo.seq_len)
    np.testing.assert_array_equal(hb.s_idx, bo.s_idx)
    assert list(hb.times) == list(bo.times)
    # nodes: same (component, entity) multiset; the product orders nodes by (component, entity id)
    comp_of = np.repeat(np.arange(len(g['comp_sizes'])), g['comp_sizes'])
    key_p = comp_of * 10 ** 6 + g['node_ent']
    comp_o = np.repeat(np.arange(len(go.comp_sizes)), go.comp_sizes)
    key_o = comp_o * 10 ** 6 + go.id
    np.testing.assert_array_equal(np.sort(key_p), np.sort(key_o))
    # per-node norm and per-edge (src key, dst key, type_s, type_o) multisets agree
    order_p, order_o = np.argsort(key_p), np.argsort(key_o)
    np.testing.assert_array_equal(g['norm'][order_p], go.norm[order_o])
    dst_p = np.repeat(np.arange(len(key_p)), np.diff(g['row_ptr']))
    ep = np.stack((key_p[g['col_src']], key_p[dst_p], g['col_type_s'], g['col_type_o']), 1)
    eo = np.stack((key_o[go.src], key_o[go.dst], go.type_s, go.type_o), 1)
    assert len(ep) == len(eo)
    np.testing.assert_array_equal(ep[np.lexsort(ep.T[::-1])], eo[np.lexsort(eo.T[::-1])])
    assert np.all(np.diff(dst_p) >= 0)
    # read-out rows point at the same (component, entity)
    np.testing.assert_array_equal(key_p[hb.readout_host], key_o[go.readout])
    # packed order == torch's pack_padded_sequence
    perm, bs = restate.packed_order(hb.seq_len)
    np.testing.assert_array_equal(hb.batch_sizes, bs)
    np.testing.assert_array_equal(hb.readout[5], perm)


def test_assemble_history_batch_matches_oracle_tiny():
    quads, num_e, num_r = _tiny()
    S, ST, O, OT = synthetic.build_history(quads)
    sel = np.arange(len(quads) - 120, len(quads))
    _check_batch(quads, num_r, sel, 0, S, ST)
    _check_batch(quads, num_r, sel, 2, O, OT)


def test_assemble_history_batch_matches_oracle_icews18_shape():
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=5, num_timestamps=14)
    S, ST, O, OT = synthetic.build_history(quads)
    sel = np.random.RandomState(0).permutation(np.arange(len(quads) // 2, len(quads)))[:256]
    _check_batch(quads, num_r, sel, 0, S, ST)
    _check_batch(quads, num_r, sel, 2, O, OT)


def test_empty_and_ragged_histories():
    quads, num_e, num_r = _tiny()
    S, ST, O, OT = synthetic.build_history(quads)
    gd = synthetic.build_graph_dict(quads, num_r)
    # first samples of the stream have empty histories; mix them with full ones
    sel = np.concatenate((np.arange(0, 10), np.arange(len(quads) - 10, len(quads))))
    hb = utils.assemble_history_batch_host([S[i] for i in sel], [ST[i] for i in sel], quads[sel][:, 0], gd)
    assert hb.num_seq == sum(1 for i in sel if len(S[i]) > 0) < len(sel)
    assert np.all(np.diff(hb.seq_len) <= 0)
    # all-empty batch
    hb = utils.assemble_history_batch_host([[], []], [[], []], np.asarray([1, 2]), gd)
    assert hb.graph is None and hb.S == 0


def test_cpp_batcher_matches_numpy_path():
    """renet_host_assemble_batch (C++) produces exactly the batch of the numpy path (same node order,
    same CSR, same bookkeeping) on an ICEWS18-shaped stream, both directions."""
    from renet_b200 import hoststore
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=11, num_timestamps=16)
    S, ST, O, OT = synthetic.build_history(quads)
    gd = synthetic.build_graph_dict(quads, num_r)
    gs = hoststore.GraphStore(gd)
    sel = np.random.RandomState(1).permutation(len(quads))[:300]     # includes empty histories
    for hist, hist_t, col in ((S, ST, 0), (O, OT, 2)):
        hs = hoststore.HistoryStore(hist, hist_t, quads[:, col], gs)
        view = hs.select(sel)
        buf = np.zeros(8, dtype=np.int32)
        r = hoststore.assemble_view_raw(view, buf)
        assert 'need_words' in r                       # too small: reports the size it needs
        buf = np.zeros(r['need_words'], dtype=np.int32)
        r = hoststore.assemble_view_raw(view, buf)
        got = hoststore.split_raw(buf, r)
        hb = utils.assemble_history_batch_host([hist[i] for i in sel], [hist_t[i] for i in sel], quads[sel][:, col], gd)
        g = hb.graph
        np.testing.assert_array_equal(r['s_idx'], hb.s_idx)
        assert (r['N'], r['E'], r['S'], r['Q']) == (len(g['node_ent']), len(g['col_src']), hb.S, hb.num_seq)
        for k in ('node_ent', 'row_ptr', 'col_src', 'col_type_s', 'col_type_o'):
            np.testing.assert_array_equal(got[k], g[k].astype(np.int32), err_msg=k)
        np.testing.assert_array_equal(got['norm'].view(np.float32), g['norm'])
        readout, row_comp, row_seq, seq_start, seq_len, packed_row = hb.readout
        for k, v in (('readout', readout), ('row_comp', row_comp), ('row_seq', row_seq), ('seq_start', seq_start),
                     ('seq_len', seq_len), ('packed_row', packed_row)):
            np.testing.assert_array_equal(got[k], np.asarray(v).astype(np.int32), err_msg=k)
        np.testing.assert_array_equal(r['batch_sizes'], hb.batch_sizes)
        np.testing.assert_array_equal(gs.times[r['comp_graph']], hb.times)
        np.testing.assert_array_equal(got['s_idx'], hb.s_idx)
    # all-empty batch
    view = hs.select(np.asarray([0, 1]))
    r = hoststore.assemble_view_raw(view, np.zeros(64, np.int32))
    assert r['S'] == 0 and r['N'] == 0


def _induce_numpy(gs, p):
    """numpy statement of what renet_induce_edges computes from a plan (candidate filter + CSR)."""
    src, ts, to, dst = [], [], [], []
    for c in range(len(p['comp_graph'])):
        g = int(p['comp_graph'][c])
        lo, hi = gs.edge_off[g], gs.edge_off[g + 1]
        assert p['cand_off'][c + 1] - p['cand_off'][c] == hi - lo
        m = p['newid'][p['mark_off'][c]:p['mark_off'][c + 1]]
        s, d = m[gs.src[lo:hi]], m[gs.dst[lo:hi]]
        keep = (s >= 0) & (d >= 0)
        src.append(s[keep]); dst.append(d[keep]); ts.append(gs.type_s[lo:hi][keep]); to.append(gs.type_o[lo:hi][keep])
    src, dst, ts, to = (np.concatenate(x) for x in (src, dst, ts, to))
    N = len(p['node_ent'])
    assert np.all(np.diff(dst) >= 0)                   # survivors are already sorted by batched destination
    row_ptr = np.searchsorted(dst, np.arange(N + 1)).astype(np.int32)
    deg = np.diff(row_ptr).astype(np.float32)
    return dict(row_ptr=row_ptr, col_src=src, col_type_s=ts, col_type_o=to, norm=np.float32(1) / np.maximum(deg, 1))


def test_plan_batch_plus_induce_matches_cpp_batcher():
    """renet_host_plan_batch (host half of the device batcher) + the induced-edge filter (numpy statement of
    renet_induce_edges here; the CUDA kernels are compared in tests/test_gpu_device_batch.py) == renet_host_assemble_batch."""
    from renet_b200 import hoststore
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=11, num_timestamps=16)
    S, ST, O, OT = synthetic.build_history(quads)
    gs = hoststore.GraphStore(synthetic.build_graph_dict(quads, num_r))
    sel = np.random.RandomState(1).permutation(len(quads))[:300]
    for hist, hist_t, col in ((S, ST, 0), (O, OT, 2)):
        view = hoststore.HistoryStore(hist, hist_t, quads[:, col], gs).select(sel)
        r = hoststore.assemble_view_raw(view, np.zeros(8, np.int32))
        buf = np.zeros(r['need_words'], dtype=np.int32)
        r = hoststore.assemble_view_raw(view, buf)
        ref = hoststore.split_raw(buf, r)
        pr = hoststore.plan_view_raw(view, np.zeros(8, np.int32))
        assert 'need_words' in pr
        pbuf = np.zeros(pr['need_words'], dtype=np.int32)
        pr = hoststore.plan_view_raw(view, pbuf)
        p = hoststore.split_plan(pbuf, pr)
        assert (pr['N'], pr['S'], pr['Q'], pr['G']) == (r['N'], r['S'], r['Q'], r['G']) and pr['E_cand'] >= r['E']
        np.testing.assert_array_equal(pr['s_idx'], r['s_idx'])
        np.testing.assert_array_equal(pr['batch_sizes'], r['batch_sizes'])
        for k in ('node_ent', 'readout', 'row_comp', 'row_seq', 'seq_start', 'seq_len', 'packed_row', 's_idx', 'comp_graph'):
            np.testing.assert_array_equal(p[k], ref[k], err_msg=k)
        ind = _induce_numpy(gs, p)
        for k in ('row_ptr', 'col_src', 'col_type_s', 'col_type_o'):
            np.testing.assert_array_equal(ind[k], ref[k], err_msg=k)
        np.testing.assert_array_equal(ind['norm'], ref['norm'].view(np.float32))
    pr = hoststore.plan_view_raw(view.store.select(np.asarray([0, 1])), np.zeros(64, np.int32))
    assert pr['S'] == 0 and pr['N'] == 0


def test_native_loader_jobs_equal_synchronous_calls():
    """renet_loader_* (C++ worker threads) produce the buffers of the synchronous entry points, in ticket order,
    and report a too-small staging buffer the same way."""
    from renet_b200 import hoststore
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=11, num_timestamps=16)
    S, ST, O, OT = synthetic.build_history(quads)
    gs = hoststore.GraphStore(synthetic.build_graph_dict(quads, num_r))
    hs = hoststore.HistoryStore(S, ST, quads[:, 0], gs)
    ld = hoststore.NativeLoader(4)
    sels = [np.random.RandomState(i).permutation(len(quads))[:300] for i in range(6)]
    for device_edges, sync in ((True, hoststore.plan_view_raw), (False, hoststore.assemble_view_raw)):
        jobs = [ld.submit(hs.select(s), np.zeros(1 << 20, np.int32), True, device_edges) for s in sels]
        for s, j in zip(sels, jobs):
            r = ld.finish(j)
            ref_buf = np.zeros(1 << 20, np.int32)
            ref = sync(hs.select(s), ref_buf)
            assert r['words'] == ref['words']
            np.testing.assert_array_equal(j['out'][:r['words']], ref_buf[:r['words']])
            np.testing.assert_array_equal(r['s_idx'], ref['s_idx'])
            np.testing.assert_array_equal(r['batch_sizes'], ref['batch_sizes'])
    small = ld.finish(ld.submit(hs.select(sels[0]), np.zeros(8, np.int32), True, True))
    assert small == {'need_words': sync and hoststore.plan_view_raw(hs.select(sels[0]), np.zeros(8, np.int32))['need_words']}
    ld.close()


def test_lazy_edge_count_resolves_once_and_trims_columns():
    """BatchedHistoryGraph.E of a device-assembled batch: produced on the GPU, read back asynchronously (PendingCount);
    E_launch never waits, E / edge_count_handle() wait once, trim the capacity-sized columns and release the slot once."""
    import torch
    from renet_b200.graph import BatchedHistoryGraph, PendingCount

    class FakeEvent:
        def __init__(self):
            self.syncs = 0

        def synchronize(self):
            self.syncs += 1

    released = []
    ev, pinned = FakeEvent(), torch.tensor([5], dtype=torch.int32)
    g = BatchedHistoryGraph.__new__(BatchedHistoryGraph)
    g.N, g.E_cap = 3, 9
    g._E_pending = PendingCount(ev, pinned, released.append)
    g.col_src, g.col_type_s, g.col_type_o = (torch.arange(9, dtype=torch.int32) for _ in range(3))
    assert g.E_launch == 9 and ev.syncs == 0                 # launch argument: the capacity bound, no wait
    h = g.edge_count_handle()
    assert g.E == 5 and ev.syncs == 1 and len(released) == 1
    assert g.E_launch == 5 and g.number_of_edges() == 5
    assert [len(x) for x in (g.col_src, g.col_type_s, g.col_type_o)] == [5, 5, 5]
    assert h.value() == 5 and ev.syncs == 1 and len(released) == 1      # the handle shares the resolved count
    assert g.edge_count_handle().value() == 5
    # handle first, graph later (bench.py keeps only handles and lets the batch go)
    ev2 = FakeEvent()
    g2 = BatchedHistoryGraph.__new__(BatchedHistoryGraph)
    g2.N, g2.E_cap = 3, 4
    g2._E_pending = PendingCount(ev2, torch.tensor([2], dtype=torch.int32), released.append)
    g2.col_src, g2.col_type_s, g2.col_type_o = (torch.arange(4, dtype=torch.int32) for _ in range(3))
    h2 = g2.edge_count_handle()
    assert h2.value() == 2 and g2.E == 2 and ev2.syncs == 1 and len(released) == 2
    # host-assembled batch: the count is known from the start
    g3 = BatchedHistoryGraph.__new__(BatchedHistoryGraph)
    g3.E = 7
    assert g3.E == 7 and g3.E_launch == 7 and g3.edge_count_handle().value() == 7


def test_batchers_agree_on_random_batches_sorted_and_unsorted():
    """Randomised cross-check of the three host paths (numpy, C++ all-host, C++ plan + induced-edge filter) on batches
    with duplicate samples, mixed empty histories, tiny and large sizes, in both sample orders (utils.py:209-244 sorts by
    history length, :246-283 keeps the given order and needs the non-empty histories first)."""
    from renet_b200 import hoststore
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=23, num_timestamps=12)
    S, ST, O, OT = synthetic.build_history(quads)
    gd = synthetic.build_graph_dict(quads, num_r)
    gs = hoststore.GraphStore(gd)
    hs = hoststore.HistoryStore(S, ST, quads[:, 0], gs)
    lens = np.asarray([len(x) for x in S])
    rng = np.random.RandomState(77)
    for trial in range(12):
        B = int(rng.choice([1, 2, 7, 64, 400]))
        sel = rng.randint(0, len(quads), B)                     # duplicates allowed
        for sort in (True, False):
            if not sort:                                        # unsorted twin: non-empty histories first
                sel = np.concatenate((sel[lens[sel] > 0], sel[lens[sel] == 0]))
            view = hs.select(sel)
            ref = utils.assemble_history_batch_host([S[i] for i in sel], [ST[i] for i in sel], quads[sel][:, 0], gd, sort)
            buf = np.zeros(1 << 20, np.int32)
            r = hoststore.assemble_view_raw(view, buf, sort)
            pbuf = np.zeros(1 << 20, np.int32)
            pr = hoststore.plan_view_raw(view, pbuf, sort)
            assert r['S'] == pr['S'] == ref.S
            if ref.S == 0:
                continue
            a, p = hoststore.split_raw(buf, r), hoststore.split_plan(pbuf, pr)
            ind = _induce_numpy(gs, p)
            g = ref.graph
            np.testing.assert_array_equal(r['s_idx'], ref.s_idx)
            np.testing.assert_array_equal(pr['s_idx'], ref.s_idx)
            for k in ('node_ent', 'row_ptr', 'col_src', 'col_type_s', 'col_type_o'):
                np.testing.assert_array_equal(a[k], g[k].astype(np.int32), err_msg=k)
            for k in ('row_ptr', 'col_src', 'col_type_s', 'col_type_o'):
                np.testing.assert_array_equal(ind[k], a[k], err_msg=k)
            np.testing.assert_array_equal(p['node_ent'], a['node_ent'])
            np.testing.assert_array_equal(ind['norm'], g['norm'])
            for k in ('readout', 'row_comp', 'row_seq', 'seq_start', 'seq_len', 'packed_row'):
                np.testing.assert_array_equal(p[k], a[k], err_msg=k)
            np.testing.assert_array_equal(pr['batch_sizes'], ref.batch_sizes)


def test_view_from_lists_equals_numpy_path_and_store_path():
    """hoststore.view_from_lists: a batch given as the reference's Python lists, flattened on the fly (no de-duplication),
    produces the numpy path's batch through the C++ batcher; unknown timestamps / entities raise KeyError."""
    import pytest
    from renet_b200 import hoststore
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=5, num_timestamps=14)
    S, ST, O, OT = synthetic.build_history(quads)
    gd = synthetic.build_graph_dict(quads, num_r)
    gs = hoststore.GraphStore(gd)
    sel = np.random.RandomState(2).permutation(len(quads))[:256]
    for hist, hist_t, col in ((S, ST, 0), (O, OT, 2)):
        h, ht, subj = [hist[i] for i in sel], [hist_t[i] for i in sel], quads[sel][:, col]
        view = hoststore.view_from_lists(h, ht, subj, gs)
        buf = np.zeros(1 << 20, np.int32)
        r = hoststore.assemble_view_raw(view, buf)
        got = hoststore.split_raw(buf, r)
        ref = utils.assemble_history_batch_host(h, ht, subj, gd)
        np.testing.assert_array_equal(r['s_idx'], ref.s_idx)
        for k in ('node_ent', 'row_ptr', 'col_src', 'col_type_s', 'col_type_o'):
            np.testing.assert_array_equal(got[k], ref.graph[k].astype(np.int32), err_msg=k)
        np.testing.assert_array_equal(got['readout'], np.asarray(ref.readout[0]).astype(np.int32))
    with pytest.raises(KeyError):
        hoststore.view_from_lists([[np.asarray([[0, 1]])]], [[10 ** 9]], [1], gs)          # unknown timestamp
    t0 = int(gs.times[0])
    with pytest.raises(KeyError):
        hoststore.view_from_lists([[np.asarray([[0, num_e + 5]])]], [[t0]], [int(gs.node_ent[0])], gs)   # unknown entity


def test_graph_store_relation_ranking():
    """GraphStore.hot_relations: relation ids of each type column by their frequency over the whole graph_dict (the list the
    batch-scale gather keeps resident rows for); host logic only (device='cpu')."""
    from renet_b200 import hoststore, synthetic
    tkg = synthetic.SyntheticTKG('icews14', seed=3, num_timestamps=12)
    gs = hoststore.GraphStore(tkg.graph_dict)
    hot = gs.hot_relations('cpu', n=32)
    for rev, col in ((False, 'type_s'), (True, 'type_o')):
        allc = np.concatenate([np.asarray(getattr(g, col), dtype=np.int64) for g in gs.graphs])
        freq = np.bincount(allc, minlength=gs.num_types)
        got = hot[rev].numpy()
        assert len(got) <= 32 and len(set(got.tolist())) == len(got)
        assert np.all(freq[got] > 0) and np.all(np.diff(freq[got]) <= 0)            # present, most frequent first
        assert freq[got].min() >= np.sort(freq)[::-1][min(31, np.count_nonzero(freq) - 1)]
    assert gs.hot_relations('cpu', n=32) is hot                                     # computed once per device


def test_graph_store_rejects_negative_edge_types():
    """Edge types index the relation weights: a GraphStore refuses a negative type_s or type_o, so neither batcher (the
    all-host one nor the device one) ever emits one."""
    import pytest
    from renet_b200 import hoststore
    from renet_b200.graph import HistoryGraph
    hoststore.GraphStore({0: HistoryGraph([3, 5], [0], [1], [0], [1])})
    for ts, to in (([-1], [1]), ([0], [-1])):
        with pytest.raises(ValueError):
            hoststore.GraphStore({0: HistoryGraph([3, 5], [0], [1], ts, to)})


def test_first_history_entry_shows_an_edge():
    """hoststore._first_entry_has_edge: True on histories drawn from the graph dict (the device batcher then never waits for
    its edge count to reject an edge-free batch), False when the first entry's neighbours are not the subject's neighbours
    in that timestamp's graph, and False for a batch of empty histories."""
    from renet_b200 import hoststore
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=5, num_timestamps=12)
    S, ST, O, OT = synthetic.build_history(quads)
    gs = hoststore.GraphStore(synthetic.build_graph_dict(quads, num_r))
    rng = np.random.RandomState(2)
    late = np.arange(len(quads) // 2, len(quads))
    for col, (hist, hist_t) in ((0, (S, ST)), (2, (O, OT))):
        store = hoststore.HistoryStore(hist, hist_t, quads[:, col], gs)
        lens = np.diff(store.samp_off)
        for _ in range(20):
            sel = rng.choice(late, 64)
            assert hoststore._first_entry_has_edge(store.select(sel)) == bool(lens[sel].any())
        assert not hoststore._first_entry_has_edge(store.select(np.flatnonzero(lens == 0)[:5]))
    # a history whose neighbour shares the subject's timestamp graph but no edge with it
    t = int(quads[0, 3])
    g = gs[t]
    ents = np.asarray(g.node_id if hasattr(g, 'node_id') else g.id)
    s = int(quads[0, 0])
    linked = set(quads[(quads[:, 3] == t) & (quads[:, 0] == s), 2]) | set(quads[(quads[:, 3] == t) & (quads[:, 2] == s), 0])
    other = next(int(e) for e in ents if int(e) != s and int(e) not in linked)
    bogus = hoststore.HistoryStore([[np.asarray([[0, other]], dtype=np.int64)]], [[t]], [s], gs, dedupe=False)
    assert not hoststore._first_entry_has_edge(bogus.select([0]))
