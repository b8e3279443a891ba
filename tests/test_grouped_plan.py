"""-m "not gpu": isolation groups in the device batcher's host half (renet_host_plan_batch_grouped), checked through the
numpy statement of the induced-edge filter that test_host_batching.py uses for renet_induce_edges."""
import numpy as np
import pytest

from renet_b200 import hoststore, synthetic
from test_host_batching import _induce_numpy


@pytest.fixture(scope='module')
def stores():
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=31, num_timestamps=14)
    S, ST, O, OT = synthetic.build_history(quads)
    gs = hoststore.GraphStore(synthetic.build_graph_dict(quads, num_r))
    return quads, gs, {0: hoststore.HistoryStore(S, ST, quads[:, 0], gs), 2: hoststore.HistoryStore(O, OT, quads[:, 2], gs)}


def _plan(view, sort=True):
    buf = np.zeros(1 << 21, np.int32)
    r = hoststore.plan_view_raw(view, buf, sort)
    assert 'need_words' not in r
    return r, buf


def _plain_plan(view, sort=True):
    """renet_host_plan_batch itself (no groups argument)."""
    from renet_b200 import _lib
    L, hs, gs = _lib.lib(), view.store, view.store.gs
    B = len(view.sample_idx)
    s_idx, bsz, sizes = np.empty(B, np.int64), np.zeros(hoststore.MAX_LEN, np.int32), np.zeros(10, np.int64)
    buf = np.zeros(1 << 21, np.int32)
    p = hoststore._p
    rc = L.renet_host_plan_batch(len(gs.times), p(gs.node_off), p(gs.node_ent), p(gs.edge_off), p(hs.samp_off), p(hs.samp_entry),
                                 p(hs.ent_graph), p(hs.ent_srow), p(hs.ent_off), p(hs.nbr_row), p(view.sample_idx), B, int(sort),
                                 p(s_idx), p(buf), buf.size, p(bsz), hoststore.MAX_LEN, p(sizes))
    _lib.check(rc, 'renet_host_plan_batch')
    return sizes, s_idx, bsz, buf


def test_null_and_equal_groups_are_the_plain_plan(stores):
    quads, gs, hss = stores
    rng = np.random.RandomState(4)
    for col, hs in hss.items():
        for B in (1, 37, 400):
            sel = rng.randint(0, len(quads), B)
            for sort in (True, False):
                if not sort:
                    lens = np.diff(hs.samp_off)[sel]
                    sel = np.concatenate((sel[lens > 0], sel[lens == 0]))
                sizes, s_idx, bsz, ref = _plain_plan(hs.select(sel), sort)
                for groups in (None, np.full(B, 7), np.full(B, -3)):
                    r, buf = _plan(hs.select(sel, groups), sort)
                    w = int(sizes[6])
                    assert r['words'] == w
                    np.testing.assert_array_equal(buf[:w], ref[:w])
                    np.testing.assert_array_equal(r['s_idx'], s_idx)
                    np.testing.assert_array_equal(r['batch_sizes'], bsz[:r['max_len']])


def _group_parts(gs, r, buf, groups):
    """Per group: its components (in plan order), its node list and, in that node numbering, its batched graph and its
    read-out rows, as what the group batched alone would give."""
    p = hoststore.split_plan(buf, r)
    ind = _induce_numpy(gs, p)
    G = r['G']
    comp_nodes = []
    for c in range(G):
        m = p['newid'][p['mark_off'][c]:p['mark_off'][c + 1]]
        comp_nodes.append(np.sort(m[m >= 0]))
    seq_group = groups[p['s_idx'][:r['Q']]]
    row_group = seq_group[p['row_seq']]
    comp_group = np.full(G, np.iinfo(np.int64).min)
    comp_group[p['row_comp']] = row_group
    dst = np.repeat(np.arange(r['N']), np.diff(ind['row_ptr']))
    out = {}
    for grp in np.unique(groups):
        comps = np.flatnonzero(comp_group == grp)
        nodes = np.concatenate([comp_nodes[c] for c in comps]) if len(comps) else np.zeros(0, np.int64)
        local = np.full(r['N'], -1)
        local[nodes] = np.arange(len(nodes))
        keep = local[dst] >= 0
        assert np.all((local[ind['col_src'][keep]] >= 0))                   # no edge crosses groups
        assert not np.any(local[ind['col_src'][~keep]] >= 0)
        rows = np.flatnonzero(row_group == grp)
        comp_local = np.full(G, -1)
        comp_local[comps] = np.arange(len(comps))
        out[int(grp)] = dict(comp_graph=p['comp_graph'][comps], node_ent=p['node_ent'][nodes],
                             edges=np.stack((local[dst[keep]], local[ind['col_src'][keep]], ind['col_type_s'][keep],
                                             ind['col_type_o'][keep]), 1),
                             norm=ind['norm'][nodes], readout=local[p['readout'][rows]], row_comp=comp_local[p['row_comp'][rows]],
                             seq_len=p['seq_len'][np.flatnonzero(seq_group == grp)])
    return out


def test_each_group_equals_the_group_batched_alone(stores):
    quads, gs, hss = stores
    rng = np.random.RandomState(9)
    late = np.arange(len(quads) // 2, len(quads))          # long histories that share most timestamps across groups
    for col, hs in hss.items():
        for B, n_groups in ((60, 5), (300, 40), (12, 12)):
            sel = rng.choice(late, B)
            sel[:3] = rng.randint(0, 20, 3)                 # a few empty or short histories
            groups = rng.randint(0, n_groups, B) * 11 - 5
            r, buf = _plan(hs.select(sel, groups))
            got = _group_parts(gs, r, buf, groups)
            total_G = 0
            for grp, part in got.items():
                mine = groups == grp
                ra, ba = _plan(hs.select(sel[mine]))
                total_G += ra['G']
                if ra['S'] == 0:
                    assert len(part['readout']) == 0 and len(part['comp_graph']) == 0
                    continue
                alone = _group_parts(gs, ra, ba, np.zeros(int(mine.sum()), np.int64))[0]
                for k in ('comp_graph', 'node_ent', 'edges', 'norm', 'readout', 'row_comp', 'seq_len'):
                    np.testing.assert_array_equal(part[k], alone[k], err_msg='group %d: %s' % (grp, k))
            assert r['G'] == total_G
            assert len(np.unique(hoststore.split_plan(buf, r)['comp_graph'])) < r['G']    # graphs repeat across groups


def test_groups_need_the_device_batcher(stores):
    quads, gs, hss = stores
    view = hss[0].select(np.arange(10), np.arange(10))
    with pytest.raises(ValueError, match='device batcher'):
        hoststore.assemble_view_raw(view, np.zeros(1 << 16, np.int32))
    with pytest.raises(ValueError, match='device batcher'):
        hoststore.assemble_view(view, 'cpu', device_edges=False)
    with pytest.raises(ValueError, match='groups'):
        hss[0].select(np.arange(10), np.arange(9))
    ld = hoststore.NativeLoader(1)
    try:
        with pytest.raises(ValueError, match='isolation groups'):
            ld.submit(view, np.zeros(1 << 16, np.int32), True, True)
    finally:
        ld.close()
