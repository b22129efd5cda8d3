"""The heaviest clients of logical services merged across ranks (GYSK_FLAG_SVC_TOP_CLIENTS with a logical map) restated on the CPU.
Each rank holds one tests/svc_top_clients.TopClients. On each rank the members' summaries are folded in map order, acc = merge(acc, s)
from the empty summary; then the ranks' results are folded in ascending rank order the same way. The merge is not associative, so the
order is part of the answer."""
from tests import svc_top_clients as tc


def fold(summaries):
    """acc = merge(acc, s) over the summaries in order, from the empty summary"""
    acc = tc.EMPTY
    for s in summaries:
        acc = tc.merge([acc, s])
    return acc


def rank_summary(model, which, members):
    """one rank's fold of the members (glob ids in map order); a member the rank does not hold gives the empty summary, which leaves the
    accumulator as it is, as the device's skip does"""
    return fold(model.get(which, m) for m in members)


def logical_summary(models, which, members):
    """the fold of every rank's fold, ranks ascending (models[r]: rank r's TopClients)"""
    return fold(rank_summary(m, which, members) for m in models)


def members_of(glob_ids, logical_ids):
    """{logical id: [glob ids in map order]} of gysk_set_logical_map's lists"""
    out = {}
    for g, l in zip(glob_ids.tolist(), logical_ids.tolist()):
        out.setdefault(l, []).append(g)
    return out
