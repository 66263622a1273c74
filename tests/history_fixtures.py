"""The CPU expectation of the grouped history call (cb200_scan_extract_decode_chunks_grouped_history_dev): the rule of include/cb200.h
restated in numpy on top of the grouped call's assignment (group_fixtures.assign).  The history's pictures come first in the
positions and are always eligible; a group needs a batch member; a group is done when its record or one of its batch members' own
records is complete; the history keeps the last `capacity` eligible pictures that are in no done group and, in the batch, whose own
record is not complete."""
from group_fixtures import assign


def history_rule(match, h, batch_eligible, own_complete, group_complete, capacity):
    """the rule of a grouped history call (cb200_scan_extract_decode_chunks_grouped_history_dev) over N = h + n positions: the h
    history pictures (always eligible), then the batch.  match: N x N booleans (only j < i is read); own_complete[i]: batch picture
    i's own record is complete; group_complete(g, members): group g's record is complete.  Returns (group_of of the batch, count,
    each group's member positions, the kept positions oldest first: the new history)"""
    N = len(match)
    eligible = [True] * h + [bool(e) for e in batch_eligible]
    of, m = assign(match, eligible)
    members = [[p for p in range(N) if of[p] == g] for g in range(m)]
    number = {}
    for g in range(m):
        if members[g][-1] >= h:                      # a group needs a batch member
            number[g] = len(number)
    groups = [members[g] for g in number]
    pos_group = [number.get(of[p], -1) if of[p] >= 0 else -1 for p in range(N)]
    done = [bool(group_complete(g, groups[g])) for g in range(len(groups))]
    for p in range(h, N):
        if pos_group[p] >= 0 and own_complete[p - h]:
            done[pos_group[p]] = True
    kept = [p for p in range(N) if eligible[p] and not (pos_group[p] >= 0 and done[pos_group[p]]) and (p < h or not own_complete[p - h])]
    return pos_group[h:], len(groups), groups, kept[max(0, len(kept) - capacity):]
