"""Deep, irregular request trees for the tests of the request-tree join and the critical-path walk
(tw_assemble_traces, tw_critical_paths), without a GPU.

A request is a spine of in-spans, one per level: the in-span at level d belongs to spine service d and calls
spine service d + 1 at callee position `spine` ("first": 0, "last": callees - 1); the deepest spine call's
server span is not in the batch.  Its other callee positions call leaf services (one per position, shared by
every level), whose in-spans are in the batch when `leaf_in_batch` and make no call of their own (one callee,
assign -1).  With `random_shape` every request draws its own depth (1 .. depth), spine position, which
leaf calls it makes and which of their server spans are in the batch; a leaf in-span then sometimes makes
its call, to a server outside the batch.

Times are int64 microseconds, built bottom-up (a call's length holds its server span plus network time),
then placed top-down, so that no window collapses; totals stay far below 2^53.  `timing` lays out the calls
of every in-span: "sequential" (one after another, in a random time order), "parallel" (overlapping, each
started before the one before it ended, the spine call ending last: the others are truncated), "nested"
(the longest call holds the others), "clipped" (sequential, the first starting before the in-span and the
last ending after it), "zero" / "negative" (sequential, with some non-spine calls of zero or negative
length), or "mixed" (every in-span draws one).  `const_times`: every leaf, gap and network time the same,
sequential calls in callee order (many equal self times).

Services come in `order`: "root" (spine level 0 first, then the leaves), "leaf" (the reverse) or
"shuffled" (services and the in-spans inside them in a random order), which changes the node ids the
join's in-place pointer jumping meets first."""
import numpy as np

from traceweaver_b200.batch import Problem, build_batch

TIMINGS = ("sequential", "parallel", "nested", "clipped", "zero", "negative")
ORDERS = ("root", "leaf", "shuffled")


def deep_trees(depth, callees=8, spine="last", leaf_in_batch=True, timing="sequential", requests=1,
               random_shape=False, order="root", seed=0, const_times=False):
    """dict: hb (HostBatch, build_batch(validate=False)), assign (the tw_pass_out.assign layout of the true
    links), in_caller (int32 [n_in]); per request: roots (node ids), depth (spine in-spans),
    open_calls (the node ids of the calls whose server span is not in the batch, deepest spine call first)."""
    assert 1 <= callees <= 8 and spine in ("first", "last") and order in ORDERS
    assert timing == "mixed" or timing in TIMINGS
    rng = np.random.default_rng(seed)
    leaf_len = (lambda: 10) if const_times else (lambda: int(rng.integers(5, 51)))
    net = (lambda: 1) if const_times else (lambda: int(rng.integers(1, 7)))
    gap = (lambda: 2) if const_times else (lambda: int(rng.integers(1, 9)))

    # 1. shapes.  node_svc[x]: (kind, index) with kind 0 = spine service `index`, 1 = leaf service `index`
    node_svc, node_calls, node_spine = [], [], []
    call_from, call_pos, call_child = [], [], []

    def new_node(svc):
        node_svc.append(svc)
        node_calls.append([])
        node_spine.append(-1)
        return len(node_svc) - 1

    def new_call(x, e, child):
        call_from.append(x)
        call_pos.append(e)
        call_child.append(child)
        node_calls[x].append(len(call_from) - 1)
        return len(call_from) - 1

    roots, depths, open_calls = [], [], []
    for _ in range(requests):
        D = int(rng.integers(1, depth + 1)) if random_shape else depth
        side = rng.choice(("first", "last")) if random_shape else spine
        sp = 0 if side == "first" else callees - 1
        x = new_node((0, 0))
        roots.append(x)
        depths.append(D)
        free = []
        for d in range(D):
            nxt = -1
            for e in range(callees):
                if e == sp:
                    nxt = new_node((0, d + 1)) if d + 1 < D else -1
                    c = new_call(x, e, nxt)
                    node_spine[x] = c
                    if nxt < 0:
                        free.insert(0, c)
                    continue
                if random_shape and rng.random() >= 0.75:
                    continue                                  # a callee this in-span does not call
                in_batch = leaf_in_batch and (not random_shape or rng.random() < 0.6)
                leaf = new_node((1, e)) if in_batch else -1
                c = new_call(x, e, leaf)
                if leaf < 0:
                    free.append(c)
                elif random_shape and rng.random() < 0.5:
                    free.append(new_call(leaf, 0, -1))
            x = nxt
        open_calls.append(free)
    n_nodes, n_calls = len(node_svc), len(call_from)

    # 2. lengths bottom-up (children are created after their parents): per call its offset from the caller's
    # start, its length and its server span's offset from the call's start; per in-span its length
    dur = np.zeros(n_nodes, np.int64)
    shrunk = {}                                               # call -> its length when zero or negative
    call_off = np.zeros(n_calls, np.int64)
    call_len = np.zeros(n_calls, np.int64)
    child_off = np.zeros(n_calls, np.int64)
    for x in range(n_nodes - 1, -1, -1):
        cs = node_calls[x]
        if not cs:
            dur[x] = leaf_len()
            continue
        for c in cs:
            y = call_child[c]
            if y >= 0:
                child_off[c] = net()
                call_len[c] = child_off[c] + dur[y] + net()
            else:
                call_len[c] = leaf_len()
        mode = timing if timing != "mixed" else TIMINGS[int(rng.integers(len(TIMINGS)))]
        dur[x] = _lay_out(rng, mode, cs, node_spine[x], call_off, call_len, gap, const_times, shrunk)

    # 3. times top-down; calls of zero or negative length end at or before their start
    in_s = np.zeros(n_nodes, np.int64)
    out_s = np.zeros(n_calls, np.int64)
    out_e = np.zeros(n_calls, np.int64)
    span = int(dur[roots].max()) + 1000
    for q, r in enumerate(roots):
        in_s[r] = 1_000_000 + q * span + int(rng.integers(0, 100))
    for x in range(n_nodes):
        for c in node_calls[x]:
            out_s[c] = in_s[x] + call_off[c]
            out_e[c] = out_s[c] + call_len[c]
            if call_child[c] >= 0:
                in_s[call_child[c]] = out_s[c] + child_off[c]
    in_e = in_s + dur
    for c, v in shrunk.items():
        out_e[c] = out_s[c] + v

    # 4. services and node ids
    keys = sorted(set(node_svc))
    n_callee = {k: (callees if k[0] == 0 else 1) for k in keys}
    if order == "root":
        keys.sort(key=lambda k: (k[0], k[1]))
    elif order == "leaf":
        keys.sort(key=lambda k: (-k[0], -k[1]))
    else:
        keys = [keys[i] for i in rng.permutation(len(keys))]
    members = {k: [] for k in keys}
    for x in range(n_nodes):
        members[node_svc[x]].append(x)
    if order == "shuffled":
        members = {k: [v[i] for i in rng.permutation(len(v))] for k, v in members.items()}
    node_id = np.zeros(n_nodes, np.int64)
    base = 0
    for k in keys:
        node_id[members[k]] = base + np.arange(len(members[k]))
        base += len(members[k])
    n_in = base
    # out-span lists: per (service, callee position) the calls in their callers' order
    out_lists = {(k, e): [] for k in keys for e in range(n_callee[k])}
    for k in keys:
        for x in members[k]:
            for c in node_calls[x]:
                out_lists[(k, call_pos[c])].append(c)
    call_id, call_j = np.zeros(n_calls, np.int64), np.zeros(n_calls, np.int64)
    base = 0
    for k in keys:
        for e in range(n_callee[k]):
            lst = out_lists[(k, e)]
            call_j[lst] = np.arange(len(lst))
            call_id[lst] = n_in + base + np.arange(len(lst))
            base += len(lst)
    problems, assign = [], []
    for k in keys:
        xs, E = members[k], n_callee[k]
        a = np.full((E, len(xs)), -1, np.int64)
        for i, x in enumerate(xs):
            for c in node_calls[x]:
                a[call_pos[c], i] = call_j[c]
        assign.append(a.reshape(-1))
        lst = [out_lists[(k, e)] for e in range(E)]
        problems.append(Problem(in_start=in_s[xs], in_end=in_e[xs], out_start=[out_s[v] for v in lst],
                                out_end=[out_e[v] for v in lst], preds=[[] for _ in range(E)],
                                name=f"{'spine' if k[0] == 0 else 'leaf'}{k[1]}"))
    in_caller = np.full(n_in, -1, np.int32)
    for c in range(n_calls):
        if call_child[c] >= 0:
            in_caller[node_id[call_child[c]]] = call_id[c]
    return dict(hb=build_batch(problems, validate=False), assign=np.concatenate(assign).astype(np.int32),
                in_caller=in_caller, roots=node_id[roots], depth=np.array(depths),
                open_calls=[call_id[f] for f in open_calls])


def _lay_out(rng, mode, cs, spine_call, off, length, gap, const_times, shrunk):
    """Offsets of the calls `cs` of one in-span from its start (off[c]), and the in-span's length; the
    calls made zero or negative go into `shrunk`."""
    order = list(cs) if const_times else [cs[i] for i in rng.permutation(len(cs))]
    if mode == "parallel" and spine_call in order:             # the spine call starts, and ends, last
        order.remove(spine_call)
        order.append(spine_call)
    if mode == "nested":
        box = max(order, key=lambda c: (length[c], c == spine_call))
        t = gap()
        off[box] = t
        t += int(length[box])
        for c in order:
            if c == box:
                continue
            if length[c] <= length[box] - 2:
                off[c] = off[box] + 1 + int(rng.integers(0, length[box] - length[c] - 1))
            else:
                off[c] = t
                t += int(length[c]) + gap()
        return t + gap()
    if mode == "parallel":
        t, end = gap(), 0
        for c in order:
            off[c] = t
            if c == spine_call and t + length[c] <= end:
                off[c] = end - length[c] + 1
            end = max(end, int(off[c] + length[c]))
            t = int(off[c]) + max(1, int(length[c]) // 2)
        return end + gap()
    t = gap()
    for c in order:
        off[c] = t
        t += int(length[c]) + gap()
    if mode == "clipped":                                     # a quarter of the first and last call outside
        off[order[0]] = -max(1, int(length[order[0]]) // 4)
        return t - gap() - max(1, int(length[order[-1]]) // 4)
    if mode in ("zero", "negative"):
        for c in order:
            if c != spine_call and rng.random() < 0.5:
                shrunk[c] = 0 if mode == "zero" else -int(rng.integers(1, 6))
    return t
