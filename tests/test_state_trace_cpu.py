"""CPU: the expected-image model and the seeded update traces of test_state_trace_gpu.

A controller uploads its image once and then reconciles in a loop: it edits rows of the resident image
(wva_system_update_servers / _update_models / _remove_server / _set_capacity), sometimes changes the shard, and calls
Analyze and Optimize again.  The GPU tests replay such traces and compare every result with a witness context that
uploads the expected image from scratch, and with the oracle.  The expected image is kept here, in numpy, independently
of the binding's own mirror (Context.image), which the GPU tests check against it array by array.

  trace A  300 servers x 6 accelerators, T = 3: every kind of update, failed updates, a zero-row update, shards,
           capacities, removes down to an empty image and growth from it
  trace B  config 5's generator at S = 8190, A = 16 (sweep slices of 8192 servers at b_max = 512): an extension into a
           second slice, an overwrite across the slice boundary, removes back to one slice
"""
import numpy as np
import pytest

from test_sweep_slices_cpu import slice_plan

SRV_BYTES = 54                    # one server row: 13 arrays of 4 B + 2 of 1 B
PERF_BYTES = 29                   # one (model, accelerator) row: 7 x 4 B + 1 B
EINVAL, ECAPACITY = -1, -6


def spare(n):
    """rows wva_system_upload lays out for n rows: n + max(n / 16, 64)"""
    return n + max(n // 16, 64)


class Op:
    """one call of the trace: kind in servers / models / remove / removes / capacity / shard"""

    def __init__(self, tag, kind, first=0, rows=None, index=None, scale=None, code=0):
        self.tag, self.kind, self.first, self.rows, self.index, self.scale, self.code = tag, kind, first, rows, index, scale, code

    def count(self):
        return self.rows.M if self.kind == "models" else self.rows.S

    def __repr__(self):
        return "Op(%s)" % self.tag


# ---- the expected image: a numpy model of the four updates ------------------------------------------------------------

def copy_image(img):
    return img.shard(0, img.S)


def update_servers(wva, img, first, rows):
    """rows [first, first + rows.S) overwritten or appended (first <= S)"""
    out = copy_image(img)
    S = max(img.S, first + rows.S)
    for name, dt in wva.abi.SRV_FIELDS:
        a = np.zeros(S, dtype=dt)
        a[:img.S] = getattr(img, name)
        a[first:first + rows.S] = getattr(rows, name)
        setattr(out, name, a)
    out.S = S
    return out


def update_models(wva, img, first, rows):
    """perf rows of models [first, first + rows.M) overwritten or appended (first <= M)"""
    out = copy_image(img)
    M, A = max(img.M, first + rows.M), img.A
    for name, dt in wva.abi.PERF_FIELDS:
        a = np.zeros(M * A, dtype=dt)
        a[:img.M * A] = getattr(img, name)
        a[first * A:(first + rows.M) * A] = getattr(rows, name)
        setattr(out, name, a)
    out.M = M
    return out


def remove_server(wva, img, index):
    """RemoveServer: the last row moves into `index`"""
    keep = np.arange(img.S - 1)
    if index < img.S - 1:
        keep[index] = img.S - 1
    return img.take(keep)


def apply(wva, op, img, shard, caps):
    """(image, shard) after op; caps = (Scap, Mcap) of the upload.  A failing op changes nothing."""
    if op.code != 0:
        return img, shard
    if op.kind == "servers":
        return (update_servers(wva, img, op.first, op.rows), (0, max(img.S, op.first + op.rows.S))) if op.rows.S else (img, shard)
    if op.kind == "models":
        return (update_models(wva, img, op.first, op.rows), (0, img.S)) if op.rows.M else (img, shard)
    if op.kind in ("remove", "removes"):
        for i in np.atleast_1d(op.index):
            img = remove_server(wva, img, int(i))
        return img, (0, img.S)
    if op.kind == "capacity":
        out = copy_image(img)
        out.type_capacity = np.floor(img.type_capacity * op.scale).astype(np.int64)
        return out, shard
    if op.kind == "shard":
        return img, (op.first, op.index)
    raise ValueError(op.kind)


def expected_bytes(op, prev, A, T):
    """wva_upload_bytes after op (prev: before it)"""
    if op.code != 0 or op.kind == "shard":
        return prev
    if op.kind == "servers":
        return op.rows.S * SRV_BYTES
    if op.kind == "models":
        return op.rows.M * A * PERF_BYTES
    if op.kind == "capacity":
        return 8 * T
    return 0


def expected_code(op, img, caps):
    """the error wva_system_update_* returns for op on img, from the header's rules"""
    if op.kind == "servers":
        r = op.rows
        if op.first > img.S:
            return EINVAL
        if op.first + r.S > caps[0]:
            return ECAPACITY
        if (r.srv_model >= img.M).any() or (r.srv_cur_acc < -2).any() or (r.srv_cur_acc >= img.A).any():
            return EINVAL
        if ((r.srv_priority < 1) | (r.srv_priority > 100)).any():
            return EINVAL
    if op.kind == "models":
        if op.first > img.M:
            return EINVAL
        if op.first + op.rows.M > caps[1]:
            return ECAPACITY
    return 0


def touched(op, before, after, cap=24):
    """servers (indices into `after`) whose rows op wrote: written rows, slots a remove moved a row into, servers of edited
    models"""
    if op.code != 0:
        return []
    if op.kind == "servers":
        out = list(range(op.first, op.first + op.rows.S))
    elif op.kind == "models":
        m = after.srv_model
        out = list(np.flatnonzero((m >= op.first) & (m < op.first + op.rows.M)))
    elif op.kind in ("remove", "removes"):
        out, S = [], before.S
        for i in np.atleast_1d(op.index):
            S -= 1
            if i < S:
                out.append(int(i))
        out = [i for i in out if i < after.S]
    else:
        out = []
    return sorted(set(int(s) for s in out))[:cap]


def models_of(wva, img, ms):
    """a rows image holding the perf rows of models ms"""
    ms = np.asarray(ms, dtype=np.int64)
    out = wva.image.SystemImage(0, img.A, len(ms), img.T)
    idx = (ms[:, None] * img.A + np.arange(img.A)).reshape(-1)
    for name, _ in wva.abi.PERF_FIELDS:
        setattr(out, name, getattr(img, name)[idx].copy())
    return out


def empty_rows(wva, img):
    return wva.image.SystemImage(0, img.A, 0, img.T)


def all_fields_differ(wva, img, a, b):
    """every one of the 15 server fields of rows a and b differs"""
    return [name for name, _ in wva.abi.SRV_FIELDS if getattr(img, name)[a] == getattr(img, name)[b]]


class Builder:
    """appends ops to a trace while keeping the expected state, so that later ops can refer to it"""

    def __init__(self, wva, base):
        self.wva, self.img, self.shard = wva, base, (0, base.S)
        self.caps = (spare(base.S), spare(base.M))
        self.ops = []

    def add(self, op):
        op.code = expected_code(op, self.img, self.caps)
        self.ops.append(op)
        self.img, self.shard = apply(self.wva, op, self.img, self.shard, self.caps)
        return op

    def row(self, s):
        return self.img.take([s])


# ---- trace A ----------------------------------------------------------------------------------------------------------

A_S, A_A, A_T = 300, 6, 3
A_BIG = {17: 3200, 83: 3073}          # server overrides above 3072 on one accelerator each: tables in HBM
A_BATCHES = [1, 64, 512]


def trace_a_base(wva):
    img = wva.synth.make_system(A_S, A_A, seed=91, n_types=A_T, max_pair_batch=512)
    for s, n in A_BIG.items():
        img.srv_arrival_rpm[s] = max(img.srv_arrival_rpm[s], np.float32(600.0))
        img.srv_out_tokens[s] = max(img.srv_out_tokens[s], 64)
        img.srv_max_batch[s] = n
        m = img.srv_model[s]
        img.perf_valid[m * A_A:(m + 1) * A_A] = 0
        img.perf_valid[m * A_A + s % A_A] = 1
    img.type_capacity[:] = [60, 45, 30]
    return img


def _pick(img, pred, start):
    """first server >= start (cyclically) satisfying pred(s)"""
    for k in range(img.S):
        s = (start + k) % img.S
        if pred(s):
            return s
    raise AssertionError("no server fits")


def trace_a(wva):
    """(base image, ops) of trace A"""
    base = trace_a_base(wva)
    b = Builder(wva, base)
    A = base.A
    donor = wva.synth.make_system(40, A, seed=92, n_types=A_T, max_pair_batch=512)
    rng = np.random.default_rng(93)

    def donor_rows(k, models_below):
        r = donor.take(rng.choice(donor.S, k))
        r.srv_model[:] = rng.integers(0, models_below, k, dtype=np.int32)
        return r

    # overwrites and growth
    b.add(Op("overwrite_middle", "servers", 150, donor_rows(1, b.img.M)))
    b.add(Op("overlap_extend", "servers", 295, donor_rows(10, b.img.M)))            # 295 < S = 300 < 305
    # model edits: perf_valid 1 -> 0 on one accelerator and 0 -> 1 on another
    img = b.img
    pv = img.perf_valid.reshape(img.M, A)
    s = _pick(img, lambda s: img.srv_model[s] >= 0 and img.srv_arrival_rpm[s] > 0 and 0 < pv[img.srv_model[s]].sum() < A, 0)
    m = int(img.srv_model[s])
    r = models_of(wva, img, [m])
    a0, a1 = int(np.flatnonzero(pv[m] == 1)[0]), int(np.flatnonzero(pv[m] == 0)[0])
    r.perf_valid[a0], r.perf_valid[a1] = 0, 1
    b.add(Op("model_valid_flip", "models", m, r))
    # a server's N = max_batch * at_tokens / out_tokens crosses 3072 (shared-memory table -> HBM table), then back
    s = _pick(img, lambda s: img.srv_max_batch[s] == 0 and img.srv_arrival_rpm[s] > 0 and img.srv_out_tokens[s] >= 32
              and img.srv_model[s] >= 0 and (img.srv_model == img.srv_model[s]).sum() == 1, 60)
    m = int(img.srv_model[s])
    up = models_of(wva, img, [m])
    up.perf_max_batch[:] = 512
    up.perf_at_tokens[:] = (3400 * int(img.srv_out_tokens[s])) // 512 + 1
    b.add(Op("model_n_above_3072", "models", m, up))
    b.add(Op("model_n_back", "models", m, models_of(wva, img, [m])))
    # more models, then servers that use them
    M = b.img.M
    b.add(Op("model_extend", "models", M, models_of(wva, donor, [0, 1, 2, 3])))
    new = donor_rows(4, 1)
    new.srv_model[:] = np.arange(M, M + 4, dtype=np.int32)
    b.add(Op("servers_of_new_models", "servers", b.img.S, new))
    # server edits that change the table plan (hostN)
    s = _pick(b.img, lambda s: b.img.srv_arrival_rpm[s] > 0 and b.img.srv_out_tokens[s] > 0 and b.img.srv_model[s] >= 0, 30)
    r = b.row(s); r.srv_max_batch[0] = 3600
    b.add(Op("max_batch_above_3072", "servers", s, r))
    r = b.row(s); r.srv_max_batch[0] = 100
    b.add(Op("max_batch_below_3072", "servers", s, r))
    s = 17                                                       # an HBM-table server
    r = b.row(s); arrival = r.srv_arrival_rpm[0]; r.srv_arrival_rpm[0] = 0.0
    b.add(Op("arrival_zero", "servers", s, r))
    r = b.row(s); r.srv_arrival_rpm[0] = arrival
    b.add(Op("arrival_back", "servers", s, r))
    r = b.row(83); r.srv_out_tokens[0] = 0
    b.add(Op("out_tokens_zero", "servers", 83, r))
    # current allocations
    s = _pick(b.img, lambda s: b.img.srv_cur_acc[s] >= 0 and b.img.srv_arrival_rpm[s] > 0, 40)
    r = b.row(s); r.srv_cur_acc[0] = wva.abi.ACC_UNKNOWN
    b.add(Op("cur_acc_unknown", "servers", s, r))
    s = _pick(b.img, lambda s: b.img.srv_cur_acc[s] >= 0 and b.img.srv_arrival_rpm[s] > 0, 50)
    r = b.row(s); r.srv_cur_acc[0] = wva.abi.ACC_NONE; r.srv_cur_replicas[0] = 0; r.srv_cur_cost[0] = 0.0
    b.add(Op("cur_acc_none", "servers", s, r))
    s = _pick(b.img, lambda s: b.img.srv_cur_acc[s] >= 0 and b.img.srv_arrival_rpm[s] > 0, 70)
    r = b.row(s); r.srv_keep_acc[0] = 1 - r.srv_keep_acc[0]
    b.add(Op("keep_acc_toggle", "servers", s, r))
    b.add(Op("capacity", "capacity", scale=0.5))
    # a shard, and updates that fail while it is set (each leaves everything as it was), a zero-row update
    b.add(Op("shard", "shard", 40, index=200))
    r = b.img.take([10, 11, 12]); r.srv_model[2] = b.img.M
    b.add(Op("fail_model_last_row", "servers", 10, r))
    r = b.row(20); r.srv_priority[0] = 0
    b.add(Op("fail_priority", "servers", 20, r))
    r = b.row(21); r.srv_cur_acc[0] = A
    b.add(Op("fail_cur_acc", "servers", 21, r))
    b.add(Op("fail_first_beyond_S", "servers", b.img.S + 1, b.row(0)))
    b.add(Op("fail_models_beyond_M", "models", b.img.M + 1, models_of(wva, b.img, [0])))
    b.add(Op("zero_rows_servers", "servers", 5, b.img.take([])))
    b.add(Op("zero_rows_models", "models", 5, empty_rows(wva, b.img)))
    b.add(Op("update_under_shard", "servers", 100, donor_rows(2, b.img.M)))
    b.add(Op("shard_again", "shard", 0, index=b.img.S - 7))
    # removes: the last row differs from row 0 in all 15 fields, then row 0 is removed
    img = b.img
    r = b.row(0)
    r.srv_model[0] = (r.srv_model[0] + 1) % img.M
    r.srv_arrival_rpm[0] = r.srv_arrival_rpm[0] * np.float32(1.5) + np.float32(10.0)
    r.srv_in_tokens[0] += 7; r.srv_out_tokens[0] += 3
    r.srv_slo_ttft[0] *= np.float32(1.5); r.srv_slo_itl[0] *= np.float32(1.5); r.srv_slo_tps[0] += np.float32(100.0)
    r.srv_target_valid[0] = 1 - r.srv_target_valid[0]
    r.srv_priority[0] = 1 + r.srv_priority[0] % 100
    r.srv_min_replicas[0] = 1 - min(r.srv_min_replicas[0], 1)
    r.srv_max_batch[0] = 200 if r.srv_max_batch[0] != 200 else 300
    r.srv_keep_acc[0] = 1 - r.srv_keep_acc[0]
    r.srv_cur_acc[0] = (r.srv_cur_acc[0] + 1) % A if r.srv_cur_acc[0] >= 0 else 2
    r.srv_cur_replicas[0] += 2; r.srv_cur_cost[0] += np.float32(11.5)
    b.add(Op("last_row_all_differ", "servers", img.S - 1, r))
    b.add(Op("remove_first", "remove", index=0))
    b.add(Op("remove_middle", "remove", index=b.img.S // 2))
    b.add(Op("remove_last", "remove", index=b.img.S - 1))
    # growth to exactly Scap, then one row too many
    b.add(Op("extend_to_scap", "servers", b.img.S, donor_rows(b.caps[0] - b.img.S, b.img.M)))
    b.add(Op("fail_ecapacity", "servers", b.img.S, donor_rows(1, b.img.M)))
    b.add(Op("capacity_again", "capacity", scale=1.5))
    b.add(Op("remove_half", "removes", index=[(k * 7) % (b.img.S - k) for k in range(b.img.S // 2)]))
    b.add(Op("remove_to_empty", "removes", index=[(k * 5) % (b.img.S - k) for k in range(b.img.S)]))
    b.add(Op("grow_from_empty", "servers", 0, donor_rows(20, b.img.M)))
    b.add(Op("overwrite_after_growth", "servers", 3, donor_rows(4, b.img.M)))
    return base, b.ops, b.caps


# ---- trace B ----------------------------------------------------------------------------------------------------------

B_S, B_R, B_B = 8190, 8, 512
B_REMOVES = [8199, 3, 8190, 4000, 8195, 0, 8100, 8192]


def trace_b(wva):
    """(base image, ops) of trace B: config 5's generator at S = 8190"""
    base, _ = wva.synth.baseline_config(5, n_servers=B_S)
    base.type_capacity[:] = 400
    b = Builder(wva, base)
    donor = wva.synth.make_system(40, base.A, seed=95, n_types=base.T)
    rng = np.random.default_rng(96)

    def rows(k):
        r = donor.take(rng.choice(donor.S, k, replace=False))
        r.srv_model[:] = rng.integers(0, base.M, k, dtype=np.int32)
        return r

    b.add(Op("extend_into_second_slice", "servers", B_S, rows(10)))
    b.add(Op("overwrite_across_boundary", "servers", 8185, rows(11)))
    b.add(Op("removes_to_one_slice", "removes", index=B_REMOVES))
    return base, b.ops, b.caps


# ---- tests --------------------------------------------------------------------------------------------------------------

def _tiny(wva, S=5):
    img = wva.synth.make_system(S, 2, seed=97, n_types=2)
    img.srv_in_tokens[:] = np.arange(S, dtype=np.int32) + 100        # a row id
    return img


def test_model_remove_moves_the_last_row(wva):
    img = _tiny(wva)
    out = remove_server(wva, img, 1)
    assert out.S == 4 and list(out.srv_in_tokens) == [100, 104, 102, 103]
    out = remove_server(wva, out, 3)                                  # the last row: nothing moves
    assert list(out.srv_in_tokens) == [100, 104, 102]
    for name, _ in wva.abi.SRV_FIELDS:
        assert getattr(out, name)[1] == getattr(img, name)[4], name
    assert out.perf_alpha.tobytes() == img.perf_alpha.tobytes()


def test_model_overlap_extend(wva):
    img = _tiny(wva)
    rows = _tiny(wva, 3)
    rows.srv_in_tokens[:] = [7, 8, 9]
    out = update_servers(wva, img, 3, rows)
    assert out.S == 6 and list(out.srv_in_tokens) == [100, 101, 102, 7, 8, 9]
    assert out.srv_model[5] == rows.srv_model[2] and img.S == 5          # the input is left as it was
    out = update_servers(wva, out, 6, rows.take([0]))                 # first == S: append
    assert out.S == 7 and out.srv_in_tokens[6] == 7
    m = models_of(wva, img, [4, 0])
    out = update_models(wva, out, 4, m)
    assert out.M == 6 and out.perf_alpha[4 * 2:6 * 2].tobytes() == m.perf_alpha.tobytes()
    assert out.perf_alpha[:8].tobytes() == img.perf_alpha[:8].tobytes()


def test_model_remove_to_empty_and_grow(wva):
    img = _tiny(wva)
    for i in [0, 3, 1, 1, 0]:
        img = remove_server(wva, img, i)
    assert img.S == 0 and all(len(getattr(img, n)) == 0 for n, _ in wva.abi.SRV_FIELDS)
    out = update_servers(wva, img, 0, _tiny(wva, 2))
    assert out.S == 2 and list(out.srv_in_tokens) == [100, 101]


def test_apply_keeps_shard_and_image_on_failures(wva):
    img = _tiny(wva)
    caps = (spare(5), spare(5))
    bad = _tiny(wva, 1); bad.srv_priority[0] = 0
    op = Op("x", "servers", 2, bad)
    assert expected_code(op, img, caps) == EINVAL
    op.code = EINVAL
    assert apply(wva, op, img, (1, 2), caps) == (img, (1, 2))
    zero = Op("z", "servers", 2, img.take([]))
    assert expected_code(zero, img, caps) == 0 and apply(wva, zero, img, (1, 2), caps) == (img, (1, 2))
    assert expected_bytes(zero, 99, 2, 2) == 0 and expected_bytes(op, 99, 2, 2) == 99


TRACE_A_CLASSES = {
    "overwrite_middle", "overlap_extend", "extend_to_scap", "fail_ecapacity", "remove_first", "remove_middle",
    "remove_last", "remove_to_empty", "grow_from_empty", "last_row_all_differ", "model_valid_flip", "model_n_above_3072",
    "model_n_back", "model_extend", "servers_of_new_models", "max_batch_above_3072", "arrival_zero", "arrival_back",
    "out_tokens_zero", "cur_acc_unknown", "cur_acc_none", "keep_acc_toggle", "capacity", "shard", "update_under_shard",
    "fail_model_last_row", "fail_priority", "fail_cur_acc", "fail_first_beyond_S", "zero_rows_servers", "zero_rows_models",
}


def test_trace_a_has_every_operation_class(wva):
    base, ops, caps = trace_a(wva)
    tags = [op.tag for op in ops]
    assert TRACE_A_CLASSES <= set(tags) and len(ops) >= 35
    img, shard = base, (0, base.S)
    states = []
    for op in ops:
        states.append((op, img, shard))
        img, shard = apply(wva, op, img, shard, caps)
    by = {op.tag: (op, img, shard) for op, img, shard in states}
    # the overlap really extends, the growth ends exactly at Scap, the next row fails with ECAPACITY
    op, img, _ = by["overlap_extend"]
    assert op.first < img.S < op.first + op.rows.S
    op, img, _ = by["extend_to_scap"]
    assert op.code == 0 and op.first + op.rows.S == caps[0] == spare(A_S)
    op, img, _ = by["fail_ecapacity"]
    assert op.code == ECAPACITY and img.S == caps[0]
    # the four failing rows, each for its own reason; the model error sits in the last row
    assert [by[t][0].code for t in ("fail_model_last_row", "fail_priority", "fail_cur_acc", "fail_first_beyond_S",
                                    "fail_models_beyond_M")] == [EINVAL] * 5
    op, img, shard = by["fail_model_last_row"]
    assert (op.rows.srv_model[:-1] < img.M).all() and op.rows.srv_model[-1] >= img.M and shard != (0, img.S)
    # the remove of row 0 moves a row that differs from it in all 15 fields
    op, img, _ = by["remove_first"]
    assert op.index == 0 and all_fields_differ(wva, img, 0, img.S - 1) == []
    assert by["remove_middle"][0].index < by["remove_middle"][1].S - 1
    assert by["remove_last"][0].index == by["remove_last"][1].S - 1
    # removes down to an empty image, growth from it
    assert by["grow_from_empty"][1].S == 0 and by["grow_from_empty"][0].first == 0
    # the model edits: 1 -> 0 and 0 -> 1 on one model, N across 3072 and back
    op, img, _ = by["model_valid_flip"]
    old = img.perf_valid.reshape(img.M, img.A)[op.first]
    assert ((old == 1) & (op.rows.perf_valid == 0)).any() and ((old == 0) & (op.rows.perf_valid == 1)).any()
    op, img, _ = by["model_n_above_3072"]
    srv = np.flatnonzero(img.srv_model == op.first)
    assert len(srv) == 1 and img.srv_max_batch[srv[0]] == 0
    n = op.rows.perf_max_batch.astype(np.int64) * op.rows.perf_at_tokens // img.srv_out_tokens[srv[0]]
    n0 = (img.perf_max_batch.reshape(img.M, img.A)[op.first].astype(np.int64) *
          img.perf_at_tokens.reshape(img.M, img.A)[op.first] // img.srv_out_tokens[srv[0]])
    assert (n > 3072).all() and (n0 <= 3072).all()
    op, img, _ = by["servers_of_new_models"]
    assert (op.rows.srv_model >= by["model_extend"][1].M).all()
    # HBM tables exist in the base image (server overrides above 3072 on loaded servers)
    assert all(base.srv_max_batch[s] > 3072 and base.srv_arrival_rpm[s] > 0 for s in A_BIG)


def test_trace_b_crosses_slice_boundaries(wva):
    base, ops, caps = trace_b(wva)
    assert caps == (spare(B_S), spare(B_S))
    img, shard = base, (0, base.S)
    assert len(slice_plan(img.S, img.A, B_B)) == 1
    sizes = []
    for op in ops:
        assert op.code == 0
        img, shard = apply(wva, op, img, shard, caps)
        sizes.append(len(slice_plan(img.S, img.A, B_B)))
    assert slice_plan(8200, 16, B_B)[0] == (0, 8192)
    assert [op.tag for op in ops] == ["extend_into_second_slice", "overwrite_across_boundary", "removes_to_one_slice"]
    assert ops[1].first < 8192 < ops[1].first + ops[1].rows.S
    assert sizes == [2, 2, 1] and img.S == 8192
