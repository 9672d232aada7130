"""CPU test (`-m "not gpu"`): every launch plan of the engine, op by op, against digests recorded in
tests/golden/engine_plans.json (written by tests/golden/make_golden_engine_plans.py).

An op is serialised as its opcode, its 15 integer and 8 float slots, and each of its 16 pointer slots resolved to the
engine buffer it points into and the byte offset there ('P', 'G', 'act:<tensor>', 'grad:<tensor>', a metric buffer,
...); the two ctypes arrays a plan points to (the filter-transpose table and the L2 segments) are serialised with their
contents.  A slot that points into no buffer is an integer argument (a byte count, `nparams`, a bucket offset) and is
kept as that integer.  So two engines with equal digests launch the same kernels with the same arguments on buffers of
the same meaning, and a change of the engine's host code that keeps every digest cannot change what a step computes."""
import hashlib
import json
import os

import pytest

import step_oracle as so

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'engine_plans.json')

# the configurations of tests/step_oracle.py, plus the embedding head's variants that those do not reach
EXTRA = [
    ('resnet-110-fc', 8, 'tf32x3', dict(tag='cls_base', cls_weight=0.1, cls_base='avg_pool', nesterov=True)),
    ('resnet-110-fc', 8, 'f32', dict(tag='cls-world2', cls_weight=0.1, world_size=2, comm='torch')),
    ('simple', 16, 'tf32x3', dict(tag='world2', world_size=2, comm='torch', grad_buckets=4)),
]
# (name, set_trainable argument) applied in this order after the engine is built; each state is its own case
TRAINABLE = [('frozen', lambda name: name.split('/')[0] in ('embedding', 'prob', 'cls_bn')), ('thawed', None)]


def _buffers(eng):
    """(role, start address, size in bytes) of every buffer a plan may point into."""
    out = []

    def add(role, t):
        if t is not None and t.numel():
            out.append((role, t.data_ptr(), t.numel() * t.element_size()))

    for role in ('P', 'G', 'V', 'PT', 'PL', 'PTL', 'S', 'E', 'stats', 'saved', 'sgd_out', 'lr_dev', 'labels',
                 'loss_buf', 'acc_buf', 'rank_buf', 'cls_loss_buf', 'cls_acc_buf', 'cls_rank_buf', 'center_buf',
                 'le_work'):
        add(role, getattr(eng, role, None))
    for name, t in eng.act.items():               # eng.x is act[<input>]: one role only
        add('act:' + name, t)
    for name, t in eng.grad.items():
        add('grad:' + name, t)
    import ctypes
    out.append(('tr_table', ctypes.addressof(eng.tr_table), ctypes.sizeof(eng.tr_table)))
    out.append(('seg_array', ctypes.addressof(eng.seg_array), ctypes.sizeof(eng.seg_array)))
    return sorted(out, key=lambda r: r[1])


def _arrays(eng):
    return {'tr_table': list(eng.tr_table),
            'seg_array': [(s.begin, s.end, float(s.l2).hex()) for s in eng.seg_array]}


def serialise_plan(eng, plan):
    """One JSON line per op of `plan` (see the module docstring)."""
    import bisect
    bufs = _buffers(eng)
    starts = [b[1] for b in bufs]
    arrays = _arrays(eng)

    def resolve(v):
        if v is None:
            return None
        k = bisect.bisect_right(starts, v) - 1
        if k >= 0 and v < bufs[k][1] + bufs[k][2]:
            role = bufs[k][0]
            return [role, v - bufs[k][1]] + ([arrays[role]] if role in arrays else [])
        return v

    lines = []
    for o in plan:
        rec = [int(o.opcode), [int(v) for v in o.i], [float(v).hex() for v in o.f], [resolve(v) for v in o.p]]
        lines.append(json.dumps(rec, separators=(',', ':')))
    return lines


def cases():
    """(case id, config) of every configuration checked."""
    return [(so.config_id(c), c) for c in so.CONFIGS + EXTRA]


def case_plans(cfg):
    """{'<case>/<plan>': [op lines]} of one configuration: its plans as built, then after each TRAINABLE step."""
    eng = so.build_engine(cfg, device='cpu', use_cuda_graph=False)
    cid = so.config_id(cfg)
    out = {}
    states = [('', None)] + [('/' + name, fn) for name, fn in TRAINABLE]
    for k, (suffix, fn) in enumerate(states):
        if k:
            eng.set_trainable(fn)
        for pname in sorted(eng.plans):
            out[cid + suffix + '/' + pname] = serialise_plan(eng, eng.plans[pname])
    return out


def digest(lines):
    return {'ops': len(lines), 'sha256': hashlib.sha256('\n'.join(lines).encode()).hexdigest()}


@pytest.fixture(scope='module')
def golden():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize('cfg', [c for _, c in cases()], ids=[i for i, _ in cases()])
def test_plans_match_golden(golden, cfg):
    got = {k: digest(v) for k, v in case_plans(cfg).items()}
    want = {k: v for k, v in golden.items() if k.split('/')[0] == so.config_id(cfg)}
    assert want, 'no recorded plans for %s' % so.config_id(cfg)
    assert sorted(got) == sorted(want)
    bad = [k for k in sorted(got) if got[k] != want[k]]
    assert not bad, 'plans differ from the recorded ones: %s' % ', '.join(bad)
