"""The contract every wae_batch_bind_* shares, checked kind by kind through the raw C entry points on a tiny batch: the status of an empty
call and of a null batch, of an unknown graph or node, of a name given twice and of a bad pointer; all-or-nothing validation; runs that
wait for the declarations until they are bound; and declarations the planner never reached, which bind without writing anything and do
not hold up runs."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SR = 48000.0
FRAMES = 1024
N_GRAPHS = 2


# Per kind: the graph (returns the declared node and param index, and a declaration the planner never reaches or None), the element
# type and count an item reads, its binding struct and its bind entry point.
def sources_graph(pkg, c):
    s = c.create_buffer_source()
    s.set_device_input(1, 256, SR)
    s.connect(c.destination())
    s.start()
    idle = c.create_buffer_source()  # never started: renders silence without reading its buffer
    idle.set_device_input(1, 256, SR)
    idle.connect(c.destination())
    return (s.id, None), (idle.id, None)


def params_graph(pkg, c):
    o = c.create_oscillator()
    g = c.create_gain()
    g.gain.set_device_value()
    o.connect(g)
    g.connect(c.destination())
    o.start()
    return (g.gain._node, g.gain._index), None


def responses_graph(pkg, c):
    s = c.create_buffer_source(pkg.AudioBuffer([np.full(FRAMES, 0.25, np.float32)], SR))
    cv = c.create_convolver()
    cv.set_device_response(1, 256, SR)
    s.connect(cv)
    cv.connect(c.destination())
    s.start()
    return (cv.id, None), None


def curves_graph(pkg, c):
    o = c.create_oscillator()
    sh = c.create_wave_shaper()
    sh.set_device_curve(16)
    o.connect(sh)
    sh.connect(c.destination())
    o.start()
    return (sh.id, None), None


def waves_graph(pkg, c):
    o = c.create_oscillator()
    o.set_device_periodic_wave(4, 64)
    o.connect(c.destination())
    o.start()
    return (o.id, None), None


def iirs_graph(pkg, c):
    o = c.create_oscillator()
    f = c.create_iir_filter([1.0, 0.0, 0.0], [1.0, 0.0, 0.0])
    f.set_device_coefficients()
    o.connect(f)
    f.connect(c.destination())
    o.start()
    return (f.id, None), None


def value_curves_graph(pkg, c):
    o = c.create_oscillator()
    g = c.create_gain()
    g.gain.set_device_value_curve(16, 0.0, 0.01)
    o.connect(g)
    g.connect(c.destination())
    o.start()
    a, b = c.create_gain(), c.create_gain()  # a cycle without a DelayNode: muted, its params never lowered
    a.connect(b)
    b.connect(a.gain)
    a.connect(c.destination())
    a.gain.set_device_value_curve(16, 0.0, 0.01)
    return (g.gain._node, g.gain._index), (a.gain._node, a.gain._index)


def schedules_graph(pkg, c):
    o = c.create_oscillator()
    o.connect(c.destination())
    o.start_at(0.0)
    o.set_device_schedule((0.0, 1.0), stop=(0.5, 1.0))
    return (o.id, None), None


KINDS = {
    "sources": (sources_graph, "float32", 256,
                lambda B, g, node, index, p: B.SourceBinding(g, node, C.cast(C.c_void_p(p), B.c_float_p), 256),
                "SourceBinding", "bind_sources"),
    "params": (params_graph, "float32", 1, lambda B, g, node, index, p: B.ParamBinding(g, node, index, C.cast(C.c_void_p(p), B.c_float_p)),
               "ParamBinding", "bind_params"),
    "responses": (responses_graph, "float32", 256,
                  lambda B, g, node, index, p: B.ResponseBinding(g, node, C.cast(C.c_void_p(p), B.c_float_p), 256),
                  "ResponseBinding", "bind_responses"),
    "curves": (curves_graph, "float32", 16, lambda B, g, node, index, p: B.CurveBinding(g, node, C.cast(C.c_void_p(p), B.c_float_p)),
               "CurveBinding", "bind_curves"),
    "waves": (waves_graph, "float32", 4,
              lambda B, g, node, index, p: B.PeriodicWaveBinding(g, node, C.cast(C.c_void_p(p), B.c_float_p), None),
              "PeriodicWaveBinding", "bind_periodic_waves"),
    "iirs": (iirs_graph, "float64", 3,
             lambda B, g, node, index, p: B.IirBinding(g, node, C.cast(C.c_void_p(p), B.c_double_p), C.cast(C.c_void_p(p), B.c_double_p)),
             "IirBinding", "bind_iir_coefficients"),
    "value_curves": (value_curves_graph, "float32", 16,
                     lambda B, g, node, index, p: B.ValueCurveBinding(g, node, index, C.cast(C.c_void_p(p), B.c_float_p)),
                     "ValueCurveBinding", "bind_value_curves"),
    "schedules": (schedules_graph, "float64", 2,
                  lambda B, g, node, index, p: B.ScheduleBinding(g, node, C.cast(C.c_void_p(p), B.c_double_p)),
                  "ScheduleBinding", "bind_schedules"),
}


def setup(pkg, engine, kind):
    torch = pytest.importorskip("torch")
    graph, dtype, count, make, struct, bind = KINDS[kind]
    made = []
    for _ in range(N_GRAPHS):
        c = pkg.OfflineAudioContext(1, FRAMES, SR, engine.backend)
        made.append((c,) + graph(pkg, c))
    b = pkg.Batch([m[0] for m in made])
    (node, index), never = made[0][1], made[0][2]
    # one row per graph; an IIR item reads both of its pointers from the row ([1, 0, 0]: a pass-through)
    rows = torch.zeros((N_GRAPHS, count), dtype=getattr(torch, dtype), device="cuda")
    rows[:, 0] = 1.0 if kind == "iirs" else 0.5
    torch.cuda.synchronize()
    B = pkg._binding
    fn = getattr(pkg.api(), "batch_" + bind)

    def raw(items, null_items=False):
        arr = None if null_items else (getattr(B, struct) * max(len(items), 1))(*[make(B, g, nd, ix, p) for g, nd, ix, p in items])
        return fn(b.handle, arr, len(items), None)
    return torch, b, rows, node, index, never, raw, fn, "wae_batch_" + bind


@pytest.mark.parametrize("kind", list(KINDS))
def test_bind_contract(pkg, engine, kind):
    torch, b, rows, node, index, never, raw, fn, bind = setup(pkg, engine, kind)
    row = rows.element_size() * rows.shape[1]
    p0, p1 = rows.data_ptr(), rows.data_ptr() + row
    assert raw([], null_items=True) == 0                                    # n = 0, null items
    assert fn(None, None, 0, None) == 1                                     # null batch
    assert raw([(N_GRAPHS, node, index, p0)]) == 2                           # graph index out of range
    assert raw([(0, node + 1000, index, p0)]) == 2                          # a node with no declaration
    assert raw([(0, node, index, p0), (0, node, index, p0)]) == 1           # named twice
    assert raw([(0, node, index, 0)]) == 1                                  # null pointer
    host = np.zeros(rows.shape[1], rows.cpu().numpy().dtype)
    assert raw([(0, node, index, host.ctypes.data)]) == 1                   # host (numpy) memory
    seg = next(x for x in torch.cuda.memory_snapshot() if x["address"] <= p0 < x["address"] + x["total_size"])
    end = seg["address"] + seg["total_size"]
    if rows.shape[1] > 1:  # (a param's value is one float: a pointer past the end of its allocation is not in it)
        assert raw([(0, node, index, end - row + rows.element_size())]) == 1  # extent past the end of the allocation
    assert raw([(0, node, index, p0), (1, node, index, host.ctypes.data)]) == 1  # all-or-nothing: the good item is not bound
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and bind in e.value.message
    assert raw([(0, node, index, p0), (1, node, index, p1)]) == 0
    b.run()                                                                 # a never-reached declaration does not hold it up
    b.sync()
    got = b.fetch()
    if never is not None:
        assert raw([(0, never[0], never[1], p0), (1, never[0], never[1], p1)]) == 0  # validated, nothing written
        b.run()
        b.sync()
        assert np.array_equal(b.fetch(), got)


@pytest.mark.parametrize("kind", list(KINDS))
def test_bind_contract_misaligned(pkg, engine, kind):
    """a pointer 2 bytes past a valid allocation's start is refused before it reaches a kernel: 4-byte alignment for floats, 8 for doubles"""
    torch, b, rows, node, index, never, raw, fn, bind = setup(pkg, engine, kind)
    assert raw([(0, node, index, rows.data_ptr() + 2)]) == 1
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2
