"""Pins the oracle's graph / mixer / scheduling semantics against the reference's integration tests
(the reference's tests/offline.rs).  Each test restates one reference `#[test]` (name + line cited)."""
import numpy as np
import pytest

RQ = 128


def ctx(pkg, oracle, ch, length, sr):
    return pkg.OfflineAudioContext(ch, length, sr, oracle)


def test_offline_render(pkg, oracle):
    # tests/offline.rs:10-46 test_offline_render: 2 + (-4) = -2 exactly, partial last quantum
    LENGTH = 555
    c = ctx(pkg, oracle, 2, LENGTH, 44100.0)
    c1 = c.create_constant_source()
    c1.offset.set_value(2.0)
    c1.connect(c.destination())
    c2 = c.create_constant_source()
    c2.offset.set_value(-4.0)
    c2.connect(c.destination())
    c1.start()
    c2.start()
    out = c.start_rendering_sync()
    assert out.number_of_channels() == 2 and out.length() == LENGTH
    assert np.array_equal(out.get_channel_data(0), np.full(LENGTH, -2.0, np.float32))
    assert np.array_equal(out.get_channel_data(1), np.full(LENGTH, -2.0, np.float32))


def test_start_stop(pkg, oracle):
    # tests/offline.rs:48-81 test_start_stop
    sr = 48000.0
    c = ctx(pkg, oracle, 1, RQ * 4, sr)
    osc = c.create_oscillator(type_=pkg.SQUARE, frequency=0.0)
    osc.connect(c.destination())
    osc.start_at(128.0 / sr)
    osc.stop_at(128.0 * 3.0 / sr)
    out = c.start_rendering_sync().get_channel_data(0)
    expected = np.concatenate([np.zeros(RQ), np.ones(2 * RQ), np.zeros(RQ)]).astype(np.float32)
    assert np.array_equal(out, expected)


def test_delayed_constant_source(pkg, oracle):
    # tests/offline.rs:83-112 test_delayed_constant_source
    sr = 48000.0
    c = ctx(pkg, oracle, 1, RQ * 4, sr)
    delay = c.create_delay(1.0)
    delay.delay_time.set_value(128.0 * 2.0 / sr)
    delay.connect(c.destination())
    src = c.create_constant_source()
    src.connect(delay)
    src.start()
    out = c.start_rendering_sync().get_channel_data(0)
    expected = np.concatenate([np.zeros(2 * RQ), np.ones(2 * RQ)]).astype(np.float32)
    assert np.abs(out - expected).max() <= 0.00001


def test_audio_param_graph(pkg, oracle):
    # tests/offline.rs:114-149 test_audio_param_graph: param intrinsic value + two audio-rate inputs
    c = ctx(pkg, oracle, 1, RQ, 48000.0)
    gain = c.create_gain()
    gain.gain.set_value(0.5)
    gain.connect(c.destination())
    source = c.create_constant_source()
    source.offset.set_value(0.8)
    source.connect(gain)
    p1 = c.create_constant_source()
    p1.offset.set_value(0.1)
    p1.connect(gain.gain)
    p2 = c.create_constant_source()
    p2.offset.set_value(0.3)
    p2.connect(gain.gain)
    source.start()
    p1.start()
    p2.start()
    out = c.start_rendering_sync().get_channel_data(0)
    expected = np.full(RQ, np.float32(0.8) * np.float32(0.9), np.float32)
    assert np.array_equal(out, expected)


def test_cycle(pkg, oracle):
    # tests/offline.rs:170-203 test_cycle: nodes in an unbroken cycle are muted
    c = ctx(pkg, oracle, 1, RQ, 48000.0)
    cycle1 = c.create_gain()
    cycle1.connect(c.destination())
    cycle2 = c.create_gain()
    cycle2.connect(cycle1)
    cycle1.connect(cycle2)
    source_cycle = c.create_constant_source()
    source_cycle.offset.set_value(1.0)
    source_cycle.connect(cycle1)
    other = c.create_constant_source()
    other.offset.set_value(2.0)
    other.connect(c.destination())
    source_cycle.start()
    other.start()
    out = c.start_rendering_sync().get_channel_data(0)
    assert np.array_equal(out, np.full(RQ, 2.0, np.float32))


def test_cycle_breaker(pkg, oracle):
    # tests/offline.rs:205-244 test_cycle_breaker: DelayNode breaks the cycle, feedback of 1 quantum
    sr = 48000.0
    c = ctx(pkg, oracle, 1, RQ * 3, sr)
    delay = c.create_delay(1.0 / sr)
    delay.delay_time.set_value(1.0 / sr)
    delay.connect(c.destination())
    delay.connect(delay)
    source = c.create_constant_source()
    source.offset.set_value(1.0)
    source.connect(delay)
    source.connect(c.destination())
    source.start()
    out = c.start_rendering_sync().get_channel_data(0)
    assert np.array_equal(out[:RQ], np.full(RQ, 1.0, np.float32))
    assert np.array_equal(out[RQ:2 * RQ], np.full(RQ, 2.0, np.float32))
    assert np.array_equal(out[2 * RQ:], np.full(RQ, 3.0, np.float32))


def test_render_order_matches_reference(pkg, builder):
    # src/render/graph.rs:443-479 + SURVEY §3.3: reverse post-order over ascending ids — the last-created
    # branch is processed first.  ids: dest 0; osc1 11 (+12,13); osc2 14 (+15,16)
    c = ctx(pkg, builder, 1, RQ, 48000.0)
    o1 = c.create_oscillator()
    o2 = c.create_oscillator()
    o1.connect(c.destination())
    o2.connect(c.destination())
    assert (o1.id, o2.id) == (11, 14)
    assert c.render_order() == [16, 15, 14, 13, 12, 11, 0]


def _gain_graph(pkg, be, n):
    """n + 1 plain nodes like the reference's graph tests: destination = 0, gains g[1..n] (each gain id is followed by its param)."""
    c = ctx(pkg, be, 1, RQ, 48000.0)
    nodes = [c.destination()] + [c.create_gain() for _ in range(n)]
    return c, nodes


def test_graph_order_add_remove(pkg, builder):  # src/render/graph.rs:659-706 test_add_remove
    c, n = _gain_graph(pkg, builder, 3)
    n[1].connect(n[0])
    n[2].connect(n[1])
    n[3].connect(n[0])
    order = c.render_order()
    ids = [x.id for x in n]
    assert all(i in order for i in ids) and order[-1] == 0  # all nodes present, the root comes last
    assert order.index(ids[2]) < order.index(ids[1])        # node 1 depends on node 2
    n[1].disconnect()                                       # detach node 1 (and thus node 2) from the root
    order = c.render_order()
    assert all(i in order for i in ids)
    assert order.index(ids[2]) < order.index(ids[1])


def test_graph_order_cycle_without_delay_is_muted(pkg, builder):  # src/render/graph.rs:708-741 test_cycle
    c, n = _gain_graph(pkg, builder, 4)
    n[4].connect(n[2])
    n[2].connect(n[1])
    n[1].connect(n[0])
    n[1].connect(n[2])
    n[3].connect(n[0])
    order = c.render_order()
    assert n[1].id not in order and n[2].id not in order    # the cycle 1 <> 2 is removed
    assert n[4].id in order                                 # the leg feeding the cycle is still rendered
    assert order.index(n[3].id) < order.index(0)            # the acyclic part is present


def test_graph_order_cycle_breaker(pkg, builder):  # src/render/graph.rs:458-479: a DelayWriter inside a cycle loses its outgoing edge
    c = ctx(pkg, builder, 1, RQ, 48000.0)
    src = c.create_constant_source()
    g = c.create_gain()
    d = c.create_delay(1.0, 0.5)
    src.connect(g)
    g.connect(d)
    d.connect(g)
    g.connect(c.destination())
    order = c.render_order()
    writer, reader = d.id, d.id + 1
    assert writer in order and reader in order and g.id in order
    # reader (the cycle's source after the break) -> gain -> writer; without the break the writer would precede the reader
    assert order.index(reader) < order.index(g.id) < order.index(writer)


def test_suspend_sync(pkg, oracle):
    # src/context/offline.rs:469-511 test_suspend_sync: a source created and started inside the first callback, disconnected
    # inside the second one
    sr = 48000.0
    c = ctx(pkg, oracle, 1, RQ * 4, sr)
    box = {}

    def first(context):
        src = context.create_constant_source()
        src.connect(context.destination())
        src.start_at(context.current_time())
        box["src"] = src

    c.suspend_sync(RQ / sr, first)
    c.suspend_sync(3 * RQ / sr, lambda context: box["src"].disconnect())
    out = c.start_rendering_sync().get_channel_data(0)
    assert np.array_equal(out[:RQ], np.zeros(RQ, np.float32))
    assert np.array_equal(out[RQ:3 * RQ], np.ones(2 * RQ, np.float32))
    assert np.array_equal(out[3 * RQ:], np.zeros(RQ, np.float32))


def test_suspend_argument_errors(pkg, oracle):
    # src/context/offline.rs:547-575: negative time, after the duration, twice at the same quantum
    for times in ([-1.0], [1.0], [0.0, 0.0]):
        c = ctx(pkg, oracle, 2, RQ, 44100.0)
        for t in times:
            c.suspend_sync(t, lambda context: None)
        with pytest.raises(pkg.WaeError):
            c.start_rendering_sync()
