"""ConvolverNode responses bound from device memory (wae_convolver_set_device_response + wae_batch_bind_responses) on the GPU.  A batch
is planned once and run with responses bound from torch tensors; each render is compared with the oracle's render of the same graphs
given the same responses through set_buffer (1e-5), and, where trimming does not cross a partition, with the engine's own render of
such graphs (bit-equal: the scale and the spectra are computed with the same operations)."""
import ctypes as C

import numpy as np
import pytest

import graphs as G
from test_device_responses_cpu import BLOCK, conv_graph, full_ir

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = G.SR


def tensor(torch, arrays):
    return torch.from_numpy(np.ascontiguousarray(np.stack(arrays).astype(np.float32))).cuda()


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def bound_render(pkg, engine, build, irs, batch=None):
    """build(backend, g, ir) -> (context, convolver); ir None = declared.  Binds irs[g] to graph g (one call), runs -> ([n][ch][len],
    (batch, convolver))"""
    torch = pytest.importorskip("torch")
    if batch is None:
        made = [build(engine.backend, g, None) for g in range(len(irs))]
        batch = (pkg.Batch([c for c, _ in made]), made[0][1])
    b, cv = batch
    b.bind_responses(cv, tensor(torch, irs))
    b.run()
    b.sync()
    return b.fetch(), batch


def check_oracle(pkg, engine, oracle, build, irs, tol=TOL, bit_equal=False):
    got, batch = bound_render(pkg, engine, build, irs)
    want = G.render(pkg, [build(oracle, g, list(irs[g]))[0] for g in range(len(irs))])
    assert np.isfinite(want).all()
    err = maxdiff(got, want)
    assert err <= tol, err
    if bit_equal:
        twin = G.render(pkg, [build(engine.backend, g, list(irs[g]))[0] for g in range(len(irs))])
        assert np.array_equal(got, twin)
    return got, batch


# ---------------------------------------------------------------------------------------------------------- routings and shapes
@pytest.mark.parametrize("normalize", [True, False], ids=["normalize", "raw"])
@pytest.mark.parametrize("ir_ch", [1, 2, 4])
@pytest.mark.parametrize("in_ch", [1, 2])
def test_routings(pkg, engine, oracle, in_ch, ir_ch, normalize):
    length, n_ir = 3 * BLOCK + 500, 20000
    irs = [np.stack(full_ir(ir_ch, n_ir, seed=10 + g)) * np.float32(1.0 if normalize else 0.01) for g in range(3)]  # (raw: outputs of order 1)

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, ir_ch, n_ir, ir=ir, in_ch=in_ch, normalize=normalize)
    check_oracle(pkg, engine, oracle, build, irs, bit_equal=True)


def test_long_synthetic_rir(pkg, engine, oracle):
    """C4's response length: 178 899 frames, 22 partitions, normalised"""
    length, n_ir = 200000, 178899
    irs = [np.stack(G.synthetic_ir(n_ir, 2, seed=99 + g)) for g in range(2)]

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 2, n_ir, ir=ir)
    check_oracle(pkg, engine, oracle, build, irs)


def test_tail_straddles_the_trim_threshold(pkg, engine, oracle):
    """the scaled tail runs around 1e-6 and below it over more than a partition: trimming decides where the response ends, per
    channel, and the spectra past it are zero"""
    length, n_ir = 4 * BLOCK, 3 * BLOCK + 100
    rng = np.random.default_rng(5)
    irs = []
    for g in range(3):
        ir = rng.uniform(-0.003, 0.003, (2, n_ir)).astype(np.float32)
        cut = [BLOCK + 700 + 900 * g, 2 * BLOCK - 5 + g]
        for c in range(2):
            tail = n_ir - cut[c]
            ir[c, cut[c]:] = rng.uniform(-9e-7, 9e-7, tail).astype(np.float32)  # below the threshold ...
            ir[c, cut[c] - 1] = np.float32(1.2e-6)                              # ... just above it right before
            ir[c, cut[c] + 7] = np.float32(-1e-6)                               # exactly the threshold is not below it: kept
        irs.append(ir)

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 2, n_ir, ir=ir, normalize=False)
    check_oracle(pkg, engine, oracle, build, irs)


def test_all_zero_response(pkg, engine, oracle):
    length, n_ir = 2 * BLOCK, 12000
    irs = [np.zeros((2, n_ir), np.float32) for _ in range(2)]

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 2, n_ir, ir=ir)
    got, _ = check_oracle(pkg, engine, oracle, build, irs)
    assert not got.any()


def test_source_that_stops(pkg, engine, oracle):
    """the tail counter runs on the declared length, not the trimmed one: the output ends where a response of that length has run out"""
    length, n_ir = 6 * BLOCK, 2 * BLOCK + 333
    irs = [np.stack(full_ir(2, n_ir, seed=40 + g)) for g in range(3)]
    for ir in irs:
        ir[:, 9000:] = 0.0  # (trimmed to 9000 frames)

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 2, n_ir, ir=ir, stop=5000 + 1000 * g)
    got, _ = check_oracle(pkg, engine, oracle, build, irs)
    assert not got[0, :, 5000 + n_ir + 256:].any() and got[0, :, 5000:5000 + 9000].any()


def test_mono_response_behind_a_switching_input(pkg, engine, oracle):
    length, n_ir = 4 * BLOCK + 500, 17000
    irs = [np.stack(full_ir(1, n_ir, seed=50 + g)) for g in range(3)]

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 1, n_ir, ir=ir, layout="switch")
    check_oracle(pkg, engine, oracle, build, irs, bit_equal=True)


@pytest.mark.parametrize("k", [1, 2])
def test_suspend_point_after_declaration(pkg, engine, oracle, k):
    length, n_ir = 4 * BLOCK, 20000
    irs = [np.stack(full_ir(2, n_ir, seed=60 + g)) for g in range(2)]

    def build(be, g, ir):
        c, cv = conv_graph(pkg, be, g, length, 2, n_ir, ir=ir)
        c.suspend_sync(k * BLOCK / SR, lambda ctx: None)
        return c, cv
    check_oracle(pkg, engine, oracle, build, irs, bit_equal=True)


def test_non_finite_samples(pkg, engine):
    """NaN and inf take part in the power (the scale then falls back to the floor) and NaN is not trimmed: the render equals the
    engine's render of the same responses given to set_buffer"""
    torch = pytest.importorskip("torch")
    length, n_ir = 2 * BLOCK, 9000
    irs = [np.stack(full_ir(2, n_ir, seed=70 + g)) for g in range(3)]
    irs[0][0, -1] = np.nan
    irs[1][1, 100] = np.inf
    irs[2][:, 4000:] = 0.0
    irs[2][1, 8999] = np.nan

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 2, n_ir, ir=ir)
    got, _ = bound_render(pkg, engine, build, irs)
    twin = G.render(pkg, [build(engine.backend, g, list(irs[g]))[0] for g in range(3)])
    assert np.array_equal(got, twin, equal_nan=True)


# ---------------------------------------------------------------------------------------------------------- binding
def test_rebinding_returns_to_the_first_output(pkg, engine, oracle):
    length, n_ir = 3 * BLOCK, 20000
    A = [np.stack(full_ir(2, n_ir, seed=80 + g)) for g in range(3)]
    Bs = [np.stack(G.synthetic_ir(n_ir, 2, seed=90 + g)) for g in range(3)]

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 2, n_ir, ir=ir)
    out_a, batch = check_oracle(pkg, engine, oracle, build, A)
    out_b, _ = bound_render(pkg, engine, build, Bs, batch)
    want_b = G.render(pkg, [build(oracle, g, list(Bs[g]))[0] for g in range(3)])
    assert maxdiff(out_b, want_b) <= TOL
    again, _ = bound_render(pkg, engine, build, A, batch)
    assert np.array_equal(again, out_a)


def c4_declared(pkg, be, g, length, n_ir, ir=None, pcm=None):
    """C4's graph with its source bound from device memory (pcm None) and its response declared (ir None)."""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    src = c.create_buffer_source()
    if pcm is None:
        src.set_device_input(2, length, SR)
    else:
        src.set_buffer(pkg.AudioBuffer(list(pcm), SR))
    cv = c.create_convolver()
    if ir is None:
        cv.set_device_response(2, n_ir, SR)
    else:
        cv.set_buffer(pkg.AudioBuffer(list(ir), SR))
    src.connect(cv)
    cv.connect(c.destination())
    src.start()
    return c, src, cv


def c4_pcm(g, length):
    rng = np.random.default_rng(4000 + g)
    pcm = (rng.uniform(-1.0, 1.0, (2, length)) * 0.05).astype(np.float32)
    pcm[:, :4096] += rng.uniform(-0.5, 0.5, (2, 4096)).astype(np.float32)
    return pcm


def test_many_c4_graphs_from_one_tensor(pkg, engine, oracle):
    """128 C4-shaped graphs, each with its own response, all from one tensor, the sources bound from device memory too; rendered by
    run, run_group and run_pipelined"""
    torch = pytest.importorskip("torch")
    n, length, n_ir = 128, 3 * BLOCK + 100, 2 * BLOCK + 77
    pcms = [c4_pcm(g, length) for g in range(n)]
    irs = [np.stack(G.synthetic_ir(n_ir, 2, seed=1000 + g)) for g in range(n)]
    made = [c4_declared(pkg, engine.backend, g, length, n_ir) for g in range(n)]
    b = pkg.Batch([c for c, _, _ in made])
    b.bind_sources(made[0][1], tensor(torch, pcms))
    b.bind_responses(made[0][2], tensor(torch, irs))
    b.run()
    b.sync()
    got = b.fetch()
    check = [0, 1, 63, 127]
    want = G.render(pkg, [c4_declared(pkg, oracle, g, length, n_ir, irs[g], pcms[g])[0] for g in check])
    assert maxdiff(got[check], want) <= TOL
    twin = pkg.Batch([c4_declared(pkg, engine.backend, g, length, n_ir, irs[g], pcms[g])[0] for g in range(n)])
    twin.run()
    twin.sync()
    assert np.array_equal(got, twin.fetch())  # (no partition trimmed: bit-equal)
    for k in range(len(b.groups())):
        b.run_group(k)
    b.sync()
    assert np.array_equal(b.fetch(), got)
    out = torch.empty((n, 2, length), dtype=torch.float32, pin_memory=True)
    b.run_pipelined(out.data_ptr())
    assert np.array_equal(out.numpy(), got)


def test_ordering_after_a_torch_kernel(pkg, engine, oracle):
    """the response is written by a torch kernel on torch's current stream right before the bind, without a synchronisation"""
    torch = pytest.importorskip("torch")
    length, n_ir = 3 * BLOCK, 50000
    base = [np.stack(G.synthetic_ir(n_ir, 2, seed=1200 + g)) for g in range(4)]

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 2, n_ir, ir=ir)
    made = [build(engine.backend, g, None) for g in range(4)]
    b = pkg.Batch([c for c, _ in made])
    src = tensor(torch, base)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)  # the write lands long after the host has bound and launched
        x = src * 0.5
        b.bind_responses(made[0][1], x)
        del x  # (kept from reuse until the bind has read it: record_stream)
        b.run()
    b.sync()
    got = b.fetch()
    want = G.render(pkg, [build(oracle, g, list(base[g] * np.float32(0.5)))[0] for g in range(4)])
    assert maxdiff(got, want) <= TOL


def test_errors_before_launch(pkg, engine):
    torch = pytest.importorskip("torch")
    B = pkg._binding
    api = pkg.api()
    n, length, n_ir = 3, 2 * BLOCK, 9000
    irs = [np.stack(full_ir(2, n_ir, seed=1300 + g)) for g in range(n)]

    def build(be, g, ir):
        return conv_graph(pkg, be, g, length, 2, n_ir, ir=ir)
    made = [build(engine.backend, g, None) for g in range(n)]
    b = pkg.Batch([c for c, _ in made])
    node = made[0][1].id
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and "graph 0" in e.value.message and f"node {node}" in e.value.message
    good = tensor(torch, irs)

    def raw(items):
        arr = (B.ResponseBinding * len(items))(*[B.ResponseBinding(g, nd, C.cast(C.c_void_p(p), B.c_float_p), st) for g, nd, p, st in items])
        return api.batch_bind_responses(b.handle, arr, len(items), None)

    host = np.stack(irs)
    assert raw([(0, node, host.ctypes.data, n_ir)]) == 1                                  # host (numpy) memory
    assert raw([(0, node, good.data_ptr(), 1 << 40)]) == 1                                # extent outside any allocation
    assert raw([(0, node, good.data_ptr(), n_ir - 1)]) == 1                               # channel stride below the declared length
    assert raw([(0, node + 1, good.data_ptr(), n_ir)]) == 2                               # not a declared response (the source)
    assert raw([(n, node, good.data_ptr(), n_ir)]) == 2                                   # graph index out of range
    assert raw([(1, node, good.data_ptr(), n_ir), (1, node, good.data_ptr(), n_ir)]) == 1  # named twice
    with pytest.raises(pkg.WaeError) as e:
        b.bind_responses(node, good[:, :, : n_ir - 1])                                    # shorter than the declared shape
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.bind_responses(node, torch.zeros((n, 1, n_ir), device="cuda"))                  # channels differ
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2  # nothing was bound by the failed calls
    b.bind_responses(node, good)
    b.run()
    b.sync()
    twin = G.render(pkg, [build(engine.backend, g, list(irs[g]))[0] for g in range(n)])
    assert np.array_equal(b.fetch(), twin)
