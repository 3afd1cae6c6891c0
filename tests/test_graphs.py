"""CUDA graph capture and replay of the fault-tolerant GEMM calls (include/ftsgemm.h, "CUDA graphs").

A captured call replays with whatever its static buffers hold at replay time and gives C bit for bit as an eager call on a
fresh handle with the same inputs, with no detections: the kernels' cross-CTA synchronisation (checksum and cut-tile flags,
the front-phase counter) follows a launch sequence kept in device memory, not values baked into the captured parameters.
Eager calls and replays interleave on one handle.  Calls that synchronise or copy to the host raise FtsgemmError(-2) inside
a capture without invalidating it.  Everything here runs on the GPU.
"""
import numpy as np
import pytest

MN, KM = 0, 1
pytestmark = pytest.mark.gpu


def _ints(rng, shape):
    """small integers: every product and sum is exact, so a corrected element equals the clean one bit for bit"""
    return rng.integers(-4, 5, shape).astype(np.float32)


def _ld(layout, rows, K):
    return rows if layout == MN else (K + 3) // 4 * 4


class _Gemm:
    """One run_ex product M x N x K on flat device buffers that stay put (a graph's static inputs)."""

    def __init__(self, torch, M, N, K, la=MN, lb=MN):
        self.t, self.M, self.N, self.K, self.la, self.lb = torch, M, N, K, la, lb
        self.lda, self.ldb = _ld(la, M, K), _ld(lb, N, K)
        self.dA = torch.zeros(self.lda * (K if la == MN else M), device="cuda")
        self.dB = torch.zeros(self.ldb * (K if lb == MN else N), device="cuda")
        self.dC = torch.zeros(M * N, device="cuda")

    def fill(self, seed):
        """new seeded operands (and C0) copied into the static buffers"""
        rng = np.random.default_rng(seed)
        for buf in (self.dA, self.dB, self.dC):
            buf.copy_(self.t.from_numpy(_ints(rng, buf.numel())))
        return self

    def inputs(self):
        return [b.clone() for b in (self.dA, self.dB, self.dC)]

    def run(self, dev, kid, alpha=1.0, beta=0.0, bufs=None, **opt):
        dA, dB, dC = bufs if bufs is not None else (self.dA, self.dB, self.dC)
        opts = _opts(self.t, **opt)
        dev.run_ex(kid, self.M, self.N, self.K, dA, self.la, self.lda, dB, self.lb, self.ldb, dC, self.M, alpha, beta, opts)
        return dC

    def reference(self, ft, kid, alpha=1.0, beta=0.0, **opt):
        """the same call eagerly on a fresh handle, on copies of the current inputs: (C, stats)"""
        bufs = self.inputs()
        h = ft.FtSgemm()
        try:
            out = self.run(h, kid, alpha, beta, bufs=bufs, **opt)
            self.t.cuda.synchronize()
            return out.cpu(), h.stats()
        finally:
            h.close()


def _opts(torch, **kw):
    import __graft_entry__ as ge
    return ge.load_package().make_opts(stream=torch.cuda.current_stream().cuda_stream, **kw)


def _capture(torch, fn):
    """fn() captured with torch's defaults (global capture mode, its own side stream)"""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def _replay(torch, g):
    g.replay()
    torch.cuda.synchronize()


def _knobs(ft, knobs):
    for k, v in knobs.items():
        ft.debug_set(k, v)


@pytest.fixture
def torch(cuda):
    cuda.cuda.set_device(0)
    return cuda


# ------------------------------------------------------------------ replays with changing inputs
@pytest.mark.parametrize("kid", [31, 40])
@pytest.mark.parametrize("layouts", [(MN, MN), (KM, KM)])
def test_replay_with_new_inputs(torch, ft, kid, layouts):
    """One captured run_ex, replayed with new operands copied into its static buffers before each replay: with MN-major
    operands the front-phase transposes run on every replay and must finish before the producers read their copies."""
    g0 = _Gemm(torch, 1024, 768, 512, *layouts).fill(1)
    dev = ft.FtSgemm()
    try:
        g = _capture(torch, lambda: g0.run(dev, kid, 0.75, -1.5))
        for r in range(3):
            g0.fill(100 + r)
            want, _ = g0.reference(ft, kid, 0.75, -1.5)
            _replay(torch, g)
            assert torch.equal(g0.dC.cpu(), want), r
            st = dev.stats()
            assert st["detected"] == 0 and st["tiles"] > 0, (r, st)
    finally:
        dev.close()


def test_eager_and_replay_interleaved(torch, ft):
    """eager -> capture -> eager -> replay -> eager -> replay on one handle: replays advance the device's launch sequence,
    and the eager calls after them must not start their producers before this launch's transposes are stored."""
    dev = ft.FtSgemm()
    try:
        static = _Gemm(torch, 768, 1024, 640).fill(1)
        eager = _Gemm(torch, 768, 1024, 640)
        results = []

        def check_eager(seed):
            eager.fill(seed)
            want, _ = eager.reference(ft, 31)
            results.append((eager.run(dev, 31).cpu(), want))

        check_eager(10)
        g = _capture(torch, lambda: static.run(dev, 31))
        for r in range(2):
            check_eager(11 + r)
            static.fill(20 + r)
            want, _ = static.reference(ft, 31)
            _replay(torch, g)
            results.append((static.dC.cpu(), want))
        check_eager(13)
        torch.cuda.synchronize()
        for i, (got, want) in enumerate(results):
            assert torch.equal(got, want), i
        assert dev.stats()["detected"] == 0
    finally:
        dev.close()


# ------------------------------------------------------------------ work-plan paths
@pytest.mark.parametrize("knobs,opt", [({"splitk": 3}, {}), ({"enc_front": 1}, {}), ({"enc_front": 0}, {}),
                                       ({}, {"reuse_b_checksums": True})],
                         ids=["cut_tiles", "enc_front", "enc_prepass", "reuse_b"])
def test_replay_work_plan_paths(torch, ft, knobs, opt):
    """cut tiles (parked and seeded accumulators), the encode in the front phase and as a pre-pass, and reuse_b_checksums
    (a captured call encodes on every replay) -- each replayed with new inputs."""
    g0 = _Gemm(torch, 768, 1024, 1600).fill(1)
    dev = ft.FtSgemm()
    try:
        _knobs(ft, knobs)
        g0.run(dev, 31, **opt)  # an eager call first: with reuse_b_checksums the handle holds B's checksums
        torch.cuda.synchronize()
        dev.stats()
        g = _capture(torch, lambda: g0.run(dev, 31, 1.0, -1.5, **opt))
        for r in range(3):
            g0.fill(50 + r)
            want, _ = g0.reference(ft, 31, 1.0, -1.5)
            _replay(torch, g)
            assert torch.equal(g0.dC.cpu(), want), r
            assert dev.stats()["detected"] == 0, r
    finally:
        _knobs(ft, {k: -1 for k in knobs})
        dev.close()


# ------------------------------------------------------------------ faults in a captured call
def test_replayed_faults_are_corrected(torch, ft):
    M, N, K = 768, 1024, 512
    g0 = _Gemm(torch, M, N, K, KM, KM).fill(3)
    clean, _ = g0.reference(ft, 31)
    cm = clean.view(N, M)

    def at(r, c):  # (r, the first column from c on where C is not small: a flipped bit there is a sizeable upset)
        while abs(float(cm[c, r])) < 1.0:
            c += 1
        return {"row": r, "col": c}

    faults = [dict(at(7, 33), xor=1 << 22), dict(at(600, 900), xor=1 << 30)]
    dev = ft.FtSgemm()
    try:
        g = _capture(torch, lambda: g0.run(dev, 31, faults=faults))
        n = 3
        for _ in range(n):
            _replay(torch, g)
            assert torch.equal(g0.dC.cpu(), clean)
        st = dev.stats()
        assert st["detected"] == st["corrected"] == 2 * n and st["uncorrectable"] == 0, st
        # an upset of the stored value (after the accumulator check): the protected store pass recomputes the row segment
        f = [dict(at(511, 130), xor=1 << 27, where="epilogue_value")]
        g = _capture(torch, lambda: g0.run(dev, 31, faults=f, protect_epilogue=True))
        for _ in range(n):
            _replay(torch, g)
            assert torch.equal(g0.dC.cpu(), clean)
        st = dev.stats()
        assert st["epilogue_faults"] == st["recomputed"] == n and st["detected"] == 0, st
    finally:
        dev.close()


# ------------------------------------------------------------------ options
@pytest.mark.parametrize("case", ["bmm_bias", "precision3", "segments4", "cublas0", "cublas7"])
def test_replay_options(torch, ft, case):
    dev = ft.FtSgemm()
    try:
        if case == "bmm_bias":  # attention-shaped scores q @ k^T + bias through bmm: both operands K-major, read in place
            q = torch.zeros(16, 256, 64, device="cuda")
            k = torch.zeros(16, 256, 64, device="cuda")
            bias = torch.zeros(256, device="cuda")
            out = torch.zeros(16, 256, 256, device="cuda")

            def fill(seed):
                r = np.random.default_rng(seed)
                for t in (q, k, bias):
                    t.copy_(torch.from_numpy(_ints(r, tuple(t.shape))))

            fill(1)
            g = _capture(torch, lambda: dev.bmm(q, k.transpose(1, 2), out, bias=bias))
            for r in range(2):
                fill(10 + r)
                h = ft.FtSgemm()
                want = h.bmm(q.clone(), k.clone().transpose(1, 2), bias=bias.clone())
                torch.cuda.synchronize()
                h.close()
                _replay(torch, g)
                assert torch.equal(out, want), r
        else:
            kid, opt = {"precision3": (31, {"precision": 1}), "segments4": (31, {"check_segments": 4}),
                        "cublas0": (0, {}), "cublas7": (7, {})}[case]
            g0 = _Gemm(torch, 512, 768, 1024).fill(1)
            if kid in (0, 7):  # cuBLAS picks and loads its kernels on the first call
                g0.run(dev, kid, **opt)
                torch.cuda.synchronize()
            g = _capture(torch, lambda: g0.run(dev, kid, 1.0, -1.5, **opt))
            for r in range(2):
                g0.fill(30 + r)
                want, _ = g0.reference(ft, kid, 1.0, -1.5, **opt)
                _replay(torch, g)
                assert torch.equal(g0.dC.cpu(), want), r
        if case not in ("cublas0", "cublas7"):
            assert dev.stats()["detected"] == 0
    finally:
        dev.close()


# ------------------------------------------------------------------ first calls inside the capture, workspaces growing
def _capture_then_grow(torch, ft, kid, kid_big=None, knobs={}, warm_up=False, **opt):
    """a handle that has never seen the shape (warm_up: has run it once, eagerly): the captured call's workspaces and plan are
    allocated and uploaded during the capture; a later, much larger eager call (kernel kid_big) grows the workspaces, which
    must not free what the graph uses -- each replay gives C as an eager call on a fresh handle"""
    kid_big = kid if kid_big is None else kid_big
    dev = ft.FtSgemm()
    try:
        _knobs(ft, knobs)
        small = _Gemm(torch, 640, 512, 384).fill(1)
        if warm_up:
            small.run(dev, kid, **opt)
            torch.cuda.synchronize()
        g = _capture(torch, lambda: small.run(dev, kid, 1.0, -1.5, **opt))
        big = _Gemm(torch, 2048, 2048, 1536).fill(2)
        want_big, _ = big.reference(ft, kid_big, **opt)
        assert torch.equal(big.run(dev, kid_big, **opt).cpu(), want_big)
        for r in range(2):
            small.fill(60 + r)
            want, _ = small.reference(ft, kid, 1.0, -1.5, **opt)
            _replay(torch, g)
            assert torch.equal(small.dC.cpu(), want), r
        assert dev.stats()["detected"] == 0
    finally:
        _knobs(ft, {k: -1 for k in knobs})
        dev.close()


def test_first_call_in_capture_and_workspace_growth(torch, ft):
    """the K-major copies, the expected checksums and the work plan"""
    _capture_then_grow(torch, ft, 40)


# each path owns a workspace of the handle that the larger call grows: the 3xTF32 lo parts, the split-K tiles, the wave
# counters (8 units: many waves), the trace (66 units captured, 132 eager), the pre-pass checksum operand and the baseline's
# vectors (cuBLAS loads its kernels on a first, eager call)
@pytest.mark.parametrize("args", [dict(kid=40, precision=1), dict(kid=40, knobs={"splitk": 3}),
                                  dict(kid=40, knobs={"wave_sync": 1, "grid": 8}), dict(kid=31, kid_big=16, knobs={"trace": 1}),
                                  dict(kid=40, knobs={"enc_front": 0}), dict(kid=10, warm_up=True, baseline_host_sync=False)],
                         ids=["lo", "sk", "wave_cnt", "trace", "chk", "aux"])
def test_workspace_growth_after_capture(torch, ft, args):
    _capture_then_grow(torch, ft, **args)


# ------------------------------------------------------------------ several calls in one graph, make_graphed_callables
def test_linear_calls_in_one_graph(torch, ft):
    dev = ft.FtSgemm()
    try:
        rng = np.random.default_rng(7)
        dims = [256, 1024, 512, 768]
        ws = [torch.from_numpy(_ints(rng, (dims[i + 1], dims[i]))).cuda() for i in range(3)]
        bs = [torch.from_numpy(_ints(rng, (dims[i + 1],))).cuda() for i in range(3)]
        x = torch.zeros(128, dims[0], device="cuda")
        outs = []

        def stack():
            h = x
            outs.clear()
            for w, b in zip(ws, bs):
                h = dev.linear(h, w, b) * 0.125  # (keeps the integers small: every sum stays exact)
                outs.append(h)

        g = _capture(torch, stack)
        for r in range(2):
            x.copy_(torch.from_numpy(_ints(np.random.default_rng(70 + r), tuple(x.shape))))
            ref = ft.FtSgemm()
            h = x.clone()
            want = []
            for w, b in zip(ws, bs):
                h = ref.linear(h, w, b) * 0.125
                want.append(h)
            torch.cuda.synchronize()
            ref.close()
            _replay(torch, g)
            for i, (a, b) in enumerate(zip(outs, want)):
                assert torch.equal(a, b), (r, i)
        assert dev.stats()["detected"] == 0
    finally:
        dev.close()


def test_make_graphed_callables_linear_module(torch, ft):
    nn = torch.nn

    class Mlp(nn.Module):
        def __init__(self, dev, w1, b1, w2):
            super().__init__()
            self.dev = dev
            self.w1, self.b1, self.w2 = nn.Parameter(w1), nn.Parameter(b1), nn.Parameter(w2)

        def forward(self, x):
            return self.dev.linear(self.dev.linear(x, self.w1, self.b1) * 0.25, self.w2)

    rng = np.random.default_rng(8)
    w1, b1, w2 = (torch.from_numpy(_ints(rng, s)).cuda() for s in ((512, 256), (512,), (128, 512)))
    x0 = torch.from_numpy(_ints(rng, (64, 256))).cuda()
    gy = torch.from_numpy(_ints(rng, (64, 128))).cuda()
    dev, ref_dev = ft.FtSgemm(), ft.FtSgemm()
    try:
        graphed = torch.cuda.make_graphed_callables(Mlp(dev, w1.clone(), b1.clone(), w2.clone()),
                                                    (x0.clone().requires_grad_(True),))
        eager = Mlp(ref_dev, w1.clone(), b1.clone(), w2.clone())
        for r in range(2):
            # (the graphed backward writes its static gradient buffers, which the first backward adopted as .grad)
            for p in (*graphed.parameters(), *eager.parameters()):
                p.grad = None
            x = (x0 + r).requires_grad_(True)
            xe = (x0 + r).requires_grad_(True)
            y = graphed(x)
            y.backward(gy)
            ye = eager(xe)
            ye.backward(gy)
            torch.cuda.synchronize()
            assert torch.equal(y, ye), r
            assert torch.equal(x.grad, xe.grad), r
            for p, pe in zip(graphed.parameters(), eager.parameters()):
                assert torch.equal(p.grad, pe.grad), r
        assert dev.stats()["detected"] == 0
    finally:
        dev.close()
        ref_dev.close()


# ------------------------------------------------------------------ calls that cannot be captured
def test_uncapturable_calls_raise_and_capture_survives(torch, ft):
    g0 = _Gemm(torch, 512, 512, 256).fill(1)
    dev = ft.FtSgemm()
    codes = []
    try:
        def body():
            g0.run(dev, 31)
            hA = np.zeros(64 * 64, np.float32)
            for call in (lambda: dev.run_host(31, 64, 64, 64, hA, hA, hA.copy(), opts=_opts(torch)),
                         lambda: dev.stats(),
                         lambda: dev.run(10, 64, 64, 64, g0.dA, g0.dB, g0.dC, opts=_opts(torch))):
                with pytest.raises(ft.FtsgemmError) as e:
                    call()
                codes.append(e.value.code)

        g = _capture(torch, body)
        assert codes == [-2, -2, -2]
        g0.fill(9)
        want, _ = g0.reference(ft, 31)
        _replay(torch, g)
        assert torch.equal(g0.dC.cpu(), want)
        assert dev.stats()["detected"] == 0
    finally:
        dev.close()
