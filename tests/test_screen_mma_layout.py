"""CPU check of the index logic of dune_screen_mma_kernel (csrc/dune_screen_mma_kernel.cuh), transcribed to numpy: the re-ordering of
the wgmma operand image (K-major core matrices) into mma.sync m16n8k16 B fragments, the permuted fp32 vectors, the bias fragments,
the accumulator -> A-fragment hand-over between layers (row slots, column pairs), the lane <-> point ownership and the transposing quad
reduction -- one warp's 32 points through the whole screening network equal the plain matrix form of the same network.
(The arithmetic itself -- HMMA, MUFU.TANH, the candidate logic -- is covered on the GPU by tests/test_gpu_screen.py.)"""
import numpy as np

f16 = lambda x: np.asarray(x, np.float16).astype(np.float32)


def _at(n, k):  # byte offset of element (n, k) in a K-major / no-swizzle operand (TcImage, build_tc_image in csrc/dune_tc.cu)
    return (k // 16) * 1024 + ((k % 16) // 8) * 512 + (n // 8) * 128 + (n % 8) * 16 + (k % 8) * 2


def _mma(A, B, C):
    """m16n8k16 from per-lane fragments: A[lane][4][2], B[lane][2][2], C[lane][4] -> D[lane][4]."""
    a, b, c = np.zeros((16, 16), np.float32), np.zeros((16, 8), np.float32), np.zeros((16, 8), np.float32)
    for lane in range(32):
        g, tq = lane >> 2, lane & 3
        a[g, 2 * tq:2 * tq + 2], a[g + 8, 2 * tq:2 * tq + 2] = A[lane][0], A[lane][1]
        a[g, 2 * tq + 8:2 * tq + 10], a[g + 8, 2 * tq + 8:2 * tq + 10] = A[lane][2], A[lane][3]
        b[2 * tq:2 * tq + 2, g], b[2 * tq + 8:2 * tq + 10, g] = B[lane][0], B[lane][1]
        c[g, 2 * tq:2 * tq + 2], c[g + 8, 2 * tq:2 * tq + 2] = C[lane][0:2], C[lane][2:4]
    d = a @ b + c
    return np.array([[d[l >> 2, 2 * (l & 3)], d[l >> 2, 2 * (l & 3) + 1], d[(l >> 2) + 8, 2 * (l & 3)], d[(l >> 2) + 8, 2 * (l & 3) + 1]] for l in range(32)], np.float32)


def _quad_transpose_sum(v):  # sm::quad_transpose_sum: lane tq of a quad ends with the quad total of slot tq
    lanes = np.arange(32)
    b0, b1 = (lanes & 1).astype(bool), (lanes & 2).astype(bool)
    k0, s0 = np.where(b0, v[:, 1], v[:, 0]), np.where(b0, v[:, 0], v[:, 1])
    k1, s1 = np.where(b0, v[:, 3], v[:, 2]), np.where(b0, v[:, 2], v[:, 3])
    k0, k1 = k0 + s0[lanes ^ 1], k1 + s1[lanes ^ 1]
    k, s = np.where(b1, k1, k0), np.where(b1, k0, k1)
    return k + s[lanes ^ 2]


def test_quad_transposing_reduction():
    rng = np.random.default_rng(1)
    v = rng.standard_normal((32, 4)).astype(np.float32)
    got = _quad_transpose_sum(v)
    for lane in range(32):
        q0 = lane & ~3
        assert abs(got[lane] - v[q0:q0 + 4, lane & 3].sum()) < 1e-5


def test_one_warp_tile_equals_the_matrix_form():
    rng = np.random.default_rng(0)
    L = 5
    W = [rng.standard_normal((32, 32)).astype(np.float32) * 0.3 for _ in range(L)]
    bias = [rng.standard_normal(32).astype(np.float32) * 0.1 for _ in range(L)]
    W[4][4:] = 0; bias[4][4:] = 0  # head: E = 4 rows, zero padded
    G = [rng.standard_normal(32).astype(np.float32) for _ in range(3)]
    BE = [rng.standard_normal(32).astype(np.float32) * 0.1 for _ in range(3)]
    W0X, W0Y, B0 = (rng.standard_normal(32).astype(np.float32) for _ in range(3))
    img = np.zeros(5 * 4096 // 2, np.float32)  # the hi halves of the operand image, indexed by byte offset / 2
    for l in range(L):
        for n in range(32):
            for k in range(32):
                img[(l * 4096 + _at(n, k)) // 2] = f16(W[l][n, k])
    # operand staging of the kernel: B fragments [layer][k-step][n-tile pair][lane][4 words], permuted vectors [tq][j][h], bias quads
    wf = np.zeros((2560, 2), np.float32)
    for x in range(2560):
        c, ln, jp, s, l = x & 3, (x >> 2) & 31, (x >> 7) & 1, (x >> 8) & 1, x >> 9
        n, k = 8 * (2 * jp + (c >> 1)) + (ln >> 2), 16 * s + 2 * (ln & 3) + 8 * (c & 1)
        off = l * 4096 + _at(n, k)
        wf[x] = img[off // 2:off // 2 + 2]
    perm = lambda v: np.array([v[8 * ((e >> 1) & 3) + 2 * (e >> 3) + (e & 1)] for e in range(32)], np.float32)
    vec = {k: perm(v) for k, v in dict(W0X=W0X, W0Y=W0Y, B0=B0, G1=G[0], BE1=BE[0], G6=G[1], BE6=BE[1], G11=G[2], BE11=BE[2]).items()}
    vq = lambda name, tq: vec[name][8 * tq:8 * tq + 8].reshape(4, 2)
    biasq = np.array([[[[bias[l][8 * j + 2 * q], bias[l][8 * j + 2 * q + 1]] * 2 for j in range(4)] for q in range(4)] for l in range(L)], np.float32)

    P = rng.standard_normal((32, 2)).astype(np.float32)
    lanes = np.arange(32)
    own = 8 * (lanes & 3) + (lanes >> 2)  # lane (g, tq) owns local point 8 tq + g
    x0, y0 = P[own, 0], P[own, 1]
    xr = np.stack([x0[(lanes & ~3) | r] for r in range(4)], 1)  # row slot r = local point g + 8 r = the point of lane (g, tq = r)
    yr = np.stack([y0[(lanes & ~3) | r] for r in range(4)], 1)
    acc = np.zeros((32, 4, 4, 2), np.float32)
    for lane in range(32):
        tq = lane & 3
        for r in range(4):
            acc[lane, r] = vq("W0Y", tq) * yr[lane, r] + (vq("W0X", tq) * xr[lane, r] + vq("B0", tq))

    def ln_tanh(acc, gn, bn):
        rs = 1 / np.sqrt(_quad_transpose_sum((acc ** 2).sum(axis=(2, 3))) / 32 + 1e-5)
        a = np.zeros((32, 2, 2, 4, 2), np.float32)
        for lane in range(32):
            for r in range(4):
                t = np.tanh(acc[lane, r] * rs[(lane & ~3) | r] * vq(gn, lane & 3) + vq(bn, lane & 3))
                for j in range(4):
                    a[lane, r >> 1, j >> 1, (j & 1) * 2 + (r & 1)] = f16(t[j])
        return a

    def relu(acc):
        a = np.zeros((32, 2, 2, 4, 2), np.float32)
        for lane in range(32):
            for r in range(4):
                for j in range(4):
                    a[lane, r >> 1, j >> 1, (j & 1) * 2 + (r & 1)] = f16(np.maximum(acc[lane, r, j], 0))
        return a

    def dense(l, a, NT):
        out = np.zeros((32, 4, NT, 2), np.float32)
        for j in range(NT):
            for mt in range(2):
                C = np.array([biasq[l, lane & 3, j] for lane in range(32)])
                for s in range(2):
                    base = lambda lane: (((l * 2 + s) * 2 + (j >> 1)) * 32 + lane) * 4 + 2 * (j & 1)
                    C = _mma([[a[lane, mt, s, i] for i in range(4)] for lane in range(32)], [[wf[base(lane)], wf[base(lane) + 1]] for lane in range(32)], C)
                out[:, 2 * mt, j], out[:, 2 * mt + 1, j] = C[:, 0:2], C[:, 2:4]
        return out

    a = ln_tanh(acc, "G1", "BE1"); acc = dense(0, a, 4)
    a = relu(acc); acc = dense(1, a, 4)
    a = ln_tanh(acc, "G6", "BE6"); acc = dense(2, a, 4)
    a = relu(acc); acc = dense(3, a, 4)
    a = ln_tanh(acc, "G11", "BE11"); mu = dense(4, a, 1)

    def ln(h, g, be):
        return np.tanh(h / np.sqrt((h ** 2).mean(1, keepdims=True) + 1e-5) * g + be)

    Wq = [f16(w) for w in W]
    h = np.outer(P[:, 0], W0X) + np.outer(P[:, 1], W0Y) + B0
    h = f16(ln(h, G[0], BE[0])) @ Wq[0].T + bias[0]
    h = f16(np.maximum(h, 0)) @ Wq[1].T + bias[1]
    h = f16(ln(h, G[1], BE[1])) @ Wq[2].T + bias[2]
    h = f16(np.maximum(h, 0)) @ Wq[3].T + bias[3]
    ref = f16(ln(h, G[2], BE[2])) @ Wq[4].T + bias[4]
    err = max(abs(mu[lane, r, 0, hh] - ref[(lane >> 2) + 8 * r, 2 * (lane & 3) + hh]) for lane in range(32) for r in range(4) for hh in range(2))
    assert err < 1e-4 * max(1.0, float(abs(ref).max())), err
