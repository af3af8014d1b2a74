"""The host reference of the philox planning mode's noise (oracle/philox_oracle.py) on its own: Random123's known-answer
vectors for Philox4x32-10, the counter / key packing of rng_bits4, the pinned extreme groups the GPU test
(tests/test_gpu_philox_plan.py) checks the device against, and the qidx rule on synthetic words.  No GPU needed."""
import numpy as np
import pytest
import torch

from oracle import philox_oracle as ph

# Random123 (Salmon et al., SC'11) known-answer vectors of Philox4x32-10: (counter, key, output)
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]

# Groups whose words sit at the ends of the 24-bit uniforms, found once by a host search: (seed, plan, stream, group,
# component).  Box-Muller components: u1 is word 0 or 2 of the group, u2 word 1 or 3.
SEED = 0x2545F4914F6CDD1D
PINNED = {
    "u1=1": (SEED, 1, 0, 20108247, 0),            # rho = 0: both normals of the pair are 0
    "u1=2^-24": (SEED, 1, 0, 17827369, 0),        # rho = sqrt(48 ln 2): the largest normal the generator produces
    "u2=0": (SEED, 1, 0, 2168928, 1),
    "u2=1/4": (SEED, 1, 0, 20964864, 3),
    "u2=1/2": (SEED, 1, 0, 1382532, 1),
    "u2=3/4": (SEED, 1, 0, 24805492, 1),
    "expo=0": (SEED, 1, ph.STREAM_EXPO, 921393, 3),          # an exponential draw of exactly 0
    "expo=24ln2": (SEED, 1, ph.STREAM_EXPO, 1368678, 0),      # the largest exponential draw
}
# A state {seed, plan counter} whose expo draw [E = 2, K = 16] holds an exact 0 at element ZERO_EXPO[2] (the pick test)
ZERO_EXPO = (1099512237574, 1, 13)


def test_known_answer_vectors():
    for ctr, key, want in KAT:
        got = ph.philox4x32_10(np.array(ctr), np.array(key))
        assert tuple(int(x) for x in got) == want
    # vectorised: the three at once, and broadcast against one key
    got = ph.philox4x32_10(np.array([c for c, _, _ in KAT]), np.array([k for _, k, _ in KAT]))
    assert [tuple(int(x) for x in row) for row in got] == [w for _, _, w in KAT]
    one = ph.philox4x32_10(np.array([c for c, _, _ in KAT]), np.array([0, 0]))
    assert tuple(int(x) for x in one[0]) == KAT[0][2]


def test_counter_and_key_packing():
    """bits4 packs counter (group lo, group hi, stream, plan lo) and key (seed lo, seed hi ^ plan hi)."""
    seed, plan, stream, group = 0x0123456789ABCDEF, (5 << 32) | 7, 0x80000003, (3 << 32) | 11
    want = ph.philox4x32_10(np.array([11, 3, 0x80000003, 7]), np.array([0x89ABCDEF, 0x01234567 ^ 5]))
    assert np.array_equal(ph.bits4(seed, plan, stream, group), want)
    # plan 2^32 differs from plan 0 only through the key's high word
    a = ph.bits4(seed, 1 << 32, 0, np.arange(4, dtype=np.uint64))
    b = ph.philox4x32_10(np.stack([np.arange(4), np.zeros(4), np.zeros(4), np.zeros(4)], -1),
                         np.array([0x89ABCDEF, 0x01234567 ^ 1]))
    assert np.array_equal(a, b) and not np.array_equal(a, ph.bits4(seed, 0, 0, np.arange(4, dtype=np.uint64)))
    # broadcasting over seeds, streams and groups gives the same as one call each
    s = np.array([1, 1 << 33])[:, None]
    g = np.array([0, (1 << 32) + 5], dtype=np.uint64)[None, :]
    many = ph.bits4(s, 9, 2, g)
    for i in range(2):
        for j in range(2):
            assert np.array_equal(many[i, j], ph.bits4(int(s[i, 0]), 9, 2, int(g[0, j])))


def test_normal_and_uniform_laws():
    w = ph.bits4(SEED, 3, 0, np.arange(1 << 12, dtype=np.uint64))
    u1, u2 = ph.box_muller_uniforms(w)
    assert np.array_equal(u1[:, 0], ((w[:, 0] >> 8).astype(np.float64) + 1) / 2 ** 24)
    assert np.array_equal(u2[:, 1], (w[:, 3] >> 8).astype(np.float64) / 2 ** 24)
    assert np.array_equal(u1.astype(np.float32).astype(np.float64), u1)       # exact in fp32
    v, rho = ph.normal4(SEED, 3, 0, np.arange(1 << 12, dtype=np.uint64))
    r = np.sqrt(-2 * np.log(u1))
    assert np.allclose(v[:, 0], r[:, 0] * np.cos(2 * np.pi * u2[:, 0]), rtol=0, atol=1e-15)
    assert np.allclose(v[:, 3], r[:, 1] * np.sin(2 * np.pi * u2[:, 1]), rtol=0, atol=1e-15)
    assert np.array_equal(rho[:, 0], rho[:, 1]) and np.array_equal(rho[:, 2], rho[:, 3])
    assert np.allclose(np.hypot(v[:, 0], v[:, 1]), rho[:, 0], rtol=1e-14, atol=0)
    assert abs(v.mean()) < 0.05 and abs(v.var() - 1) < 0.05
    u = ph.uniform4(SEED, 3, 0, np.arange(4, dtype=np.uint64))
    assert np.array_equal(u, (ph.bits4(SEED, 3, 0, np.arange(4, dtype=np.uint64)) >> 8) / 2 ** 24)
    # draw elements: component i % 4 of group i / 4
    n, rn = ph.normals(SEED, 3, 0, 10)
    assert np.array_equal(n, v.reshape(-1)[:10]) and np.array_equal(rn, rho.reshape(-1)[:10])


@pytest.mark.parametrize("name", list(PINNED))
def test_pinned_extremes(name):
    seed, plan, stream, group, comp = PINNED[name]
    w = ph.bits4(seed, plan, stream, group)
    top = int(w[comp]) >> 8
    if name.startswith("expo"):
        assert stream == ph.STREAM_EXPO
        x = -np.log(1.0 - ph.uniform4(seed, plan, stream, group)[comp])
        assert (top, x) == ((0, 0.0) if name == "expo=0" else (0xFFFFFF, 24 * np.log(2.0)))
        return
    v, rho = ph.normal4(seed, plan, stream, group)
    if name.startswith("u1"):
        assert comp in (0, 2)
        if name == "u1=1":
            assert top == 0xFFFFFF and rho[comp] == 0.0 and v[comp] == 0.0 and v[comp + 1] == 0.0
        else:
            assert top == 0 and rho[comp] == ph.RHO_MAX and abs(ph.RHO_MAX - 5.768) < 1e-3
    else:
        assert comp in (1, 3)
        q = {"u2=0": 0, "u2=1/4": 1, "u2=1/2": 2, "u2=3/4": 3}[name]
        assert top == q << 22
        c, s = v[comp - 1] / rho[comp], v[comp] / rho[comp]
        assert abs(c - (1, 0, -1, 0)[q]) < 1e-15 and abs(s - (0, 1, 0, -1)[q]) < 1e-15


def test_zero_expo_state():
    seed, plan, elem = ZERO_EXPO
    x = ph.expo(seed, plan, 2 * 16)
    assert x[elem] == 0.0 and np.count_nonzero(x == 0.0) >= 1 and bool((x >= 0).all())
    d = ph.plan_draws(seed, plan, 2, 3, 8, 6, 3, 16, 3)
    assert d["expo"].reshape(-1)[elem] == 0.0


@pytest.mark.parametrize("num_q", [2, 3, 4, 5, 8, 10])
def test_qidx_rule_on_synthetic_words(num_q):
    rng = np.random.default_rng(num_q)
    rows = rng.integers(0, 8, size=(400, num_q), dtype=np.uint64)        # few distinct values: ties everywhere
    got = ph.two_smallest(rows)
    for w, (i, j) in zip(rows, got):
        order = sorted(range(num_q), key=lambda k: (int(w[k]), k))      # smallest first, the lower index on ties
        assert (i, j) == tuple(order[:2])
    assert np.array_equal(ph.two_smallest(np.zeros((1, num_q), dtype=np.uint64)), [[0, 1]])
    assert np.array_equal(ph.two_smallest(np.arange(num_q, dtype=np.uint64)[::-1][None]), [[num_q - 1, num_q - 2]])
    # rows read ceil(num_q / 4) groups each: one, two or three
    G = (num_q + 3) // 4
    words = ph.qidx_words(SEED, 4, 6, num_q)
    flat = ph.bits4(SEED, 4, ph.STREAM_QIDX, np.arange(6 * G, dtype=np.uint64)).reshape(6, 4 * G)
    assert np.array_equal(words, flat[:, :num_q])
    q = ph.qidx(SEED, 4, 2, 3, num_q)
    assert q.shape == (2, 3, 2) and np.array_equal(q.reshape(6, 2), ph.two_smallest(words))
    assert bool((q[..., 0] != q[..., 1]).all()) and bool((q < num_q).all())


def test_plan_draws_and_layout():
    E, H, P, A, I, K, N = 3, 2, 7, 5, 3, 9, 16
    d = ph.plan_draws(SEED, 6, E, H, P, A, I, K, 5, pixel=True)
    v, _ = ph.normals(SEED, 6, ph.STREAM_PRIOR, E * H * P * A)
    assert np.array_equal(d["prior"].reshape(-1), v) and d["final"].shape == (E, A) and d["shift"].shape == (E, 2)
    assert set(np.unique(ph.shift(SEED, 6, 4096))) == set(range(7))
    e = ph.plan_draws(SEED, 6, E, H, 0, A, I, K, 5, eval_mode=True)
    assert e["prior"] is None and e["final"] is None and e["shift"] is None and np.array_equal(e["expo"], d["expo"])
    # noise_r (e, t, n, a): group ((e H + t) N + n) A4 + a / 4 of stream 2 it, component a % 4; n counts the prior rows
    r, _ = ph.noise_r(SEED, 6, 2, E, H, N, P, A)
    pi, _ = ph.noise_pi(SEED, 6, 2, E, N, A)
    assert r.shape == (E, H, N - P, A) and pi.shape == (E, N, A)
    for (e, t, n, a) in ((0, 0, P, 0), (2, 1, N - 1, 4), (1, 0, P + 3, 3)):
        g = ((e * H + t) * N + n) * 2 + a // 4
        assert r[e, t, n - P, a] == ph.normal4(SEED, 6, 4, g)[0][a % 4]
    for (e, n, a) in ((0, 0, 0), (2, N - 1, 4), (1, 5, 2)):
        assert pi[e, n, a] == ph.normal4(SEED, 6, 5, (e * N + n) * 2 + a // 4)[0][a % 4]
    nz = ph.plan_noise(r[None], pi[None], d["prior"], d["qidx"][:1], d["expo"], d["final"], d["shift"])
    assert nz.r.shape == (E, 1, H, N - P, A) and nz.pi.shape == (E, 1, N, A) and nz.qidx.shape == (E, 1, 2)
    assert nz.qidx.dtype == torch.int64 and torch.equal(nz.r[1, 0], torch.as_tensor(r[1]))
    nz0 = ph.plan_noise(r[None], pi[None], None, d["qidx"][:1], d["expo"], None, H=H, A=A)
    assert nz0.prior.shape == (E, H, 0, A) and torch.equal(nz0.final, torch.zeros(E, A, dtype=nz0.final.dtype))
