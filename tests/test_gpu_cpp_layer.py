"""The C++ host layer (include/zkb200.hpp: Srs, Radix2EvaluationDomain, Bases, IpaRounds — the C++ mirror of the reference's
SRS<G> trait, poly-commitment/src/lib.rs:61-241, and of the open rounds, ipa.rs:929-1007) driven by a C++ program
(tests/cpp/host_layer.cpp) and checked against the oracle."""
import os
import shutil
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def b_poly_coefficients(chals, m):
    k = len(chals)
    s = [1] * (1 << k)
    for i in range(1, 1 << k):
        kk = i.bit_length() - 1
        s[i] = s[i - (1 << kk)] * chals[k - 1 - kk] % m
    return s


def test_cpp_host_layer_matches_the_oracle(orc, pallas_srs, tmp_path):
    gxx = shutil.which("g++", path="/usr/bin") or shutil.which("g++")
    if not gxx:
        pytest.skip("no C++ compiler on this box")
    lib_dir = os.path.join(ROOT, "proof_systems_b200")
    exe = str(tmp_path / "host_layer")
    subprocess.check_call([gxx, "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "host_layer.cpp"), "-L", lib_dir, "-lzkb200", f"-Wl,-rpath,{lib_dir}", "-o", exe])
    G = pallas_srs
    m = orc.FQ_MODULUS
    n, k = 64, 6
    g = G.g[:n]
    h = G.mont_points(G.h_xy_canon)[0]
    coeffs_i = orc.limbs_to_ints(orc.random_scalars(G.scalar, n + n // 2, seed=51))
    evals_i = orc.limbs_to_ints(orc.random_scalars(G.scalar, n, seed=52))
    blind_i = orc.limbs_to_ints(orc.random_scalars(G.scalar, 2, seed=53))
    u = orc.limbs_to_ints(orc.random_scalars(G.scalar, 1, seed=54))[0]
    mont = lambda xs: orc.to_mont(G.scalar, orc.ints_to_limbs(xs))
    blob = np.concatenate([np.array([n], dtype=np.uint64), g.reshape(-1), h.reshape(-1), mont(coeffs_i).reshape(-1), mont(evals_i).reshape(-1),
                           mont(blind_i).reshape(-1), mont([u]).reshape(-1), mont([pow(u, -1, m)]).reshape(-1)])
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    blob.astype("<u8").tofile(fin)
    run = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert run.returncode == 0, (run.returncode, run.stdout, run.stderr)
    out = np.fromfile(fout, dtype="<u8")
    pos = 0

    def take(count, width):
        nonlocal pos
        v = out[pos:pos + count * width].reshape(count, width)
        pos += count * width
        return v

    chunks, masked, ce = take(2, 8), take(2, 8), take(1, 8)[0]
    fft, back = take(n, 4), take(n, 4)
    msm, lr, ips = take(1, 8)[0], take(2, 8), take(2, 4)
    a0, b0, sg = take(1, 4)[0], take(1, 4)[0], take(1, 8)[0]
    open_pts, open_z = take(4, 8), take(2, 4)            # Srs::open: l_0, r_0, delta, sg; z1, z2
    assert pos == out.size
    want0 = orc.msm(G.cid, g, orc.ints_to_limbs(coeffs_i[:n]))
    want1 = orc.msm(G.cid, g[: n // 2], orc.ints_to_limbs(coeffs_i[n:]))
    assert np.array_equal(chunks[0], want0) and np.array_equal(chunks[1], want1)          # ipa.rs:663-676
    for j, w in enumerate((want0, want1)):
        assert np.array_equal(masked[j], orc.affine_add(G.cid, w, orc.scalar_mul(G.cid, h, blind_i[j])))   # ipa.rs:605-622
    assert np.array_equal(ce, orc.msm(G.cid, G.lagrange_small(n), orc.ints_to_limbs(evals_i)))              # ipa.rs:706-728
    assert np.array_equal(fft, orc.ntt(G.scalar, mont(coeffs_i[:n]))) and np.array_equal(back, mont(coeffs_i[:n]))
    assert np.array_equal(msm, want0)
    a, b, hh = coeffs_i[:n], evals_i, n // 2
    assert np.array_equal(lr[0], orc.msm(G.cid, g[:hh], orc.ints_to_limbs(a[hh:])))        # ipa.rs:943-951
    assert np.array_equal(lr[1], orc.msm(G.cid, g[hh:], orc.ints_to_limbs(a[:hh])))        # ipa.rs:953-961
    assert orc.fe_int(G.scalar, ips[0]) == sum(x * y for x, y in zip(a[hh:], b[:hh])) % m
    assert orc.fe_int(G.scalar, ips[1]) == sum(x * y for x, y in zip(a[:hh], b[hh:])) % m
    s = b_poly_coefficients([u] * k, m)
    s_inv = b_poly_coefficients([pow(u, -1, m)] * k, m)
    assert orc.fe_int(G.scalar, a0) == sum(x * y for x, y in zip(a, s_inv)) % m
    assert orc.fe_int(G.scalar, b0) == sum(x * y for x, y in zip(b, s)) % m
    assert np.array_equal(sg, orc.msm(G.cid, g, orc.ints_to_limbs(s)))                      # commitment.rs:565-581
    # OpenProof::open through the C++ layer == the same call through the ctypes layer (itself pinned to the reference's 700-byte
    # opening proof in tests/test_gpu_srs.py), same stand-in sponge: U = g[7], every challenge = u
    import proof_systems_b200 as zk
    with zk.Context(0) as ctx:
        srs = zk.SRS(ctx, G.cid, g, h)
        um, uim = mont([u])[0], mont([pow(u, -1, m)])[0]
        pr = zk.srs_open(srs, [(mont(coeffs_i[:n]), 0, mont(blind_i[:1]))], np.stack([um, uim]), um, uim, mont(evals_i[:2 * k + 2]),
                         lambda cip: g[7], lambda i, l, r: um, lambda d: um)
        assert np.array_equal(open_pts[0], pr.lr[0][0]) and np.array_equal(open_pts[1], pr.lr[0][1])
        assert np.array_equal(open_pts[2], pr.delta) and np.array_equal(open_pts[3], pr.sg)
        assert np.array_equal(open_z[0], pr.z1) and np.array_equal(open_z[1], pr.z2)
        srs.close()
