// zkb200.hpp — header-only C++17 host layer over the C ABI (zkb200.h), mirroring the reference's own interfaces on this path by
// name, argument meaning and error behaviour, so that C++ callers (and a cxx/bindgen-based Rust shim) read like the reference:
//
//   zkb200::Srs                      trait SRS<G> / ipa::SRS<G>              poly-commitment/src/lib.rs:61-241, ipa.rs:56-75,596-800
//   zkb200::PolyComm, BlindedCommitment                                      poly-commitment/src/commitment.rs:47-50,110-116
//   zkb200::BlindersDontMatch        CommitmentError::BlindersDontMatch      poly-commitment/src/error.rs:3-9
//   zkb200::Radix2EvaluationDomain   ark_poly::Radix2EvaluationDomain<F>     kimchi/src/prover.rs:41, circuits/domains.rs:24-33
//   zkb200::Srs::open -> OpeningProof  OpenProof::open / SRS::open          poly-commitment/src/lib.rs:254-298, ipa.rs:823-1061, 1175-1191
//   zkb200::IpaRounds                the folding loop of SRS::open           poly-commitment/src/ipa.rs:929-1007
//   zkb200::Bases::msm / msm_bigint  VariableBaseMSM::{msm, msm_bigint}      ipa.rs:649,658,659,672,943,953
//
// Where the reference returns Result<_, CommitmentError> this layer throws BlindersDontMatch; where it panics
// ("desired commitment domain size greater than evaluations' domain size", ipa.rs:723-725) it throws zkb200::Error.  Field
// elements are 4 x u64 Montgomery limbs, points x||y (identity = zeros): the reference's in-memory form (zkb200.h).
// There is no CPU fallback: Context's constructor throws Error{ZK_ERR_NO_DEVICE} without a CUDA device.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <functional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "zkb200.h"

namespace zkb200 {

using Fe = std::array<uint64_t, 4>;         // Fp / Fq element, Montgomery
using Affine = std::array<uint64_t, 8>;     // x || y
using Jacobian = std::array<uint64_t, 12>;  // X || Y || Z

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& what) : std::runtime_error(what), code(c) {}
};
// CommitmentError::BlindersDontMatch(blinders_len, commitment_len)
struct BlindersDontMatch : Error {
    size_t blinders, commitment;
    BlindersDontMatch(size_t b, size_t c) : Error(ZK_ERR_LENGTH, "BlindersDontMatch(" + std::to_string(b) + ", " + std::to_string(c) + ")"), blinders(b), commitment(c) {}
};
inline void check(int rc) {
    if (rc != ZK_OK) throw Error(rc, zk_last_error());
}

class Context {
  public:
    explicit Context(int device = 0) { check(zk_ctx_create(device, &h_)); }
    ~Context() { zk_ctx_destroy(h_); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    zk_ctx* handle() const { return h_; }
    // nullptr = the context's own (non-blocking) stream; for the legacy default stream pass cudaStreamLegacy, not 0 (zkb200.h)
    void set_stream(void* cuda_stream) { check(zk_ctx_set_stream(h_, cuda_stream)); }
    void set_option(const char* name, long value) { check(zk_ctx_set_option(h_, name, value)); }
    uint64_t launch_count() const { return zk_ctx_launch_count(h_); }

  private:
    zk_ctx* h_ = nullptr;
};

inline Affine into_affine(int curve, const Jacobian& p) {
    Affine a{};
    check(zk_jacobian_to_affine(curve, p.data(), a.data()));
    return a;
}

// A resident Vec<G> (SRS::g or one Lagrange basis) with its window table.
class Bases {
  public:
    Bases(Context& ctx, int curve, const std::vector<Affine>& points, int window_bits = -1) : ctx_(ctx), curve_(curve) {
        check(zk_bases_upload(ctx.handle(), curve, points.empty() ? nullptr : points[0].data(), points.size(), window_bits, 0, &h_));
    }
    ~Bases() { zk_bases_free(h_); }
    Bases(const Bases&) = delete;
    Bases& operator=(const Bases&) = delete;
    zk_bases* handle() const { return h_; }
    int curve() const { return curve_; }
    size_t len() const { return zk_bases_len(h_); }
    // <G::Group as VariableBaseMSM>::msm(&bases[off..off + scalars.len()], scalars): Montgomery scalars
    Jacobian msm(const std::vector<Fe>& scalars, size_t off = 0) const { return run(scalars, off, 1); }
    // msm_bigint: canonical scalars
    Jacobian msm_bigint(const std::vector<Fe>& scalars, size_t off = 0) const { return run(scalars, off, 0); }

  private:
    Jacobian run(const std::vector<Fe>& scalars, size_t off, int mont) const {
        Jacobian out{};
        check(zk_msm(ctx_.handle(), h_, off, scalars.size(), scalars.empty() ? nullptr : scalars[0].data(), mont, 0, out.data()));
        return out;
    }
    Context& ctx_;
    int curve_;
    zk_bases* h_ = nullptr;
};

struct PolyComm {
    std::vector<Affine> chunks;
    size_t len() const { return chunks.size(); }
};
struct BlindedCommitment {
    PolyComm commitment;
    std::vector<Fe> blinders;
};

// ipa::OpeningProof<G> (ipa.rs:1175-1191)
struct OpeningProof {
    std::vector<std::pair<Affine, Affine>> lr;
    Affine delta{}, sg{};
    Fe z1{}, z2{};
};
// one entry of `plnms`: DensePolynomialOrEvaluations + the blinders of its commitment (utils.rs:18-23); data may live in host or
// device memory (zk_open_poly); domain_size = 0 for coefficient form
struct OpenPolynomial {
    const Fe* data = nullptr;
    size_t len = 0, domain_size = 0;
    std::vector<Fe> blinders;
};
// the caller's sponge and group map, seen through the three points where SRS::open consults them (ipa.rs:898-910, 962-970, 1040-1041)
struct OpenTranscript {
    std::function<Affine(const Fe& combined_inner_product)> u_base;        // absorb shift_scalar(cip); U = group_map.to_group(challenge_fq)
    std::function<Fe(unsigned round, const Affine& l, const Affine& r)> round;   // absorb l, r; squeeze_prechallenge().to_field(endo_r)
    std::function<Fe(const Affine& delta)> final_challenge;                // absorb delta; ScalarChallenge(challenge()).to_field(endo_r)
};

// ipa::SRS<G>{g, h, lagrange_bases}, g and every Lagrange basis resident on the device.
class Srs {
  public:
    Srs(Context& ctx, int curve, std::vector<Affine> g, const Affine& h, int window_bits = -1) : g_(std::move(g)), h_xy_(h) {
        check(zk_srs_create(ctx.handle(), curve, g_.empty() ? nullptr : g_[0].data(), g_.size(), h_xy_.data(), window_bits, &h_));
    }
    ~Srs() { zk_srs_destroy(h_); }
    Srs(const Srs&) = delete;
    Srs& operator=(const Srs&) = delete;

    size_t max_poly_size() const { return zk_srs_max_poly_size(h_); }
    size_t size() const { return max_poly_size(); }
    const Affine& blinding_commitment() const { return h_xy_; }
    const std::vector<Affine>& g() const { return g_; }

    // fn get_lagrange_basis_from_domain_size(&self, domain_size) -> &Vec<PolyComm<G>>  (computed on the device, cached)
    std::vector<Affine> get_lagrange_basis_from_domain_size(size_t domain_size) {
        check(zk_srs_lagrange_basis(h_, domain_size, -1));
        std::vector<Affine> out(domain_size);
        check(zk_srs_get_lagrange_basis(h_, domain_size, out.empty() ? nullptr : out[0].data(), domain_size));
        return out;
    }
    // fn open(&self, group_map, plnms, elm, polyscale, evalscale, sponge, rng) -> OpeningProof<G>   (ipa.rs:823-1061), one zk_srs_open;
    // rng_scalars: the 2 * rounds + 2 scalars the reference draws from `rng` (rand_l, rand_r per round, then d, r_delta)
    OpeningProof open(const std::vector<OpenPolynomial>& plnms, const std::vector<Fe>& elm, const Fe& polyscale, const Fe& evalscale,
                      const std::vector<Fe>& rng_scalars, OpenTranscript& sponge) {
        std::vector<zk_open_poly> polys(plnms.size());
        for (size_t k = 0; k < plnms.size(); k++)
            polys[k] = zk_open_poly{plnms[k].data ? plnms[k].data->data() : nullptr, plnms[k].len, plnms[k].domain_size,
                                    plnms[k].blinders.empty() ? nullptr : plnms[k].blinders[0].data(), plnms[k].blinders.size()};
        zk_open_transcript tr{};
        tr.user = &sponge;
        tr.u_base = [](void* u, const uint64_t cip[4], uint64_t out[8]) -> int {
            try { Fe c; std::copy(cip, cip + 4, c.begin()); Affine p = static_cast<OpenTranscript*>(u)->u_base(c); std::copy(p.begin(), p.end(), out); return 0; } catch (...) { return 1; }
        };
        tr.round = [](void* u, unsigned r, const uint64_t l[8], const uint64_t rr[8], uint64_t out[4]) -> int {
            try { Affine a, b; std::copy(l, l + 8, a.begin()); std::copy(rr, rr + 8, b.begin()); Fe c = static_cast<OpenTranscript*>(u)->round(r, a, b); std::copy(c.begin(), c.end(), out); return 0; } catch (...) { return 1; }
        };
        tr.final_challenge = [](void* u, const uint64_t d[8], uint64_t out[4]) -> int {
            try { Affine a; std::copy(d, d + 8, a.begin()); Fe c = static_cast<OpenTranscript*>(u)->final_challenge(a); std::copy(c.begin(), c.end(), out); return 0; } catch (...) { return 1; }
        };
        size_t rounds = 0;
        while ((size_t(1) << rounds) < g_.size()) rounds++;
        std::vector<uint64_t> lr(16 * rounds);
        OpeningProof pr;
        check(zk_srs_open(h_, polys.empty() ? nullptr : polys.data(), polys.size(), elm.empty() ? nullptr : elm[0].data(), elm.size(), polyscale.data(),
                          evalscale.data(), rng_scalars.empty() ? nullptr : rng_scalars[0].data(), rng_scalars.size(), &tr, lr.data(), rounds, &rounds,
                          pr.delta.data(), pr.z1.data(), pr.z2.data(), pr.sg.data()));
        pr.lr.resize(rounds);
        for (size_t r = 0; r < rounds; r++) {
            std::copy(lr.begin() + 16 * r, lr.begin() + 16 * r + 8, pr.lr[r].first.begin());
            std::copy(lr.begin() + 16 * r + 8, lr.begin() + 16 * r + 16, pr.lr[r].second.begin());
        }
        return pr;
    }
    // fn commit_non_hiding(&self, plnm, num_chunks) -> PolyComm<G>
    PolyComm commit_non_hiding(const std::vector<Fe>& coeffs, size_t num_chunks) {
        const size_t n = max_poly_size();
        size_t cap = (coeffs.size() + n - 1) / n;
        if (cap < num_chunks) cap = num_chunks;
        if (cap < 1) cap = 1;
        PolyComm c;
        c.chunks.resize(cap);
        size_t k = 0;
        check(zk_srs_commit_non_hiding(h_, coeffs.empty() ? nullptr : coeffs[0].data(), coeffs.size(), num_chunks, c.chunks[0].data(), cap, &k));
        c.chunks.resize(k);
        return c;
    }
    // fn commit_evaluations_non_hiding(&self, domain, plnm: &Evaluations) -> PolyComm<G>
    PolyComm commit_evaluations_non_hiding(size_t domain_size, const std::vector<Fe>& evals) {
        PolyComm c;
        c.chunks.resize(1);
        check(zk_srs_commit_evaluations_non_hiding(h_, domain_size, evals.empty() ? nullptr : evals[0].data(), evals.size(), c.chunks[0].data()));
        return c;
    }
    // the witness columns of one proof in a single call (kimchi/src/prover.rs:329-351)
    std::vector<PolyComm> commit_evaluations_non_hiding_batch(size_t domain_size, const std::vector<Fe>& evals_k_by_n) {
        if (domain_size == 0 || evals_k_by_n.size() % domain_size) throw Error(ZK_ERR_INVALID, "evaluations are not k x domain_size");
        const size_t k = evals_k_by_n.size() / domain_size;
        std::vector<Affine> out(k);
        if (k) check(zk_srs_commit_evaluations_batch(h_, domain_size, evals_k_by_n[0].data(), k, out[0].data()));
        std::vector<PolyComm> r(k);
        for (size_t j = 0; j < k; j++) r[j].chunks.assign(1, out[j]);
        return r;
    }
    // fn mask_custom(&self, com, blinders) -> Result<BlindedCommitment<G>, CommitmentError>
    BlindedCommitment mask_custom(const PolyComm& com, const std::vector<Fe>& blinders) {
        if (blinders.size() != com.len()) throw BlindersDontMatch(blinders.size(), com.len());
        BlindedCommitment b;
        b.blinders = blinders;
        b.commitment.chunks.resize(com.len());
        if (com.len())
            check(zk_srs_mask_custom(h_, com.chunks[0].data(), com.len(), blinders[0].data(), blinders.size(), b.commitment.chunks[0].data()));
        return b;
    }
    BlindedCommitment commit_custom(const std::vector<Fe>& coeffs, size_t num_chunks, const std::vector<Fe>& blinders) {
        return mask_custom(commit_non_hiding(coeffs, num_chunks), blinders);
    }
    BlindedCommitment commit_evaluations_custom(size_t domain_size, const std::vector<Fe>& evals, const std::vector<Fe>& blinders) {
        return mask_custom(commit_evaluations_non_hiding(domain_size, evals), blinders);
    }

  private:
    std::vector<Affine> g_;
    Affine h_xy_;
    zk_srs* h_ = nullptr;
};

// ark_poly::Radix2EvaluationDomain::<F>::new(size): size is rounded up to a power of two; transforms run in place on the host
// vector (resized with zeros to the domain size, like ark's fft_in_place).
class Radix2EvaluationDomain {
  public:
    Radix2EvaluationDomain(Context& ctx, int field, size_t size) : ctx_(ctx), field_(field) {
        if (size == 0) throw Error(ZK_ERR_INVALID, "domain size must be positive");
        while ((size_t(1) << log_) < size) log_++;
    }
    size_t size() const { return size_t(1) << log_; }
    unsigned log_size_of_group() const { return log_; }
    void fft_in_place(std::vector<Fe>& coeffs) const { run(coeffs, 0, 0); }
    void ifft_in_place(std::vector<Fe>& evals) const { run(evals, 1, 0); }
    void coset_fft_in_place(std::vector<Fe>& coeffs) const { run(coeffs, 0, 1); }
    void coset_ifft_in_place(std::vector<Fe>& evals) const { run(evals, 1, 1); }

  private:
    void run(std::vector<Fe>& v, int inverse, int coset) const {
        if (v.size() > size()) throw Error(ZK_ERR_INVALID, "more coefficients than the domain size");
        const size_t in_len = v.size();
        v.resize(size(), Fe{});
        check(zk_ntt_batch(ctx_.handle(), field_, v[0].data(), log_, 1, inverse ? 0 : in_len, inverse, coset));
    }
    Context& ctx_;
    int field_;
    unsigned log_ = 0;
};

// The folding loop of SRS::open with a and b resident on the device and the bases read from the SRS table.
class IpaRounds {
  public:
    struct LR {
        Jacobian l, r;    // <a_hi, g_lo>, <a_lo, g_hi>
        Fe ip_l, ip_r;    // <a_hi, b_lo>, <a_lo, b_hi>
    };
    IpaRounds(Context& ctx, const Bases& g, std::vector<Fe> a, std::vector<Fe> b) : curve_(g.curve()) {
        size_t n = 2;
        while (n < g.len()) n <<= 1;                         // ipa.rs:848-850 padded_length
        if (a.size() > n || b.size() > n) throw Error(ZK_ERR_INVALID, "a and b must not be longer than the padded SRS");
        a.resize(n, Fe{});                                   // ipa.rs:858-862
        b.resize(n, Fe{});
        check(zk_ipa_begin(ctx.handle(), g.handle(), a[0].data(), b[0].data(), n, &h_));
    }
    ~IpaRounds() { zk_ipa_free(h_); }
    IpaRounds(const IpaRounds&) = delete;
    IpaRounds& operator=(const IpaRounds&) = delete;
    size_t len() const { return zk_ipa_len(h_); }
    LR lr() {
        LR o{};
        check(zk_ipa_round_lr(h_, o.l.data(), o.r.data(), o.ip_l.data(), o.ip_r.data()));
        return o;
    }
    void fold(const Fe& u, const Fe& u_inv) { check(zk_ipa_round_fold(h_, u.data(), u_inv.data())); }
    // after the last fold: (a0, b0, sg)
    struct Final {
        Fe a0, b0;
        Affine sg;
    };
    Final finish() {
        Final f{};
        Jacobian g0{};
        check(zk_ipa_read(h_, f.a0.data(), f.b0.data(), 1, g0.data()));
        f.sg = into_affine(curve_, g0);
        return f;
    }

  private:
    int curve_;
    zk_ipa* h_ = nullptr;
};

}  // namespace zkb200
