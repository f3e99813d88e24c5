// DuplexChallenger<KoalaBear, Poseidon2-16, 16, 8> on the host side of the library plus the
// proof-of-work grind kernel.
// Semantics: sp1-gpu/crates/sys/include/challenger/challenger.cuh:22-112 (== p3 DuplexChallenger);
// grind replaces grindKernel (challenger.cuh:114-158, racing threads + found_flag => ANY witness) with a
// deterministic search: candidates are scanned in increasing canonical order in fixed batches and the
// MINIMUM valid witness of the first batch that contains one is returned, so proofs are reproducible.
#include "ctx.cuh"
#include "challenger.cuh"
#include "poseidon2.cuh"

namespace {

// st: 34 words. One candidate per thread: w = base + tid (canonical).
__global__ void __launch_bounds__(256) grind_kernel(const uint32_t* __restrict__ st, uint32_t bits, uint32_t base, uint32_t count,
                                                    uint32_t* __restrict__ best) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    uint32_t w = base + t;
    if (w >= kb::P) return;
    uint32_t s[16];
#pragma unroll
    for (int i = 0; i < 16; i++) s[i] = st[i];
    const uint32_t nin = st[32];
#pragma unroll
    for (int i = 0; i < 8; i++)
        if ((uint32_t)i < nin) s[i] = st[16 + i];
    const uint32_t wm = kb::from_canonical(w);
#pragma unroll
    for (int i = 0; i < 8; i++)
        if ((uint32_t)i == nin) s[i] = wm;
    p2::permute(s);
    uint32_t v = kb::to_canonical(s[7]) & ((1u << bits) - 1u);
    if (v == 0) atomicMin(best, w);
}

// recompute for the chosen witness and write the post-check_witness challenger state
__global__ void grind_finalize_kernel(uint32_t* __restrict__ st, uint32_t w) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t s[16];
    for (int i = 0; i < 16; i++) s[i] = st[i];
    const uint32_t nin = st[32];
    for (uint32_t i = 0; i < nin; i++) s[i] = st[16 + i];
    s[nin] = kb::from_canonical(w);
    st[16 + nin] = s[nin];  // the observed witness stays in the (logically empty) input buffer words
    p2::permute(s);
    for (int i = 0; i < 16; i++) st[i] = s[i];
    for (int i = 0; i < 8; i++) st[24 + i] = s[i];
    st[32] = 0;
    st[33] = 7;  // one output element consumed by sample_bits
}

}  // namespace

// d_state: 34 words on device (in/out); returns the witness as a Montgomery word in *witness_monty
sp1b200_err sp1b200_grind_device(sp1b200_ctx* ctx, uint32_t* d_state, uint32_t bits, uint32_t* witness_canonical) {
    if (bits > 30) return sp1b200_set_error("grind: %u bits unsupported", bits);
    uint32_t* d_best;
    SP1_CUDA(cudaMallocFromPoolAsync((void**)&d_best, sizeof(uint32_t), ctx->pool, ctx->stream));
    uint32_t batch = 1u << (bits + 2 < 16 ? 16 : (bits + 2 > 22 ? 22 : bits + 2));
    uint32_t best = 0xffffffffu;
    for (uint64_t base = 0; base < kb::P; base += batch) {
        SP1_CUDA(cudaMemsetAsync(d_best, 0xff, sizeof(uint32_t), ctx->stream));
        SP1_LAUNCH(ctx, grind_kernel, (batch + 255) / 256, 256, 0, d_state, bits, (uint32_t)base, batch, d_best);
        SP1_CUDA(cudaMemcpyAsync(&best, d_best, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
        SP1_CUDA(cudaStreamSynchronize(ctx->stream));
        if (best != 0xffffffffu) break;
    }
    cudaFreeAsync(d_best, ctx->stream);
    if (best == 0xffffffffu) return sp1b200_set_error("grind: no witness");
    SP1_LAUNCH(ctx, grind_finalize_kernel, 1, 32, 0, d_state, best);
    *witness_canonical = best;
    return nullptr;
}

// ---- host challenger -----------------------------------------------------------------------------------------
namespace {
using p2::RC_HOST;
inline uint32_t h_cube(uint32_t x) { return kb::mul(kb::sqr(x), x); }
inline void h_ext_layer(uint32_t* s) {
    for (int q = 0; q < 16; q += 4) {
        uint32_t a = s[q], b = s[q + 1], c = s[q + 2], d = s[q + 3];
        uint32_t t = kb::add(kb::add(a, b), kb::add(c, d));
        // rows of [[2,3,1,1],[1,2,3,1],[1,1,2,3],[3,1,1,2]]
        s[q] = kb::add(t, kb::add(a, kb::add(b, b)));
        s[q + 1] = kb::add(t, kb::add(b, kb::add(c, c)));
        s[q + 2] = kb::add(t, kb::add(c, kb::add(d, d)));
        s[q + 3] = kb::add(t, kb::add(d, kb::add(a, a)));
    }
    uint32_t col[4];
    for (int j = 0; j < 4; j++) col[j] = kb::add(kb::add(s[j], s[4 + j]), kb::add(s[8 + j], s[12 + j]));
    for (int i = 0; i < 16; i++) s[i] = kb::add(s[i], col[i & 3]);
}
inline void h_int_layer(uint32_t* s) {
    uint64_t sum = 0;
    for (int i = 0; i < 16; i++) sum += s[i];
    uint32_t o0 = kb::monty_reduce(sum - s[0] + (kb::P - s[0]));
    for (int i = 1; i < 16; i++) s[i] = kb::monty_reduce(sum + ((uint64_t)s[i] << (i == 15 ? 15 : i - 1)));
    s[0] = o0;
}
}  // namespace

void host_poseidon2_permute(uint32_t* s) {
    h_ext_layer(s);
    for (int r = 0; r < 4; r++) {
        for (int i = 0; i < 16; i++) s[i] = h_cube(kb::add(s[i], RC_HOST.ext[r * 16 + i]));
        h_ext_layer(s);
    }
    for (int r = 0; r < 20; r++) {
        s[0] = h_cube(kb::add(s[0], RC_HOST.inr[r]));
        h_int_layer(s);
    }
    for (int r = 4; r < 8; r++) {
        for (int i = 0; i < 16; i++) s[i] = h_cube(kb::add(s[i], RC_HOST.ext[r * 16 + i]));
        h_ext_layer(s);
    }
}

void host_hash(const uint32_t* in, size_t n, uint32_t* out8) {
    uint32_t s[16] = {0};
    size_t fill = 0;
    for (size_t i = 0; i < n; i++) { s[fill++] = in[i]; if (fill == 8) { host_poseidon2_permute(s); fill = 0; } }
    if (fill) host_poseidon2_permute(s);
    memcpy(out8, s, 32);
}
void host_compress(const uint32_t* l8, const uint32_t* r8, uint32_t* out8) {
    uint32_t s[16];
    memcpy(s, l8, 32); memcpy(s + 8, r8, 32);
    host_poseidon2_permute(s);
    memcpy(out8, s, 32);
}

void table_size_commitment(const uint32_t* original8, const std::vector<std::pair<uint64_t, uint64_t>>& tables, uint32_t* out8) {
    std::vector<uint32_t> meta{kb::to_monty_c(tables.size())};
    for (auto& t : tables) meta.push_back(kb::to_monty_c(t.first));
    for (auto& t : tables) meta.push_back(kb::to_monty_c(t.second));
    uint32_t h[8];
    host_hash(meta.data(), meta.size(), h);
    host_compress(original8, h, out8);
}

void observe_chip_shapes(HostChallenger& ch, size_t n_chips, const uint64_t* heights, const char* const* names) {
    ch.observe(kb::to_monty_c(n_chips));
    for (size_t k = 0; k < n_chips; k++) {
        ch.observe(kb::to_monty_c(heights[k]));
        const size_t len = strlen(names[k]);
        ch.observe(kb::to_monty_c(len));
        for (size_t i = 0; i < len; i++) ch.observe(kb::to_monty_c((uint8_t)names[k][i]));
    }
}

hf::E4 batched_opening_claim(const uint32_t* main, uint32_t main_w, const uint32_t* prep, uint32_t prep_w, const hf::E4& gamma) {
    hf::E4 acc, g = gamma;
    for (uint32_t j = 0; j < main_w; j++) { acc = acc + hf::E4::load(main + 4 * j) * g; g = g * gamma; }
    for (uint32_t j = 0; j < prep_w; j++) { acc = acc + hf::E4::load(prep + 4 * j) * g; g = g * gamma; }
    return acc;
}

void HostChallenger::duplexing() {
    for (uint32_t i = 0; i < nin; i++) sponge[i] = inbuf[i];
    nin = 0;
    host_poseidon2_permute(sponge);
    for (int i = 0; i < 8; i++) outbuf[i] = sponge[i];
    nout = 8;
}
sp1b200_err HostChallenger::init(sp1b200_ctx* c, const uint32_t* st34) {
    ctx = c;
    SP1_CUDA(cudaMallocFromPoolAsync((void**)&d_scratch, 34 * sizeof(uint32_t), c->pool, c->stream));
    load(st34);
    return nullptr;
}
HostChallenger::~HostChallenger() {
    if (d_scratch) cudaFreeAsync(d_scratch, ctx->stream);
}
void HostChallenger::load(const uint32_t* s) {
    memcpy(sponge, s, 64); memcpy(inbuf, s + 16, 32); memcpy(outbuf, s + 24, 32);
    nin = s[32]; nout = s[33];
}
void HostChallenger::store(uint32_t* s) const {
    memcpy(s, sponge, 64); memcpy(s + 16, inbuf, 32); memcpy(s + 24, outbuf, 32);
    s[32] = nin; s[33] = nout;
}
void HostChallenger::observe(uint32_t v) {
    nout = 0;
    inbuf[nin++] = v;
    if (nin == 8) duplexing();
}
void HostChallenger::observe_n(const uint32_t* v, size_t n) { for (size_t i = 0; i < n; i++) observe(v[i]); }
uint32_t HostChallenger::sample() {
    if (nin != 0 || nout == 0) duplexing();
    return outbuf[--nout];
}
void HostChallenger::sample_ext(uint32_t* out4) { for (int i = 0; i < 4; i++) out4[i] = sample(); }
uint32_t HostChallenger::sample_bits(uint32_t bits) { return kb::to_canonical(sample()) & ((1u << bits) - 1u); }
bool HostChallenger::check_witness(uint32_t bits, uint32_t w_monty) { observe(w_monty); return sample_bits(bits) == 0; }
sp1b200_err HostChallenger::grind(uint32_t bits, uint32_t* w_monty) {
    uint32_t st[34];
    store(st);
    SP1_CUDA(cudaMemcpyAsync(d_scratch, st, sizeof(st), cudaMemcpyHostToDevice, ctx->stream));
    uint32_t wc;
    SP1_TRY(sp1b200_grind_device(ctx, d_scratch, bits, &wc));
    SP1_CUDA(cudaMemcpyAsync(st, d_scratch, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
    SP1_CUDA(cudaStreamSynchronize(ctx->stream));
    load(st);
    *w_monty = kb::to_monty_c(wc);
    return nullptr;
}

extern "C" sp1b200_err sp1b200_grind(sp1b200_ctx* ctx, uint32_t* h_state34, uint32_t bits, uint32_t* h_witness) { SP1_DEVICE_GUARD(ctx);
    HostChallenger ch;
    SP1_TRY(ch.init(ctx, h_state34));
    PhaseTimer t(ctx, "grind");
    SP1_TRY(ch.grind(bits, h_witness));
    t.stop();
    ch.store(h_state34);
    return nullptr;
}

extern "C" {
void sp1b200_challenger_init(uint32_t* st) { memset(st, 0, 34 * sizeof(uint32_t)); }
void sp1b200_challenger_observe(uint32_t* st, const uint32_t* v, uint64_t n) {
    HostChallenger ch; ch.load(st); ch.observe_n(v, n); ch.store(st);
}
void sp1b200_challenger_sample(uint32_t* st, uint32_t* out, uint64_t n) {
    HostChallenger ch; ch.load(st); for (uint64_t i = 0; i < n; i++) out[i] = ch.sample(); ch.store(st);
}
uint32_t sp1b200_challenger_sample_bits(uint32_t* st, uint32_t bits) {
    HostChallenger ch; ch.load(st); uint32_t r = ch.sample_bits(bits); ch.store(st); return r;
}
int sp1b200_challenger_check_witness(uint32_t* st, uint32_t bits, uint32_t w) {
    HostChallenger ch; ch.load(st); bool ok = ch.check_witness(bits, w); ch.store(st); return ok;
}
}
