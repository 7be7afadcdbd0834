// pbs_plus_b200/csrc/capi_crypt.cu -- encrypt mode's key handle (pbsgpu_crypt_*): the K11 tables of one AES-256 key, the
// id_key of keyed digests derived on the host, and the IVs of a stream's encrypted blobs.
#include <errno.h>
#include <sys/random.h>

#include <cstring>

#include "host.hpp"

using namespace pbsgpu;

// Host SHA-256 (FIPS 180-4) for the key derivation: 20 compressions per crypt handle, so no device work
struct HostSha256 {
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    uint8_t buf[64];
    uint64_t n = 0;
    static uint32_t ror(uint32_t x, int r) { return (x >> r) | (x << (32 - r)); }
    void block(const uint8_t *p) {
        static const uint32_t K[64] = {
            0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
            0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
            0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
            0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
            0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
            0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
            0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
        uint32_t w[64], v[8];
        for (int i = 0; i < 16; i++) w[i] = (uint32_t)p[4 * i] << 24 | (uint32_t)p[4 * i + 1] << 16 | (uint32_t)p[4 * i + 2] << 8 | p[4 * i + 3];
        for (int i = 16; i < 64; i++)
            w[i] = w[i - 16] + (ror(w[i - 15], 7) ^ ror(w[i - 15], 18) ^ (w[i - 15] >> 3)) + w[i - 7] +
                   (ror(w[i - 2], 17) ^ ror(w[i - 2], 19) ^ (w[i - 2] >> 10));
        memcpy(v, h, sizeof v);
        for (int i = 0; i < 64; i++) {
            const uint32_t t1 = v[7] + (ror(v[4], 6) ^ ror(v[4], 11) ^ ror(v[4], 25)) + ((v[4] & v[5]) ^ (~v[4] & v[6])) + K[i] + w[i];
            const uint32_t t2 = (ror(v[0], 2) ^ ror(v[0], 13) ^ ror(v[0], 22)) + ((v[0] & v[1]) ^ (v[0] & v[2]) ^ (v[1] & v[2]));
            memmove(v + 1, v, 7 * sizeof(uint32_t));
            v[4] += t1; v[0] = t1 + t2;
        }
        for (int i = 0; i < 8; i++) h[i] += v[i];
    }
    void update(const uint8_t *p, size_t len) {
        for (size_t i = 0; i < len; i++) { buf[n++ & 63] = p[i]; if ((n & 63) == 0) block(buf); }
    }
    void final(uint8_t out[32]) {
        const uint64_t bits = n * 8;
        const uint8_t one = 0x80, zero = 0;
        update(&one, 1);
        while ((n & 63) != 56) update(&zero, 1);
        for (int i = 7; i >= 0; i--) { const uint8_t b = (uint8_t)(bits >> (8 * i)); update(&b, 1); }
        for (int i = 0; i < 8; i++) for (int k = 0; k < 4; k++) out[4 * i + k] = (uint8_t)(h[i] >> (24 - 8 * k));
    }
};
static void hmac_sha256(const uint8_t key[32], const uint8_t *msg, size_t len, uint8_t out[32]) {
    uint8_t pad[64], inner[32];
    HostSha256 a, b;
    for (int i = 0; i < 64; i++) pad[i] = (uint8_t)((i < 32 ? key[i] : 0) ^ 0x36);
    a.update(pad, 64); a.update(msg, len); a.final(inner);
    for (int i = 0; i < 64; i++) pad[i] ^= 0x36 ^ 0x5c;
    b.update(pad, 64); b.update(inner, 32); b.final(out);
}
// upstream CryptConfig::new: id_key = PBKDF2-HMAC-SHA256(key, "_id_key", 10 iterations, 32 bytes) -- one output block
static void derive_id_key(const uint8_t key[32], uint8_t out[32]) {
    const uint8_t salt[11] = {'_', 'i', 'd', '_', 'k', 'e', 'y', 0, 0, 0, 1};   // salt || INT(1)
    uint8_t u[32], t[32];
    hmac_sha256(key, salt, sizeof salt, u);
    memcpy(t, u, 32);
    for (int it = 1; it < 10; it++) {
        hmac_sha256(key, u, 32, u);
        for (int i = 0; i < 32; i++) t[i] ^= u[i];
    }
    memcpy(out, t, 32);
    volatile uint8_t *z = u;
    for (int i = 0; i < 32; i++) z[i] = 0, t[i] = 0;
}

int pbsgpu_stream_ivs(pbsgpu_ctx *ctx, const uint8_t *seed, uint64_t first, uint32_t n, uint8_t *iv) {
    if (!seed) {
        for (size_t got = 0; got < 16ull * n;) {
            const ssize_t r = getrandom(iv + got, 16ull * n - got, 0);
            if (r < 0 && errno != EINTR) return fail(ctx, PBSGPU_EINVAL, "getrandom failed: %s", strerror(errno));
            if (r > 0) got += (size_t)r;
        }
        return PBSGPU_OK;
    }
    for (uint32_t i = 0; i < n; i++) {
        uint8_t msg[40], d[32];
        memcpy(msg, seed, 32);
        for (int k = 0; k < 8; k++) msg[32 + k] = (uint8_t)((first + i) >> (8 * k));
        HostSha256 h;
        h.update(msg, sizeof msg);
        h.final(d);
        memcpy(iv + 16ull * i, d, 16);
    }
    return PBSGPU_OK;
}

extern "C" int pbsgpu_crypt_create(pbsgpu_ctx *ctx, const uint8_t key[32], pbsgpu_crypt **out) {
    if (!ctx || !key || !out) return PBSGPU_EINVAL;
    Guard g(ctx);
    pbsgpu_crypt *c = new pbsgpu_crypt{ctx, std::vector<uint8_t>(gcm_tables_bytes() + 32), nullptr};
    gcm_fill_tables_host(key, c->tab.data());
    derive_id_key(key, c->tab.data() + gcm_tables_bytes());
    cudaError_t e = cudaMalloc((void **)&c->d_tab, c->tab.size());
    if (e == cudaSuccess) e = cudaMemcpy(c->d_tab, c->tab.data(), c->tab.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        pbsgpu_crypt_destroy(c);
        return fail(ctx, PBSGPU_ECUDA, "crypt tables: %s", cudaGetErrorString(e));
    }
    *out = c;
    return PBSGPU_OK;
}

extern "C" void pbsgpu_crypt_destroy(pbsgpu_crypt *c) {
    if (!c) return;
    Guard g(c->ctx);
    if (c->d_tab) {
        if (cudaMemset(c->d_tab, 0, c->tab.size()) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) (void)cudaGetLastError();
        cudaFree(c->d_tab);
    }
    volatile uint8_t *p = c->tab.data();   // volatile: the zeroing of memory that is freed next is not optimised away
    for (size_t i = 0; i < c->tab.size(); i++) p[i] = 0;
    delete c;
}
