// tests/cxx/fidx_driver.cpp -- C++ caller of the fixed-index surface of include/pbsgpu.hpp (transfer::FixedIndexWriter,
// KnownSet::SeedFromFidx), standing in for the Go image writer.  Usage: fidx_driver <chunk_size> <image> <out.fidx>.
// Backs the image up in slices of 4 chunks with _lzh blobs and prints `chunk <digest hex> <known>` per chunk and
// `blob <digest hex> <chunk len> <blob hex>` per new chunk, writes the .fidx, then seeds a new set from it and backs the
// image up again: `seeded-rerun-known all` when every chunk is known.  tests/test_gpu_fidx.py checks the output.
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/pbsgpu.hpp"

static void hex(const uint8_t *p, uint64_t n) { for (uint64_t k = 0; k < n; k++) std::printf("%02x", p[k]); }

int main(int argc, char **argv) {
    if (argc != 4) return 2;
    try {
        const uint32_t cs = (uint32_t)std::stoul(argv[1]);
        FILE *f = std::fopen(argv[2], "rb");
        if (!f) return 2;
        std::vector<uint8_t> img;
        uint8_t buf[1 << 16];
        for (size_t k; (k = std::fread(buf, 1, sizeof buf, f)) > 0;) img.insert(img.end(), buf, buf + k);
        std::fclose(f);
        pbsgpu::Engine eng(0);
        pbsgpu::KnownSet known(eng);
        std::vector<std::vector<uint8_t>> blobs;
        pbsgpu::transfer::FixedIndexWriter w(eng, cs, &known, PBSGPU_BLOB_LZH,
                                             [&](const uint8_t *, const uint8_t *b, uint64_t len) { blobs.emplace_back(b, b + len); });
        const uint64_t step = 4ull * cs;
        for (uint64_t a = 0; a < img.size(); a += step) w.WriteSlice(img.data() + a, std::min<uint64_t>(step, img.size() - a));
        const std::vector<uint8_t> fidx = w.Finish();
        const uint64_t n = w.Digests().size() / 32;
        size_t b = 0;
        for (uint64_t i = 0; i < n; i++) {
            const uint8_t *d = w.Digests().data() + 32 * i;
            std::printf("chunk "); hex(d, 32); std::printf(" %d\n", w.Known()[i] ? 1 : 0);
            if (w.Known()[i]) continue;
            if (b >= blobs.size()) { std::fprintf(stderr, "fewer blobs than new chunks\n"); return 1; }
            std::printf("blob "); hex(d, 32);
            std::printf(" %llu ", (unsigned long long)std::min<uint64_t>(cs, img.size() - i * cs));
            hex(blobs[b].data(), blobs[b].size()); std::printf("\n");
            b++;
        }
        if (b != blobs.size()) { std::fprintf(stderr, "more blobs than new chunks\n"); return 1; }
        FILE *o = std::fopen(argv[3], "wb");
        if (!o || std::fwrite(fidx.data(), 1, fidx.size(), o) != fidx.size()) return 2;
        std::fclose(o);
        pbsgpu::KnownSet seeded(eng);
        if (seeded.SeedFromFidx(fidx) != n) { std::fprintf(stderr, "seed count differs\n"); return 1; }
        pbsgpu::transfer::FixedIndexWriter again(eng, cs, &seeded);
        again.WriteSlice(img.data(), img.size());
        bool all = true;
        for (bool k : again.Known()) all = all && k;
        std::printf("seeded-rerun-known %s\n", all && again.Finish() == fidx ? "all" : "NOT");
    } catch (const pbsgpu::Error &e) {
        std::fprintf(stderr, "pbsgpu error %d: %s\n", e.code, e.what());
        return 1;
    }
    return 0;
}
