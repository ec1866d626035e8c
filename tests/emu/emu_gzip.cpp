// tests/emu/emu_gzip.cpp -- the deflate pieces of dp_core.cuh that gzip_block_kernel runs (code lengths, canonical codes, the
// dynamic header, CRC-32 and its combination) compiled for the host, so that the no-GPU tier can check them against zlib.
// A whole block is encoded here with a plain host LZ77 (one hash candidate per position, greedy) and the same header and code
// writers.  TEST ONLY: the product never builds or loads this file.
#include <cstdint>
#include <cstring>
#include <vector>
#include "../../porechop_b200/csrc/dp_core.cuh"

extern "C" void emu_code_lengths(const uint32_t *freq, int n, int limit, uint8_t *len) {
    std::vector<uint32_t> work(2 * n + 16);
    pb::gz_code_lengths(freq, n, limit, len, work.data());
}

extern "C" uint32_t emu_crc32(uint32_t crc, const uint8_t *p, int64_t n) {
    uint32_t table[256];
    for (uint32_t i = 0; i < 256; ++i) table[i] = pb::gz_crc_table_entry(i);
    return pb::gz_crc_update(crc, table, p, n);
}

extern "C" uint32_t emu_crc32_combine(uint32_t a, uint32_t b, int64_t len_b) { return pb::gz_crc_combine(a, b, len_b); }

// one final dynamic deflate block of in[0 .. n) into out (zeroed, cap bytes); returns its bytes, or -1 when it does not fit
extern "C" int64_t emu_deflate_block(const uint8_t *in, int n, uint8_t *out, int64_t cap) {
    using namespace pb;
    std::vector<uint32_t> tok;
    std::vector<int> head(1 << 15, -1);
    for (int p = 0; p < n;) {
        int best = 0, dist = 0;
        if (p + 3 <= n) {
            const uint32_t h = (((uint32_t)in[p] << 16) | ((uint32_t)in[p + 1] << 8) | in[p + 2]) * 2654435761u >> 17;
            const int q = head[h];
            head[h] = p;
            if (q >= 0 && p - q <= 32768) {
                int l = 0;
                while (l < 258 && p + l < n && in[q + l] == in[p + l]) ++l;
                if (l >= 3) { best = l; dist = p - q; }
            }
        }
        if (best) { tok.push_back(0x80000000u | ((uint32_t)(best - 3) << 16) | (uint32_t)(dist - 1)); p += best; }
        else tok.push_back(in[p++]);
    }
    uint32_t ll_freq[GZ_LITLEN] = {0}, d_freq[GZ_DIST] = {0};
    for (uint32_t t : tok) {
        if (t >> 31) {
            int ls, le, lv, ds, de, dv;
            gz_len_sym((int)((t >> 16) & 255u) + 3, ls, le, lv);
            gz_dist_sym((int)(t & 32767u) + 1, ds, de, dv);
            ll_freq[ls]++; d_freq[ds]++;
        } else {
            ll_freq[t]++;
        }
    }
    ll_freq[256] = 1;
    uint8_t ll_len[GZ_LITLEN], d_len[GZ_DIST], all[GZ_LITLEN + GZ_DIST];
    uint16_t ll_code[GZ_LITLEN], d_code[GZ_DIST];
    std::vector<uint32_t> work(2 * GZ_LITLEN + 16);
    gz_code_lengths(ll_freq, GZ_LITLEN, GZ_MAX_BITS, ll_len, work.data());
    gz_code_lengths(d_freq, GZ_DIST, GZ_MAX_BITS, d_len, work.data());
    gz_canonical_codes(ll_len, GZ_LITLEN, ll_code);
    gz_canonical_codes(d_len, GZ_DIST, d_code);
    GzDynHeader H;
    gz_dynamic_header(ll_len, d_len, H, all, work.data());
    std::vector<uint32_t> w((size_t)(cap / 4 + 2), 0u);
    GzBitWriter bw{w.data(), 0};
    gz_write_dynamic_header(bw, 1, H);
    for (uint32_t t : tok) {
        if ((int64_t)(bw.pos / 8) + 16 > cap) return -1;
        if (!(t >> 31)) { bw.put(ll_code[t], ll_len[t]); continue; }
        int ls, le, lv, ds, de, dv;
        gz_len_sym((int)((t >> 16) & 255u) + 3, ls, le, lv);
        gz_dist_sym((int)(t & 32767u) + 1, ds, de, dv);
        bw.put(ll_code[ls], ll_len[ls]); bw.put((uint32_t)lv, le);
        bw.put(d_code[ds], d_len[ds]); bw.put((uint32_t)dv, de);
    }
    bw.put(ll_code[256], ll_len[256]);
    const int64_t bytes = (int64_t)((bw.pos + 7) / 8);
    if (bytes > cap) return -1;
    memcpy(out, w.data(), (size_t)bytes);
    return bytes;
}
