// Reader of the self-contained model file (layout: include/dd3d_b200.h, dd3d_create_from_file; writer:
// dd3d_b200/lib.py write_model_file).  Host code only.
#include <errno.h>
#include <stdio.h>
#include <string.h>
#include <sys/stat.h>

#include <set>

#include "model_file.cuh"

static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "the model file is little-endian and read in place");

namespace dd3d {
namespace {

// ------------------------------------------------------------------------------------------------ BLAKE2b (RFC 7693)
constexpr uint64_t kBlakeIV[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull,
                                  0xa54ff53a5f1d36f1ull, 0x510e527fade682d1ull, 0x9b05688c2b3e6c1full,
                                  0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
constexpr uint8_t kBlakeSigma[12][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};

inline uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

void blake2b_compress(uint64_t h[8], const uint8_t block[128], uint64_t t, bool last) {
    uint64_t m[16], v[16];
    memcpy(m, block, 128);
    for (int i = 0; i < 8; ++i) v[i] = h[i], v[i + 8] = kBlakeIV[i];
    v[12] ^= t;  // low word of the byte counter; the high word stays 0 below 2^64 bytes
    if (last) v[14] = ~v[14];
    auto G = [&](int a, int b, int c, int d, uint64_t x, uint64_t y) {
        v[a] = v[a] + v[b] + x;
        v[d] = rotr64(v[d] ^ v[a], 32);
        v[c] = v[c] + v[d];
        v[b] = rotr64(v[b] ^ v[c], 24);
        v[a] = v[a] + v[b] + y;
        v[d] = rotr64(v[d] ^ v[a], 16);
        v[c] = v[c] + v[d];
        v[b] = rotr64(v[b] ^ v[c], 63);
    };
    for (int r = 0; r < 12; ++r) {
        const uint8_t* s = kBlakeSigma[r];
        G(0, 4, 8, 12, m[s[0]], m[s[1]]);
        G(1, 5, 9, 13, m[s[2]], m[s[3]]);
        G(2, 6, 10, 14, m[s[4]], m[s[5]]);
        G(3, 7, 11, 15, m[s[6]], m[s[7]]);
        G(0, 5, 10, 15, m[s[8]], m[s[9]]);
        G(1, 6, 11, 12, m[s[10]], m[s[11]]);
        G(2, 7, 8, 13, m[s[12]], m[s[13]]);
        G(3, 4, 9, 14, m[s[14]], m[s[15]]);
    }
    for (int i = 0; i < 8; ++i) h[i] ^= v[i] ^ v[i + 8];
}

// Unkeyed BLAKE2b with an 8-byte digest: Python's hashlib.blake2b(data, digest_size=8).digest().
void blake2b_64(const uint8_t* data, size_t n, uint8_t digest[8]) {
    uint64_t h[8];
    memcpy(h, kBlakeIV, sizeof(h));
    h[0] ^= 0x01010000ull ^ 8ull;  // depth 1, fanout 1, no key, 8-byte digest
    size_t done = 0;
    while (n - done > 128) {
        blake2b_compress(h, data + done, done + 128, false);
        done += 128;
    }
    uint8_t last[128] = {};
    memcpy(last, data + done, n - done);
    blake2b_compress(h, last, n, true);
    memcpy(digest, h, 8);
}

// ------------------------------------------------------------------------------------------------ bounded cursor
struct Cursor {
    const uint8_t* p;
    size_t left;
    std::string* err;

    bool take(void* dst, size_t n, const std::string& what) {
        if (n > left) {
            *err = what + " overruns the file (" + std::to_string(n) + " bytes needed, " + std::to_string(left) +
                   " left before the checksum)";
            return false;
        }
        if (n) memcpy(dst, p, n);
        p += n;
        left -= n;
        return true;
    }
    bool u32(uint32_t* v, const std::string& what) { return take(v, 4, what); }
    bool i32_list(std::vector<int32_t>* v, const std::string& what) {
        uint32_t n;
        if (!u32(&n, what + " count")) return false;
        if (static_cast<uint64_t>(n) * 4 > left) return take(nullptr, static_cast<uint64_t>(n) * 4, what);  // fails
        v->resize(n);
        return take(v->data(), static_cast<size_t>(n) * 4, what);
    }
};

struct Header {
    char magic[8];
    uint32_t version;
    uint32_t desc_bytes;
    uint32_t layout_bytes;
    uint32_t num_tensors;
    uint64_t file_bytes;
};
static_assert(sizeof(Header) == 32, "model file header is 32 bytes");

bool read_all(const char* path, std::vector<uint8_t>* bytes, std::string* err) {
    const std::string p = std::string("model file '") + path + "'";
    FILE* f = fopen(path, "rb");
    if (f == nullptr) {
        *err = "cannot open " + p + ": " + strerror(errno);
        return false;
    }
    struct stat st;
    if (fstat(fileno(f), &st) != 0 || !S_ISREG(st.st_mode)) {
        *err = "cannot read " + p + ": not a regular file";
        fclose(f);
        return false;
    }
    bytes->resize(static_cast<size_t>(st.st_size));
    const size_t got = bytes->empty() ? 0 : fread(bytes->data(), 1, bytes->size(), f);
    const bool ok = got == bytes->size() && !ferror(f);
    if (!ok) *err = "cannot read " + p + ": " + (ferror(f) ? strerror(errno) : "short read");
    fclose(f);
    return ok;
}

}  // namespace

bool read_model_file(const char* path, ModelFile* out, std::string* err) {
    if (!read_all(path, &out->bytes, err)) return false;
    const std::vector<uint8_t>& b = out->bytes;
    const size_t size = b.size();
    const auto truncated = [&](uint64_t need) {
        *err = "model file truncated: " + std::to_string(size) + " bytes, " + std::to_string(need) + " expected";
        return false;
    };
    // header: the magic first, so that any other file is named as such
    if (size < sizeof(kModelFileMagic)) return truncated(sizeof(Header));
    if (memcmp(b.data(), kModelFileMagic, sizeof(kModelFileMagic)) != 0) {
        *err = "bad magic: not a DD3DB200 model file";
        return false;
    }
    if (size < sizeof(Header)) return truncated(sizeof(Header));
    Header hd;
    memcpy(&hd, b.data(), sizeof(hd));
    if (hd.version != kModelFileVersion) {
        *err = "unknown model file version " + std::to_string(hd.version) + " (this library reads version " +
               std::to_string(kModelFileVersion) + ")";
        return false;
    }
    if (hd.desc_bytes != sizeof(dd3d_model_desc) || hd.layout_bytes != sizeof(dd3d_layout_desc)) {
        *err = "struct size mismatch: the file holds a " + std::to_string(hd.desc_bytes) + "-byte dd3d_model_desc and a " +
               std::to_string(hd.layout_bytes) + "-byte dd3d_layout_desc, this library has " +
               std::to_string(sizeof(dd3d_model_desc)) + " and " + std::to_string(sizeof(dd3d_layout_desc));
        return false;
    }
    if (size < hd.file_bytes) return truncated(hd.file_bytes);
    if (size > hd.file_bytes) {
        *err = "model file has " + std::to_string(size - hd.file_bytes) + " bytes after its checksum (" +
               std::to_string(size) + " bytes, the header says " + std::to_string(hd.file_bytes) + ")";
        return false;
    }
    if (size < sizeof(Header) + 8) return truncated(sizeof(Header) + 8);
    uint8_t digest[8];
    blake2b_64(b.data(), size - 8, digest);
    if (memcmp(digest, b.data() + size - 8, 8) != 0) {
        *err = "checksum mismatch: the model file is corrupt";
        return false;
    }

    // body: every read is bounded by the bytes before the checksum
    Cursor c{b.data() + sizeof(Header), size - sizeof(Header) - 8, err};
    if (!c.take(&out->desc, sizeof(out->desc), "dd3d_model_desc") ||
        !c.take(&out->layout, sizeof(out->layout), "dd3d_layout_desc") ||
        !c.take(&out->backbone_norm, 4, "backbone norm") || !c.take(&out->fpn_channels, 4, "FPN width") ||
        !c.i32_list(&out->fpn_inputs, "FPN input list") || !c.i32_list(&out->in_features, "head level list"))
        return false;
    uint32_t canon = 0;
    if (!c.u32(&canon, "canonical size count")) return false;
    if (canon > DD3D_MAX_NUM_CLASSES) {
        *err = "canonical sizes for " + std::to_string(canon) + " classes (at most " +
               std::to_string(DD3D_MAX_NUM_CLASSES) + ")";
        return false;
    }
    out->canon_classes = static_cast<int32_t>(canon);
    out->canon.resize(3 * canon);
    if (!c.take(out->canon.data(), 12 * canon, "canonical sizes")) return false;

    std::set<std::string> names;
    out->tensors.resize(hd.num_tensors);
    for (uint32_t i = 0; i < hd.num_tensors; ++i) {
        ModelFileTensor& t = out->tensors[i];
        const std::string rec = "tensor record " + std::to_string(i);
        uint32_t name_len, ndim;
        if (!c.u32(&name_len, rec + " name length")) return false;
        if (name_len > c.left) return c.take(nullptr, name_len, rec + " name");
        t.name.resize(name_len);
        c.take(&t.name[0], name_len, rec + " name");
        if (name_len == 0 || t.name.find('\0') != std::string::npos) {
            *err = rec + ": empty name or a name with a NUL byte";
            return false;
        }
        const std::string what = rec + " ('" + t.name + "')";
        if (!names.insert(t.name).second) {
            *err = "duplicate tensor name '" + t.name + "' (" + rec + ")";
            return false;
        }
        if (!c.u32(&ndim, what + " ndim")) return false;
        if (ndim > static_cast<uint32_t>(kModelFileMaxNdim)) {
            *err = what + ": ndim " + std::to_string(ndim) + " out of range (0.." + std::to_string(kModelFileMaxNdim) + ")";
            return false;
        }
        t.shape.resize(ndim);
        if (!c.take(t.shape.data(), 8 * ndim, what + " shape")) return false;
        // number of floats, checked against the bytes left before it can overflow
        const uint64_t max_count = c.left / 4;
        uint64_t count = 1;
        bool overrun = false;
        for (int64_t d : t.shape) {
            if (d < 0) {
                *err = what + ": negative dimension " + std::to_string(d);
                return false;
            }
            if (d == 0) count = 0;
        }
        for (int64_t d : t.shape) {
            if (count == 0) break;
            if (static_cast<uint64_t>(d) > max_count / count) {
                overrun = true;
                break;
            }
            count *= static_cast<uint64_t>(d);
        }
        if (overrun) {
            *err = what + " shape overruns the file (" + std::to_string(c.left) + " bytes left before the checksum)";
            return false;
        }
        t.count = static_cast<size_t>(count);
        t.data_offset = static_cast<size_t>(c.p - b.data());
        c.p += 4 * t.count;
        c.left -= 4 * t.count;
    }
    if (c.left != 0) {
        *err = "model file has " + std::to_string(c.left) + " bytes after its last tensor record";
        return false;
    }
    return true;
}

}  // namespace dd3d
