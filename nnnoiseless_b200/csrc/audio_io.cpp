// audio_io.cpp -- see audio_io.hpp.  Sample decoding follows src/nnnoiseless.rs:57-77 (raw) and :190-228 (WAV):
//   integer PCM of b bits : b < 16 -> s << (16 - b);  b >= 16 -> s >> (b - 16)   (8-bit WAV is unsigned: u8 - 128)
//   32-bit float          : s * 32767.0
#include "audio_io.hpp"

#include <cerrno>
#include <cstdio>
#include <cstring>

namespace nnb {

namespace {

bool slurp(const std::string& path, std::vector<unsigned char>* data, std::string* err, const char* what) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) {
        *err = std::string("Failed to open ") + what + " file \"" + path + "\": " + strerror(errno);  // :251-253
        return false;
    }
    unsigned char chunk[1 << 16];
    size_t n;
    while ((n = fread(chunk, 1, sizeof chunk, f)) > 0) data->insert(data->end(), chunk, chunk + n);
    const bool bad = ferror(f) != 0;
    fclose(f);
    if (bad) {
        *err = "read error on \"" + path + "\"";
        return false;
    }
    return true;
}

inline uint32_t le32(const unsigned char* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
inline uint16_t le16(const unsigned char* p) { return (uint16_t)(p[0] | (p[1] << 8)); }

void put16(std::vector<unsigned char>& v, uint16_t x) {
    v.push_back((unsigned char)(x & 0xff));
    v.push_back((unsigned char)(x >> 8));
}
void put32(std::vector<unsigned char>& v, uint32_t x) {
    for (int i = 0; i < 4; i++) v.push_back((unsigned char)((x >> (8 * i)) & 0xff));
}

bool write_all(const std::string& path, const std::vector<unsigned char>& head, const int16_t* pcm, size_t n, std::string* err) {
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) {
        *err = "Failed to open output file \"" + path + "\": " + strerror(errno);  // :255-257
        return false;
    }
    bool ok = head.empty() || fwrite(head.data(), 1, head.size(), f) == head.size();
    // int16 little-endian: this library only targets little-endian hosts (x86-64 / aarch64 + CUDA)
    if (ok && n) ok = fwrite(pcm, sizeof(int16_t), n, f) == n;
    if (fclose(f) != 0) ok = false;
    if (!ok) *err = "write error on \"" + path + "\"";
    return ok;
}

}  // namespace

bool has_wav_extension(const std::string& path) {
    const size_t slash = path.find_last_of('/');
    const std::string name = slash == std::string::npos ? path : path.substr(slash + 1);
    const size_t dot = name.find_last_of('.');
    if (dot == std::string::npos || dot == 0) return false;  // ".wav" alone has no extension (Path::extension)
    return name.substr(dot + 1) == "wav";
}

bool read_raw_file(const std::string& path, int channels, double sample_rate, AudioData* out, std::string* err) {
    if (channels < 1) {
        *err = "channels must be at least 1";
        return false;
    }
    std::vector<unsigned char> d;
    if (!slurp(path, &d, err, "input")) return false;
    if (d.size() % 2) {
        *err = "Unexpected end of input (expected an even number of bytes)";  // :68-70
        return false;
    }
    const size_t n = d.size() / 2;
    if (n % (size_t)channels) {
        *err = "Unexpected end of input (expected a multiple of " + std::to_string(channels) + " samples)";  // :88-91
        return false;
    }
    out->channels = channels;
    out->sample_rate = sample_rate;
    out->samples.resize(n);
    for (size_t i = 0; i < n; i++) out->samples[i] = (float)(int16_t)le16(&d[2 * i]);
    return true;
}

namespace {

// Reads n bytes at pos of a WAV source into dst; false if fewer are there.
struct ByteSource {
    size_t size;
    virtual bool read(size_t pos, size_t n, unsigned char* dst) const = 0;
};

struct MemorySource : ByteSource {
    const unsigned char* d;
    MemorySource(const std::vector<unsigned char>& v) : d(v.data()) { size = v.size(); }
    bool read(size_t pos, size_t n, unsigned char* dst) const override {
        if (pos > size || n > size - pos) return false;
        memcpy(dst, d + pos, n);
        return true;
    }
};

struct FileSource : ByteSource {
    FILE* f;
    bool read(size_t pos, size_t n, unsigned char* dst) const override {
        if (pos > size || n > size - pos) return false;
        return fseeko(f, (off_t)pos, SEEK_SET) == 0 && fread(dst, 1, n, f) == n;
    }
};

// The RIFF/fmt/data walk of hound 3.x up to the first sample: format checks and the data chunk's place.
bool parse_wav_header(const ByteSource& src, WavHeader* h, std::string* err) {
    auto bad = [&](const char* why) {
        *err = std::string("Ill-formed WAVE file: ") + why;  // hound::Error::FormatError
        return false;
    };
    unsigned char b[40];
    if (!src.read(0, 4, b) || memcmp(b, "RIFF", 4) != 0) return bad("no RIFF tag found");
    if (!src.read(8, 4, b) || memcmp(b, "WAVE", 4) != 0) return bad("no WAVE tag found");
    size_t p = 12;
    bool have_fmt = false;
    int fmt_tag = 0, channels = 0, bits = 0, block_align = 0;
    uint32_t rate = 0;
    for (;;) {
        if (!src.read(p, 8, b)) return bad(have_fmt ? "no data chunk found" : "no fmt chunk found");
        unsigned char id[4];
        memcpy(id, b, 4);
        const size_t len = le32(&b[4]);
        p += 8;
        if (memcmp(id, "fmt ", 4) == 0) {
            if (len < 16 || len > src.size - p || !src.read(p, len < 40 ? len : 40, b)) return bad("invalid fmt chunk size");
            fmt_tag = le16(&b[0]);
            channels = le16(&b[2]);
            rate = le32(&b[4]);
            block_align = le16(&b[12]);
            bits = le16(&b[14]);
            if (fmt_tag == 0xfffe) {  // WAVE_FORMAT_EXTENSIBLE: the sub-format GUID starts with the real tag
                if (len < 40) return bad("unexpected fmt chunk size");
                fmt_tag = le16(&b[24]);
            }
            have_fmt = true;
        } else if (memcmp(id, "data", 4) == 0) {
            if (!have_fmt) return bad("data chunk before fmt chunk");
            if (channels < 1) return bad("file contains zero channels");
            const int bytes = block_align / channels;
            if (fmt_tag == 1) {
                if (bytes < 1 || bytes > 4 || bits < 1 || bits > 8 * bytes) {
                    *err = "The wave format of the file is not supported.";
                    return false;
                }
            } else if (fmt_tag == 3) {
                if (bits != 32 || bytes != 4) {
                    *err = "The wave format of the file is not supported.";
                    return false;
                }
            } else {
                *err = "The wave format of the file is not supported.";
                return false;
            }
            size_t avail = src.size - p;
            if (len > avail) {
                *err = "Failed to read enough bytes.";
                return false;
            }
            const size_t n = len / (size_t)bytes;
            if (n % (size_t)channels) {
                *err = "Unexpected end of input (expected a multiple of " + std::to_string(channels) + " samples)";
                return false;
            }
            h->fmt_tag = fmt_tag;
            h->channels = channels;
            h->sample_rate = rate;
            h->bits = bits;
            h->bytes = bytes;
            h->data_offset = p;
            h->n_frames = n / (size_t)channels;
            return true;
        }
        p += len + (len & 1);  // chunks are word aligned
    }
}

}  // namespace

bool probe_wav_file(const std::string& path, WavHeader* h, std::string* err) {
    FileSource src;
    src.f = fopen(path.c_str(), "rb");
    if (!src.f) {
        *err = std::string("Failed to open input file \"") + path + "\": " + strerror(errno);
        return false;
    }
    bool ok = fseeko(src.f, 0, SEEK_END) == 0;
    const off_t size = ok ? ftello(src.f) : -1;
    if (!ok || size < 0) {
        fclose(src.f);
        *err = "read error on \"" + path + "\"";
        return false;
    }
    src.size = (size_t)size;
    ok = parse_wav_header(src, h, err);
    fclose(src.f);
    return ok;
}

bool read_wav_file(const std::string& path, AudioData* out, std::string* err) {
    std::vector<unsigned char> d;
    if (!slurp(path, &d, err, "input")) return false;
    WavHeader h;
    if (!parse_wav_header(MemorySource(d), &h, err)) return false;
    const size_t n = h.n_frames * (size_t)h.channels;
    const int bytes = h.bytes, bits = h.bits;
    out->channels = h.channels;
    out->sample_rate = (double)h.sample_rate;
    out->samples.resize(n);
    const unsigned char* s = d.data() + h.data_offset;
    for (size_t i = 0; i < n; i++, s += bytes) {
        if (h.fmt_tag == 3) {
            float v;
            uint32_t u = le32(s);
            memcpy(&v, &u, 4);
            out->samples[i] = v * 32767.0f;  // :216-218
            continue;
        }
        int32_t v;
        switch (bytes) {
            case 1: v = (int32_t)s[0] - 128; break;  // hound: unsigned 8-bit -> i8
            case 2: v = (int16_t)le16(s); break;
            case 3: v = (int32_t)((uint32_t)s[0] | ((uint32_t)s[1] << 8) | ((uint32_t)s[2] << 16)); v = (v << 8) >> 8; break;
            default: v = (int32_t)le32(s); break;
        }
        out->samples[i] = bits < 16 ? (float)(int32_t)((uint32_t)v << (16 - bits)) : (float)(v >> (bits - 16));  // :199-205
    }
    return true;
}

bool write_raw_file(const std::string& path, const int16_t* pcm, long n_frames, int channels, std::string* err) {
    return write_all(path, {}, pcm, (size_t)n_frames * (size_t)channels, err);
}

bool write_wav_file(const std::string& path, const int16_t* pcm, long n_frames, int channels, std::string* err) {
    const uint64_t data_bytes = (uint64_t)n_frames * (uint64_t)channels * 2;
    const bool ext = channels > 2;  // hound writes WAVEFORMATEXTENSIBLE beyond stereo / 16 bits
    const uint32_t fmt_len = ext ? 40 : 16;
    if (data_bytes + 20 + fmt_len > 0xffffffffull) {
        *err = "output too large for a RIFF/WAVE file";
        return false;
    }
    std::vector<unsigned char> h;
    h.insert(h.end(), {'R', 'I', 'F', 'F'});
    put32(h, (uint32_t)(4 + 8 + fmt_len + 8 + data_bytes));
    h.insert(h.end(), {'W', 'A', 'V', 'E', 'f', 'm', 't', ' '});
    put32(h, fmt_len);
    put16(h, ext ? 0xfffe : 1);
    put16(h, (uint16_t)channels);
    put32(h, 48000);
    put32(h, 48000u * (uint32_t)channels * 2);
    put16(h, (uint16_t)(channels * 2));
    put16(h, 16);
    if (ext) {
        put16(h, 22);                                                     // cbSize
        put16(h, 16);                                                     // valid bits per sample
        put32(h, channels >= 32 ? 0xffffffffu : ((1u << channels) - 1));  // speaker mask: the first `channels` positions
        static const unsigned char pcm_guid[16] = {0x01, 0x00, 0x00, 0x00, 0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xaa, 0x00, 0x38, 0x9b, 0x71};
        h.insert(h.end(), pcm_guid, pcm_guid + 16);
    }
    h.insert(h.end(), {'d', 'a', 't', 'a'});
    put32(h, (uint32_t)data_bytes);
    return write_all(path, h, pcm, (size_t)n_frames * (size_t)channels, err);
}

}  // namespace nnb
