// model.cpp -- see model.hpp.  Host only (g++).
#include "model.hpp"

#include <cctype>
#include <cstdlib>
#include <cstring>

#ifndef NNB_WEIGHTS_PATH
#error "NNB_WEIGHTS_PATH must point at data/weights.rnn"
#endif

// Embed the built-in model (the reference does the same with include_bytes!, src/rnn.rs:237).
__asm__(".section .rodata\n"
        ".global nnb_builtin_weights\n"
        ".global nnb_builtin_weights_end\n"
        ".balign 16\n"
        "nnb_builtin_weights:\n"
        ".incbin \"" NNB_WEIGHTS_PATH "\"\n"
        "nnb_builtin_weights_end:\n"
        ".byte 0\n"
        ".text\n");
extern "C" const unsigned char nnb_builtin_weights[];
extern "C" const unsigned char nnb_builtin_weights_end[];

namespace nnb {

const float kTansigTable[201] = {
    0.000000f, 0.039979f, 0.079830f, 0.119427f, 0.158649f, 0.197375f, 0.235496f, 0.272905f, 0.309507f, 0.345214f, 0.379949f,
    0.413644f, 0.446244f, 0.477700f, 0.507977f, 0.537050f, 0.564900f, 0.591519f, 0.616909f, 0.641077f, 0.664037f, 0.685809f,
    0.706419f, 0.725897f, 0.744277f, 0.761594f, 0.777888f, 0.793199f, 0.807569f, 0.821040f, 0.833655f, 0.845456f, 0.856485f,
    0.866784f, 0.876393f, 0.885352f, 0.893698f, 0.901468f, 0.908698f, 0.915420f, 0.921669f, 0.927473f, 0.932862f, 0.937863f,
    0.942503f, 0.946806f, 0.950795f, 0.954492f, 0.957917f, 0.961090f, 0.964028f, 0.966747f, 0.969265f, 0.971594f, 0.973749f,
    0.975743f, 0.977587f, 0.979293f, 0.980869f, 0.982327f, 0.983675f, 0.984921f, 0.986072f, 0.987136f, 0.988119f, 0.989027f,
    0.989867f, 0.990642f, 0.991359f, 0.992020f, 0.992631f, 0.993196f, 0.993718f, 0.994199f, 0.994644f, 0.995055f, 0.995434f,
    0.995784f, 0.996108f, 0.996407f, 0.996682f, 0.996937f, 0.997172f, 0.997389f, 0.997590f, 0.997775f, 0.997946f, 0.998104f,
    0.998249f, 0.998384f, 0.998508f, 0.998623f, 0.998728f, 0.998826f, 0.998916f, 0.999000f, 0.999076f, 0.999147f, 0.999213f,
    0.999273f, 0.999329f, 0.999381f, 0.999428f, 0.999472f, 0.999513f, 0.999550f, 0.999585f, 0.999617f, 0.999646f, 0.999673f,
    0.999699f, 0.999722f, 0.999743f, 0.999763f, 0.999781f, 0.999798f, 0.999813f, 0.999828f, 0.999841f, 0.999853f, 0.999865f,
    0.999875f, 0.999885f, 0.999893f, 0.999902f, 0.999909f, 0.999916f, 0.999923f, 0.999929f, 0.999934f, 0.999939f, 0.999944f,
    0.999948f, 0.999952f, 0.999956f, 0.999959f, 0.999962f, 0.999965f, 0.999968f, 0.999970f, 0.999973f, 0.999975f, 0.999977f,
    0.999978f, 0.999980f, 0.999982f, 0.999983f, 0.999984f, 0.999986f, 0.999987f, 0.999988f, 0.999989f, 0.999990f, 0.999990f,
    0.999991f, 0.999992f, 0.999992f, 0.999993f, 0.999994f, 0.999994f, 0.999994f, 0.999995f, 0.999995f, 0.999996f, 0.999996f,
    0.999996f, 0.999997f, 0.999997f, 0.999997f, 0.999997f, 0.999997f, 0.999998f, 0.999998f, 0.999998f, 0.999998f, 0.999998f,
    0.999998f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f,
    0.999999f, 0.999999f, 0.999999f, 1.000000f, 1.000000f, 1.000000f, 1.000000f, 1.000000f, 1.000000f, 1.000000f, 1.000000f,
    1.000000f, 1.000000f, 1.000000f,
};

namespace {
struct Cursor {
    const int8_t* base;
    size_t pos, len;
    size_t left() const { return len - pos; }
};

bool read_header(Cursor& c, int* ni, int* nn, int* act) {
    if (c.left() < 3) return false;
    const int8_t* b = c.base + c.pos;
    // header byte order is [nb_inputs, nb_neurons, activation] (src/rnn.rs:150-152, 171-173);
    // negative sizes are rejected by `unsigned` (src/rnn.rs:128-134)
    if (b[0] < 0 || b[1] < 0) return false;
    if (b[2] < 0 || b[2] > 2) return false;  // src/rnn.rs:136-143
    *ni = b[0];
    *nn = b[1];
    *act = b[2];
    c.pos += 3;
    return true;
}

bool take(Cursor& c, size_t n, size_t* off) {
    if (c.left() < n) return false;
    *off = c.pos;
    c.pos += n;
    return true;
}

bool read_dense(Cursor& c, HostDense* l) {
    return read_header(c, &l->ni, &l->nn, &l->act) && take(c, (size_t)l->ni * l->nn, &l->w_off) &&
           take(c, (size_t)l->nn, &l->b_off);
}

bool read_gru(Cursor& c, HostGru* l) {
    return read_header(c, &l->ni, &l->nn, &l->act) && take(c, (size_t)3 * l->nn * l->ni, &l->w_off) &&
           take(c, (size_t)3 * l->nn * l->nn, &l->r_off) && take(c, (size_t)3 * l->nn, &l->b_off);
}
}  // namespace

bool HostModel::parse(const uint8_t* data, size_t len, HostModel* m) {
    m->bytes.assign(reinterpret_cast<const int8_t*>(data), reinterpret_cast<const int8_t*>(data) + len);
    Cursor c{m->bytes.data(), 0, len};
    // layer order: src/rnn.rs:189-194
    bool ok = read_dense(c, &m->input_dense) && read_gru(c, &m->vad_gru) && read_gru(c, &m->noise_gru) &&
              read_gru(c, &m->denoise_gru) && read_dense(c, &m->denoise_output) && read_dense(c, &m->vad_output);
    if (!ok || c.left() != 0) return false;  // src/rnn.rs:196-198
    // src/rnn.rs:204-222
    if (m->input_dense.ni != 42 || m->denoise_output.nn != 22 || m->vad_output.nn != 1) return false;
    if (m->input_dense.nn != m->vad_gru.ni || m->vad_gru.nn != m->vad_output.ni) return false;
    if (42 + m->input_dense.nn + m->vad_gru.nn != m->noise_gru.ni) return false;
    if (42 + m->vad_gru.nn + m->noise_gru.nn != m->denoise_gru.ni) return false;
    if (m->denoise_gru.nn != m->denoise_output.ni) return false;
    return true;
}

bool HostModel::parse_text(const char* text, size_t len, HostModel* out) {
    static const char kHeader[] = "rnnoise-nu model file version 1";
    size_t eol = 0;
    while (eol < len && text[eol] != '\n') eol++;
    size_t h = eol;
    while (h > 0 && std::isspace((unsigned char)text[h - 1])) h--;
    size_t b = 0;
    while (b < h && std::isspace((unsigned char)text[b])) b++;
    if (h - b != sizeof(kHeader) - 1 || std::memcmp(text + b, kHeader, h - b) != 0) return false;
    std::vector<uint8_t> bin;
    size_t i = eol;
    while (i < len) {
        while (i < len && std::isspace((unsigned char)text[i])) i++;
        if (i >= len) break;
        bool neg = false;
        if (text[i] == '-' || text[i] == '+') {
            neg = text[i] == '-';
            i++;
        }
        if (i >= len || !std::isdigit((unsigned char)text[i])) return false;
        long v = 0;
        while (i < len && std::isdigit((unsigned char)text[i])) {
            v = v * 10 + (text[i] - '0');
            if (v > 1000000) return false;
            i++;
        }
        if (neg) v = -v;
        long mod = ((v % 256) + 256) % 256;  // python's int(s) % 256
        bin.push_back((uint8_t)mod);
    }
    return parse(bin.data(), bin.size(), out);
}

const HostModel& HostModel::builtin() {
    static const HostModel* m = [] {
        HostModel* p = new HostModel();
        bool ok = HostModel::parse(nnb_builtin_weights, (size_t)(nnb_builtin_weights_end - nnb_builtin_weights), p);
        if (!ok) std::abort();  // the reference unwrap()s (src/rnn.rs:238)
        return p;
    }();
    return *m;
}

}  // namespace nnb
