// nnnoiseless-b200 -- command-line front-end with the reference binary's interface (src/nnnoiseless.rs:230-248):
//
//   nnnoiseless-b200 [--wav-in] [--wav-out] [--sample-rate RATE] [--channels N] [--model PATH] INPUT OUTPUT
//
// plus one additive mode for feeding a GPU: `--batch LIST` reads "INPUT<TAB>OUTPUT" lines and denoises all files
// together on recycled GPU streams (every channel of a file is one stream while the file runs; `--slots N` and
// `--chunk-frames K` override the library's defaults), and `--link-channels max|mean` denoises the channels of each
// multi-channel file with one gain curve.  All the work happens in libnnnoiseless_b200.so (rnnoise_denoise_corpus;
// rnnoise_denoise_files_linked when neither option is given, so that a one-file call creates its output before it
// parses the input, as the reference does); there is no CPU path.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "../include/rnnoise.h"

#ifndef NNB_VERSION
#define NNB_VERSION "0.1.0"
#endif

static void usage(FILE* f) {
    fprintf(f,
            "nnnoiseless-b200 %s\nRemove noise from audio files\n\n"
            "USAGE:\n    nnnoiseless-b200 [OPTIONS] <INPUT> <OUTPUT>\n    nnnoiseless-b200 [OPTIONS] --batch <LIST>\n\n"
            "ARGS:\n    <INPUT>     input audio file\n    <OUTPUT>    output audio file\n\n"
            "OPTIONS:\n"
            "        --wav-in                 the input is a wav file (default is to detect wav files by their filename\n"
            "        --wav-out                the output is a wav file (default is to detect wav files by their filename)\n"
            "        --sample-rate <RATE>     for raw input, the sample rate of the input (defaults to 48kHz)\n"
            "        --channels <CHANNELS>    for raw input, the number of channels (defaults to 1)\n"
            "        --model <PATH>           path to a custom model file\n"
            "        --batch <LIST>           file of INPUT<TAB>OUTPUT lines, denoised together on recycled GPU streams\n"
            "        --link-channels <MODE>   max or mean: one gain curve for all channels of a file (at most 64 channels)\n"
            "        --slots <N>              with --batch: the number of recycled streams (default: up to 256, at least the widest file's channels)\n"
            "        --chunk-frames <K>       with --slots: 10 ms frames per device call (default 64, fewer beyond 32768 streams)\n"
            "        --device <N>             CUDA device (default: current)\n"
            "    -h, --help                   Print help information\n"
            "    -V, --version                Print version information\n",
            NNB_VERSION);
}

static int die(const std::string& msg) {
    fprintf(stderr, "Error: %s\n", msg.c_str());
    return 1;
}

int main(int argc, char** argv) {
    RNNoiseFileOptions opt;
    memset(&opt, 0, sizeof opt);
    opt.device = -1;
    std::string model_path, batch_list;
    int link_mode = 0, slots = 0, chunk_frames = 0;
    std::vector<std::string> pos;
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        auto value = [&](const char* name, std::string* out) -> bool {
            const std::string eq = std::string(name) + "=";
            if (a == name) {
                if (i + 1 >= argc) return false;
                *out = argv[++i];
                return true;
            }
            *out = a.substr(eq.size());
            return true;
        };
        auto is = [&](const char* name) { return a == name || a.rfind(std::string(name) + "=", 0) == 0; };
        std::string v;
        if (a == "-h" || a == "--help") {
            usage(stdout);
            return 0;
        } else if (a == "-V" || a == "--version") {
            printf("nnnoiseless-b200 %s\n", NNB_VERSION);
            return 0;
        } else if (a == "--wav-in") {
            opt.wav_in = 1;
        } else if (a == "--wav-out") {
            opt.wav_out = 1;
        } else if (is("--sample-rate")) {
            char* end = nullptr;
            if (!value("--sample-rate", &v)) return die("--sample-rate needs a value");
            opt.sample_rate = strtod(v.c_str(), &end);
            if (v.empty() || *end) return die("Invalid value for '--sample-rate <RATE>': invalid float literal");
        } else if (is("--channels")) {
            char* end = nullptr;
            if (!value("--channels", &v)) return die("--channels needs a value");
            const long c = strtol(v.c_str(), &end, 10);
            if (v.empty() || *end || c < 0 || c > 65535) return die("Invalid value for '--channels <CHANNELS>': invalid digit found in string");
            opt.channels = (int)c;
        } else if (is("--model")) {
            if (!value("--model", &model_path)) return die("--model needs a value");
        } else if (is("--batch")) {
            if (!value("--batch", &batch_list)) return die("--batch needs a value");
        } else if (is("--link-channels")) {
            if (!value("--link-channels", &v)) return die("--link-channels needs a value");
            if (v == "max") link_mode = RNNOISE_LINK_MAX;
            else if (v == "mean") link_mode = RNNOISE_LINK_MEAN;
            else return die("Invalid value for '--link-channels <MODE>': expected max or mean, found '" + v + "'");
        } else if (is("--slots") || is("--chunk-frames")) {
            const bool sl = is("--slots");
            const char* name = sl ? "--slots" : "--chunk-frames";
            if (!value(name, &v)) return die(std::string(name) + " needs a value");
            char* end = nullptr;
            const long n = strtol(v.c_str(), &end, 10);
            if (v.empty() || *end || n < 1 || n > (sl ? (1 << 20) : (1 << 16)))
                return die(std::string("Invalid value for '") + name + (sl ? " <N>'" : " <K>'") + ": expected 1.." +
                           std::to_string(sl ? (1 << 20) : (1 << 16)) + ", found '" + v + "'");
            (sl ? slots : chunk_frames) = (int)n;
        } else if (is("--device")) {
            if (!value("--device", &v)) return die("--device needs a value");
            opt.device = atoi(v.c_str());
        } else if (a.size() > 1 && a[0] == '-' && a != "-") {
            usage(stderr);
            return die("Found argument '" + a + "' which wasn't expected");
        } else {
            pos.push_back(a);
        }
    }
    if (slots && batch_list.empty()) return die("--slots is only valid with --batch");
    if (chunk_frames && !slots) return die("--chunk-frames is only valid with --slots");
    std::vector<std::string> ins, outs;
    if (!batch_list.empty()) {
        if (!pos.empty()) return die("--batch takes no positional arguments");
        std::ifstream f(batch_list);
        if (!f) return die("Failed to open batch list \"" + batch_list + "\"");
        std::string line;
        while (std::getline(f, line)) {
            if (line.empty()) continue;
            const size_t tab = line.find('\t');
            if (tab == std::string::npos) return die("batch list lines must be INPUT<TAB>OUTPUT");
            ins.push_back(line.substr(0, tab));
            outs.push_back(line.substr(tab + 1));
        }
    } else {
        if (pos.size() != 2) {
            usage(stderr);
            return die("The following required arguments were not provided: <INPUT> <OUTPUT>");
        }
        ins.push_back(pos[0]);
        outs.push_back(pos[1]);
    }
    RNNModel* model = nullptr;
    if (!model_path.empty()) {
        FILE* mf = fopen(model_path.c_str(), "rb");
        if (!mf) return die("Failed to open model file");           // src/nnnoiseless.rs:295
        model = rnnoise_model_from_file(mf);                          // closes mf
        if (!model) return die("Failed to parse model file");        // :296
        opt.model = model;
    }
    std::vector<const char*> ip, op;
    for (size_t i = 0; i < ins.size(); i++) {
        ip.push_back(ins[i].c_str());
        op.push_back(outs[i].c_str());
    }
    RNNoiseCorpusOptions copt;
    memset(&copt, 0, sizeof copt);
    copt.slots = slots;
    copt.chunk_frames = chunk_frames;
    const int rc = slots ? rnnoise_denoise_corpus((int)ip.size(), ip.data(), op.data(), &opt, link_mode, &copt, nullptr)
                         : rnnoise_denoise_files_linked((int)ip.size(), ip.data(), op.data(), &opt, link_mode);
    std::string err = rc ? rnnoise_last_error() : "";
    if (model) rnnoise_model_free(model);
    return rc ? die(err) : 0;
}
