// corpus.cu -- every file call (rnnoise_denoise_file, _files, _files_linked and _corpus; DESIGN.md §7o): a list of
// files of any size denoised on one batch of `slots` recycled streams, in chunks of `chunk_frames` frames.
//
// Decode threads take the files in list order, reserve room for the decoded source in a device pool in list order,
// upload it and hand it to the scheduler (this thread).  At every chunk boundary the scheduler gives each file that
// has ended its slots back, and admits the next files in list order on reset (and, with a link mode, linked) streams.
// A chunk is three launches and one copy back: the feed kernel reads every slot's samples (resampled to 48 kHz) into
// the [frame][sample][slot] input, the fused frame-step runs all slots, and the drain kernel scatters the int16 output
// file-major into a staging area, dropping each file's frame 0 and its frames past the end.  The host issues chunk n+1
// before it copies chunk n's staging into the files' outputs, and a writer thread writes each output once it is whole.
#include <algorithm>
#include <chrono>
#include <climits>
#include <condition_variable>
#include <cstdio>
#include <deque>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <sys/stat.h>
#include <thread>
#include <vector>

#include "../../include/rnnoise.h"
#include "abi.hpp"
#include "audio_io.hpp"
#include "common.cuh"
#include "frontend.cuh"
#include "owners.hpp"

using namespace nnb;

namespace {

// One slot's part of a chunk.  An idle slot is all zeros: zero input, nothing drained.
struct SlotRow {
    const float* src;    // the file's decoded source [n_in][C]
    const int* mk;       // position table (frontend.cuh), NULL at 48 kHz
    const double* pos;
    long K;              // samples of the file's whole frames, F * 480; later samples are zero
    long f0;             // the file's frame at the chunk's first frame
    long dst;            // staging element of this file's first drained sample in this chunk
    int C, c;            // the file's channels, this slot's channel
    int lo, hi;          // chunk frames lo <= f < hi are output frames of the file
};

// One thread per (chunk sample r, slot s), slot fastest, so the stores into in [frame][sample][slot] coalesce.
__global__ void __launch_bounds__(256) corpus_feed_kernel(const SlotRow* __restrict__ rows, int S, long n, float* __restrict__ in) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const long r = t / S;
    const SlotRow& w = rows[t - r * S];
    const long k = w.f0 * FRAME_SIZE + r;
    in[t] = w.src && k < w.K ? dasp_sample(w.src, w.C, w.c, w.mk, w.pos, k) : 0.0f;
}

// The same threads over the chunk's int16 output: chunk frame f of slot s goes to
// staging[dst + ((f - lo) * 480 + i) * C + c] when lo <= f < hi, so each file's frames of the chunk are one block of
// interleaved PCM.
__global__ void __launch_bounds__(256) corpus_drain_kernel(const SlotRow* __restrict__ rows, int S, long n, const int16_t* __restrict__ out,
                                                           int16_t* __restrict__ staging) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const long r = t / S;
    const SlotRow& w = rows[t - r * S];
    const long f = r / FRAME_SIZE;
    if (f < w.lo || f >= w.hi) return;
    staging[w.dst + ((f - w.lo) * FRAME_SIZE + (r - f * FRAME_SIZE)) * w.C + w.c] = out[t];
}

using Clock = std::chrono::steady_clock;
double seconds_since(Clock::time_point t0) { return std::chrono::duration<double>(Clock::now() - t0).count(); }

// A path's identity for the up-front checks: device and inode when it exists, else its directory's real path and name.
std::string file_key(const char* path) {
    struct stat st;
    if (stat(path, &st) == 0) return "i" + std::to_string((unsigned long long)st.st_dev) + ":" + std::to_string((unsigned long long)st.st_ino);
    std::string p = path, dir = ".", base = p;
    const size_t slash = p.find_last_of('/');
    if (slash != std::string::npos) {
        dir = slash ? p.substr(0, slash) : "/";
        base = p.substr(slash + 1);
    }
    char* real = realpath(dir.c_str(), nullptr);
    if (!real) return "p" + p;
    std::string k = "p" + std::string(real) + "/" + base;
    free(real);
    return k;
}

// A decoded source in the device pool.
struct Source {
    float* d = nullptr;
    size_t bytes = 0;
    long frames = 0;
    int channels = 1;
    double rate = 48000.0;
};

enum class Stage { pending, room, ready, failed };

struct Settings {
    int n = 0;
    const char* const* in = nullptr;
    const char* const* out = nullptr;
    RNNoiseFileOptions o{};
    double raw_rate = 48000.0;
    int raw_channels = 1;
    int link = 0, S = 0, chunk = 0, threads = 0;
    size_t budget = 0;
    std::vector<int> channels;  // per file, from the up-front checks
    bool needs_device = false;  // some file feeds two whole frames
};

// The decode-ahead.  Files are decoded in parallel, but reserve pool room in list order: a file never waits for room
// held by a later file, so the scheduler, which admits in list order, always gets the file it waits for.  A file
// larger than the budget takes its room when the pool is empty.
struct Feeder {
    const Settings* cfg = nullptr;
    int device = 0;
    std::mutex mu;
    std::condition_variable cv;
    std::vector<Stage> stage;
    std::vector<Source> src;
    std::vector<std::string> err;
    std::set<float*> live;  // pool allocations not yet freed
    int next_decode = 0, next_reserve = 0;
    size_t used = 0, peak = 0;
    bool stop = false;
    std::vector<std::thread> threads;

    void run() {
        Stream ust;
        const cudaError_t se = cudaSetDevice(device);
        const cudaError_t ce = se == cudaSuccess ? cudaStreamCreateWithFlags(ust.put(), cudaStreamNonBlocking) : se;
        for (;;) {
            int i;
            {
                std::lock_guard<std::mutex> lk(mu);
                if (stop || next_decode >= cfg->n) return;
                i = next_decode++;
            }
            const std::string in = cfg->in[i];
            AudioData a;
            std::string e;
            const bool wav_in = cfg->o.wav_in || has_wav_extension(in);
            bool ok = wav_in ? read_wav_file(in, &a, &e) : read_raw_file(in, cfg->raw_channels, cfg->raw_rate, &a, &e);
            if (ok && ce != cudaSuccess) ok = false, e = std::string("upload stream: ") + cudaGetErrorString(ce);
            const size_t bytes = std::max<size_t>(1, a.samples.size()) * sizeof(float);
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return stop || next_reserve == i; });
            if (stop) return;
            if (!ok) {  // later files keep waiting for their turn until the scheduler stops the feeder
                stage[i] = Stage::failed;
                err[i] = "\"" + in + "\": " + e;
                cv.notify_all();
                return;
            }
            stage[i] = Stage::room;
            cv.notify_all();
            cv.wait(lk, [&] { return stop || used == 0 || used + bytes <= cfg->budget; });
            if (stop) return;
            used += bytes;
            peak = std::max(peak, used);
            next_reserve++;
            stage[i] = Stage::pending;
            cv.notify_all();
            lk.unlock();
            float* d = nullptr;
            cudaError_t r = cudaMallocAsync(reinterpret_cast<void**>(&d), bytes, ust);
            if (r == cudaSuccess) r = cudaMemcpyAsync(d, a.samples.data(), a.samples.size() * sizeof(float), cudaMemcpyHostToDevice, ust);
            if (r == cudaSuccess) r = cudaStreamSynchronize(ust);
            lk.lock();
            if (d) live.insert(d);
            if (r != cudaSuccess) {
                stage[i] = Stage::failed;
                err[i] = "\"" + in + "\": uploading the source: " + cudaGetErrorString(r);
            } else {
                stage[i] = Stage::ready;
                src[i] = Source{d, bytes, a.frames(), a.channels, a.sample_rate};
            }
            cv.notify_all();
        }
    }

    // Frees a source behind the work queued on st.  Its room is given back by give_back, once that work has completed,
    // so the device never holds more than the budget (or one larger file).
    void free_source(const Source& s, cudaStream_t st) {
        cudaFreeAsync(s.d, st);
        std::lock_guard<std::mutex> lk(mu);
        live.erase(s.d);
    }
    void give_back(size_t bytes) {
        std::lock_guard<std::mutex> lk(mu);
        used -= bytes;
        cv.notify_all();
    }

    void shut(cudaStream_t st) {
        {
            std::lock_guard<std::mutex> lk(mu);
            stop = true;
            cv.notify_all();
        }
        for (std::thread& t : threads) t.join();
        threads.clear();
        for (float* d : live) cudaFreeAsync(d, st);
        live.clear();
    }
};

// Writes one output.  An output that fails after it was opened is removed, so none is left half written; a file that
// could not be opened is left as it was.  Errors name the file.
bool write_output_file(const std::string& path, bool wav, const int16_t* pcm, long frames, int C, std::string* e) {
    bool opened = false;
    const bool ok = wav ? write_wav_file(path, pcm, frames, C, e, &opened) : write_raw_file(path, pcm, frames, C, e, &opened);
    if (!ok && opened) remove(path.c_str());
    if (!ok && e->find(path) == std::string::npos) *e = "\"" + path + "\": " + *e;
    return ok;
}

// Writes each finished output on its own thread.  The outputs handed over and not yet written hold at most `cap` bytes
// of host memory (one output larger than that is taken alone): push waits for room.
struct Writer {
    struct Job {
        std::string path;
        bool wav;
        std::vector<int16_t> pcm;
        long frames;
        int C;
    };
    std::mutex mu;
    std::condition_variable cv;
    std::deque<Job> q;
    bool done = false;
    std::string err;
    long long written = 0;
    size_t queued = 0, cap = 0;  // bytes of the outputs handed over and not yet written
    std::thread th;

    void start() {
        th = std::thread([this] {
            for (;;) {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return done || !q.empty(); });
                if (q.empty()) return;
                Job j = std::move(q.front());
                q.pop_front();
                lk.unlock();
                std::string e;
                const bool ok = write_output_file(j.path, j.wav, j.pcm.data(), j.frames, j.C, &e);
                const size_t bytes = j.pcm.size() * sizeof(int16_t);
                j.pcm = std::vector<int16_t>();
                lk.lock();
                queued -= bytes;
                cv.notify_all();
                if (ok) written++;
                else if (err.empty()) err = e;
            }
        });
    }
    // Returns the seconds it waited for room.
    double push(Job j) {
        const size_t bytes = j.pcm.size() * sizeof(int16_t);
        std::unique_lock<std::mutex> lk(mu);
        const auto t0 = Clock::now();
        cv.wait(lk, [&] { return queued == 0 || queued + bytes <= cap; });
        const double waited = seconds_since(t0);
        queued += bytes;
        q.push_back(std::move(j));
        cv.notify_all();
        return waited;
    }
    std::string error() {
        std::lock_guard<std::mutex> lk(mu);
        return err;
    }
    void finish() {
        if (!th.joinable()) return;
        {
            std::lock_guard<std::mutex> lk(mu);
            done = true;
            cv.notify_all();
        }
        th.join();
    }
};

// A file in slots.
struct Active {
    int idx;
    Source s;
    const double* ratio;  // key of its position table, NULL at 48 kHz
    long F, f = 0;        // whole frames; frames issued so far
    std::vector<int> slots;  // ascending: channel c runs on slots[c]
    std::vector<int16_t> out;  // [(F - 1) * 480][C]
};

// A chunk's staging blocks, copied into the files' outputs once the chunk is back.
struct Drained {
    Active* file;
    long at, n;  // out[at, at + n) = staging[dst, dst + n)
    long dst;
};

// Whether a source of n frames at `rate` feeds two whole 48 kHz frames.  A shorter file's output is empty, because the
// first frame's output is discarded (src/nnnoiseless.rs:319-327).  The same recurrence as samples_of, for 960 outputs.
bool feeds_two_frames(double rate, long n) {
    if (rate == 48000.0) return n >= 2 * FRAME_SIZE;
    PosTable t;
    build_pos_table(rate / 48000.0, n, &t, 2 * FRAME_SIZE);
    return t.m.size() >= 2 * FRAME_SIZE;
}

// who: the entry point named in argument errors.  one_file: the one-file call, which opens the input and creates the
// output before anything else is checked, as the reference binary does (src/nnnoiseless.rs:251-258).
int check_options(const char* who, bool one_file, int n_files, const char* const* in_paths, const char* const* out_paths,
                  const RNNoiseFileOptions* opt, int link_mode, const RNNoiseCorpusOptions* copt, Settings* cfg) {
    if (n_files < 0 || (n_files > 0 && (!in_paths || !out_paths))) return fail(std::string(who) + ": bad argument");
    if (link_mode != 0 && link_mode != RNNOISE_LINK_MAX && link_mode != RNNOISE_LINK_MEAN)
        return fail("link mode " + std::to_string(link_mode) + " is neither 0, RNNOISE_LINK_MAX (1) nor RNNOISE_LINK_MEAN (2)");
    RNNoiseCorpusOptions c{};
    if (copt) c = *copt;
    if (c.slots < 0 || c.slots > (1 << 20)) return fail("slots must be 1..1048576 (0: default), not " + std::to_string(c.slots));
    if (c.chunk_frames < 0 || c.chunk_frames > (1 << 16)) return fail("chunk_frames must be 1..65536 (0: default), not " + std::to_string(c.chunk_frames));
    if (c.device_pool_bytes < 0) return fail("device_pool_bytes must be >= 0 (0: 1 GiB), not " + std::to_string(c.device_pool_bytes));
    if (c.decode_threads < 0 || c.decode_threads > 256) return fail("decode_threads must be 1..256 (0: default), not " + std::to_string(c.decode_threads));
    cfg->budget = c.device_pool_bytes ? (size_t)c.device_pool_bytes : (size_t(1) << 30);
    cfg->threads = c.decode_threads ? c.decode_threads : (int)std::max(1u, std::min(8u, std::thread::hardware_concurrency()));
    cfg->n = n_files;
    cfg->in = in_paths;
    cfg->out = out_paths;
    cfg->o.device = -1;
    if (opt) cfg->o = *opt;
    cfg->raw_rate = cfg->o.sample_rate > 0.0 ? cfg->o.sample_rate : 48000.0;  // src/nnnoiseless.rs:270-271
    cfg->raw_channels = cfg->o.channels > 0 ? cfg->o.channels : 1;
    cfg->link = link_mode;
    for (int i = 0; i < n_files; i++)
        if (!in_paths[i] || !out_paths[i]) return fail(std::string(who) + ": null path at index " + std::to_string(i));
    if (one_file && n_files == 1) {
        FILE* f = fopen(in_paths[0], "rb");
        if (!f) return fail(std::string("Failed to open input file \"") + in_paths[0] + "\"");
        fclose(f);
        f = fopen(out_paths[0], "wb");
        if (!f) return fail(std::string("Failed to open output file \"") + out_paths[0] + "\"");
        fclose(f);
    }
    std::set<std::string> ins, outs;
    for (int i = 0; i < n_files; i++) ins.insert(file_key(in_paths[i]));
    for (int i = 0; i < n_files; i++) {
        const std::string k = file_key(out_paths[i]);
        if (ins.count(k)) return fail(std::string("output file \"") + out_paths[i] + "\" is also an input of this call");
        if (!outs.insert(k).second) return fail(std::string("output file \"") + out_paths[i] + "\" is listed twice");
    }
    const int max_channels = c.slots ? c.slots : (1 << 20);
    long long total = 0;
    int widest = 1;
    for (int i = 0; i < n_files; i++) {
        const std::string in = in_paths[i];
        FILE* probe = fopen(in.c_str(), "rb");
        if (!probe) return fail("Failed to open input file \"" + in + "\"");
        fclose(probe);
        int C = cfg->raw_channels;
        double rate = cfg->raw_rate;
        long frames = 0;
        if (cfg->o.wav_in || has_wav_extension(in)) {
            WavHeader h;
            std::string err;
            if (!probe_wav_file(in, &h, &err)) return fail(err);
            C = h.channels;
            rate = (double)h.sample_rate;
            frames = (long)h.n_frames;
        } else {
            struct stat st;
            if (stat(in.c_str(), &st) == 0) frames = (long)(st.st_size / 2 / C);  // the decoder refuses a partial frame
        }
        cfg->channels.push_back(C);
        if (C > max_channels)
            return fail("\"" + in + "\" has " + std::to_string(C) + " channels: more than " +
                        (c.slots ? "the " + std::to_string(c.slots) + " slots" : std::to_string(max_channels)));
        if (link_mode && C > RNNOISE_LINK_MAX_MEMBERS)
            return fail("\"" + in + "\" has " + std::to_string(C) + " channels: linked channels are at most " +
                        std::to_string(RNNOISE_LINK_MAX_MEMBERS) + " per file");
        total += C;
        widest = std::max(widest, C);
        cfg->needs_device = cfg->needs_device || feeds_two_frames(rate, frames);
    }
    // defaults (DESIGN.md 7o, measured): 256 slots, or fewer when the list has fewer channels, but never fewer than the
    // widest file's; 64-frame chunks, or fewer when the slots would make the chunk larger than 2^21 slot-frames
    cfg->S = c.slots ? c.slots : std::max(widest, (int)std::min<long long>(256, total));
    cfg->chunk = c.chunk_frames ? c.chunk_frames : std::min(64, (1 << 21) / cfg->S);
    if ((long long)cfg->S * cfg->chunk > (1LL << 21))
        return fail("slots * chunk_frames must be at most 2097152, not " + std::to_string((long long)cfg->S * cfg->chunk));
    return 0;
}

// Every file of a call whose files are all shorter than two frames: decoded in list order, its empty output written.
// No CUDA call.
int write_short_outputs(const Settings& cfg, RNNoiseCorpusStats* st) {
    for (int i = 0; i < cfg.n; i++) {
        const std::string in = cfg.in[i];
        AudioData a;
        std::string e;
        const bool ok = cfg.o.wav_in || has_wav_extension(in) ? read_wav_file(in, &a, &e) : read_raw_file(in, cfg.raw_channels, cfg.raw_rate, &a, &e);
        if (!ok) return fail("\"" + in + "\": " + e);
        if (!write_output_file(cfg.out[i], cfg.o.wav_out || has_wav_extension(cfg.out[i]), nullptr, 0, a.channels, &e)) return fail(e);
        st->files++;
    }
    return 0;
}

// The scheduler.  Members are destroyed in reverse order: the feeder and writer are stopped by run()'s caller first.
struct Corpus {
    const Settings& cfg;
    int device;
    RNNoiseCorpusStats st{};
    Feeder feed;
    Writer writer;
    DeviceWork dw;
    std::map<double, PosTable> tables;
    std::vector<DeviceMem> table_mem;  // position tables, replaced when a longer file arrives
    std::vector<std::unique_ptr<Active>> active;
    std::vector<int> free_slots;
    SlotRow* h_rows[2] = {nullptr, nullptr};
    int16_t* h_stage[2] = {nullptr, nullptr};
    PinnedMem pin_rows, pin_stage;
    Event ev[2];
    std::vector<Drained> drained[2];
    std::vector<std::unique_ptr<Active>> finished[2];  // files whose last frames are in that chunk
    SlotRow* d_rows = nullptr;
    float* d_in = nullptr;
    int16_t* d_out = nullptr;
    int16_t* d_stage = nullptr;
    int next = 0;
    std::string failed;  // a decoder refusal: no file after it is admitted

    Corpus(const Settings& c, int dev) : cfg(c), device(dev) {}

    int setup() {
        const size_t S = (size_t)cfg.S, per_chunk = (size_t)cfg.chunk * FRAME_SIZE * S;
        CK(cudaStreamCreateWithFlags(dw.st.put(), cudaStreamNonBlocking));
        CK(dalloc(&dw.dev, &d_rows, S));
        CK(dalloc(&dw.dev, &d_in, per_chunk));
        CK(dalloc(&dw.dev, &d_out, per_chunk));
        CK(dalloc(&dw.dev, &d_stage, per_chunk));
        CK(cudaMallocHost(pin_rows.put(), 2 * S * sizeof(SlotRow)));
        CK(cudaMallocHost(pin_stage.put(), 2 * per_chunk * sizeof(int16_t)));
        for (int b = 0; b < 2; b++) {
            h_rows[b] = static_cast<SlotRow*>(static_cast<void*>(pin_rows)) + b * S;
            h_stage[b] = static_cast<int16_t*>(static_cast<void*>(pin_stage)) + b * per_chunk;
            CK(cudaEventCreateWithFlags(ev[b].put(), cudaEventDisableTiming));
        }
        dw.batch.reset(rnnoise_batch_create(cfg.o.model, cfg.S, device));
        if (!dw.batch) return -1;
        for (int s = cfg.S - 1; s >= 0; s--) free_slots.push_back(s);  // back() is the lowest free slot
        feed.cfg = &cfg;
        feed.device = device;
        feed.stage.assign((size_t)cfg.n, Stage::pending);
        feed.src.assign((size_t)cfg.n, Source{});
        feed.err.assign((size_t)cfg.n, std::string());
        for (int t = 0; t < cfg.threads; t++) feed.threads.emplace_back([this] { feed.run(); });
        writer.cap = cfg.budget;
        writer.start();
        return 0;
    }

    void write_output(int i, std::vector<int16_t> pcm, long frames, int C) {
        st.write_wait_seconds += writer.push(Writer::Job{cfg.out[i], cfg.o.wav_out || has_wav_extension(cfg.out[i]), std::move(pcm), frames, C});
    }

    // The number of 48 kHz samples the file feeds, as the resampler makes them; extends the rate's table.
    int samples_of(const Source& s, const double** key, long* K) {
        *key = nullptr;
        if (s.rate == 48000.0) {
            *K = s.frames;
            return 0;
        }
        const double ratio = s.rate / 48000.0;
        auto it = tables.find(ratio);
        if (it == tables.end()) it = tables.emplace(ratio, PosTable{}).first;
        PosTable& t = it->second;
        if (t.m.empty() || t.n_in_max < s.frames) {  // a longer file: rebuild to twice the length, so rebuilds stay rare
            build_pos_table(ratio, std::max(s.frames, 2 * t.n_in_max), &t);
            const size_t n = std::max<size_t>(1, t.m.size());
            table_mem.emplace_back();
            CK(table_mem.back().alloc(n * sizeof(int)));
            t.d_m = table_mem.back().get<int>();
            table_mem.emplace_back();
            CK(table_mem.back().alloc(n * sizeof(double)));
            t.d_pos = table_mem.back().get<double>();
            CK(cudaMemcpyAsync(t.d_m, t.m.data(), t.m.size() * sizeof(int), cudaMemcpyHostToDevice, dw.st));
            CK(cudaMemcpyAsync(t.d_pos, t.pos.data(), t.pos.size() * sizeof(double), cudaMemcpyHostToDevice, dw.st));
        }
        *key = &it->first;
        *K = (long)(std::upper_bound(t.m.begin(), t.m.end(), (int)std::min<long>(s.frames, INT_MAX)) - t.m.begin());
        return 0;
    }

    // Admits files in list order while their channels fit in the free slots.  in_flight: a chunk is issued and not yet
    // drained; the room of the files that ended in it comes back when it is.
    int admit(bool in_flight) {
        std::vector<int> fresh;
        while (next < cfg.n && failed.empty()) {
            // a file that cannot get slots before running files end is not waited for: run them
            if (!active.empty() && (int)free_slots.size() < cfg.channels[(size_t)next]) break;
            Source s;
            {
                std::unique_lock<std::mutex> lk(feed.mu);
                const auto t0 = Clock::now();
                // a file waiting for room gets it only when running or drained files give theirs back, so run or
                // drain them rather than wait
                feed.cv.wait(lk, [&] {
                    const Stage g = feed.stage[(size_t)next];
                    return g == Stage::ready || g == Stage::failed || (g == Stage::room && (!active.empty() || in_flight));
                });
                st.decode_wait_seconds += seconds_since(t0);
                const Stage g = feed.stage[(size_t)next];
                if (g == Stage::failed) {
                    failed = feed.err[(size_t)next];
                    break;
                }
                if (g == Stage::room) break;
                s = feed.src[(size_t)next];
            }
            const double* key;
            long K;
            if (samples_of(s, &key, &K)) return -1;
            const long F = K / FRAME_SIZE;
            if (F < 2) {  // shorter than two frames: an empty output, no slot (src/nnnoiseless.rs:319-327)
                feed.free_source(s, dw.st);
                feed.give_back(s.bytes);
                feed.src[(size_t)next] = Source{};
                write_output(next, {}, 0, s.channels);
                next++;
                continue;
            }
            if ((int)free_slots.size() < s.channels) break;
            auto a = std::make_unique<Active>();
            a->idx = next;
            a->s = s;
            a->ratio = key;
            a->F = F;
            for (int c = 0; c < s.channels; c++) {
                a->slots.push_back(free_slots.back());
                free_slots.pop_back();
            }
            std::sort(a->slots.begin(), a->slots.end());  // linked means are taken in ascending stream order
            a->out.resize((size_t)(F - 1) * FRAME_SIZE * (size_t)s.channels);
            fresh.insert(fresh.end(), a->slots.begin(), a->slots.end());
            if (cfg.link && s.channels > 1 && rnnoise_batch_link_streams(dw.batch.get(), a->slots.data(), s.channels, cfg.link) != 0) return -1;
            st.useful_stream_frames += (long long)s.channels * F;
            active.push_back(std::move(a));
            next++;
        }
        if (!fresh.empty() && rnnoise_batch_reset_streams(dw.batch.get(), fresh.data(), (int)fresh.size(), dw.st) != 0) return -1;
        std::sort(free_slots.rbegin(), free_slots.rend());
        return 0;
    }

    // Issues one chunk into buffer b; files that end in it move to finished[b].
    int issue(int b) {
        long nf = 0;
        for (const auto& a : active) nf = std::max(nf, a->F - a->f);
        nf = std::min<long>(nf, cfg.chunk);
        SlotRow* rows = h_rows[b];
        std::fill(rows, rows + cfg.S, SlotRow{});
        drained[b].clear();
        long dst = 0;
        for (const auto& a : active) {
            const int C = a->s.channels;
            const long lo = std::max<long>(a->f, 1) - a->f, hi = std::max(lo, std::min(a->f + nf, a->F) - a->f);
            const PosTable* t = a->ratio ? &tables.at(*a->ratio) : nullptr;
            for (int c = 0; c < C; c++)
                rows[a->slots[(size_t)c]] = SlotRow{a->s.d, t ? t->d_m : nullptr, t ? t->d_pos : nullptr, a->F * FRAME_SIZE, a->f, dst, C, c, (int)lo, (int)hi};
            const long n = (hi - lo) * FRAME_SIZE * C;
            if (n) drained[b].push_back(Drained{a.get(), (a->f + lo - 1) * FRAME_SIZE * C, n, dst});
            dst += n;
        }
        const long n = nf * FRAME_SIZE * cfg.S;
        const unsigned grid = (unsigned)((n + 255) / 256);
        CK(cudaMemcpyAsync(d_rows, rows, (size_t)cfg.S * sizeof(SlotRow), cudaMemcpyHostToDevice, dw.st));
        corpus_feed_kernel<<<grid, 256, 0, dw.st>>>(d_rows, cfg.S, n, d_in);
        CK(cudaGetLastError());
        if (rnnoise_batch_process_device_strided(dw.batch.get(), d_out, d_in, 2, nullptr, (int)nf, 1, cfg.S, (long)FRAME_SIZE * cfg.S, dw.st) != 0)
            return -1;
        corpus_drain_kernel<<<grid, 256, 0, dw.st>>>(d_rows, cfg.S, n, d_out, d_stage);
        CK(cudaGetLastError());
        count_launches(2);
        CK(cudaMemcpyAsync(h_stage[b], d_stage, (size_t)dst * sizeof(int16_t), cudaMemcpyDeviceToHost, dw.st));
        // the sources of files that end in this chunk are freed before its event, so its completion returns their room
        for (const auto& a : active)
            if (a->f + nf >= a->F) feed.free_source(a->s, dw.st);
        CK(cudaEventRecord(ev[b], dw.st));
        st.chunks++;
        st.issued_slot_frames += nf * cfg.S;
        // files that end in this chunk leave their slots at this boundary, and give their room back when it is drained
        std::vector<std::unique_ptr<Active>> still;
        for (auto& a : active) {
            a->f += nf;
            if (a->f < a->F) {
                still.push_back(std::move(a));
                continue;
            }
            if (cfg.link && a->s.channels > 1 && rnnoise_batch_unlink_streams(dw.batch.get(), a->slots.data(), a->s.channels) != 0) return -1;
            free_slots.insert(free_slots.end(), a->slots.begin(), a->slots.end());
            finished[b].push_back(std::move(a));
        }
        active = std::move(still);
        std::sort(free_slots.rbegin(), free_slots.rend());
        return 0;
    }

    // Copies chunk b's staging into the outputs, gives the room of the files that ended in it back and hands them to the
    // writer.
    int drain(int b) {
        const auto t0 = Clock::now();
        CK(cudaEventSynchronize(ev[b]));
        st.device_wait_seconds += seconds_since(t0);
        for (const Drained& d : drained[b]) std::copy(h_stage[b] + d.dst, h_stage[b] + d.dst + d.n, d.file->out.data() + d.at);
        drained[b].clear();
        for (auto& a : finished[b]) {
            feed.give_back(a->s.bytes);
            write_output(a->idx, std::move(a->out), (a->F - 1) * FRAME_SIZE, a->s.channels);
        }
        finished[b].clear();
        const std::string e = writer.error();
        return e.empty() ? 0 : fail(e);
    }

    int run() {
        if (setup()) return -1;
        int b = 0, pending = -1;
        for (;;) {
            if (admit(pending >= 0)) return -1;
            if (active.empty()) {  // nothing to run: drain the chunk in flight, whose files give room back, and admit again
                if (pending < 0) break;
                if (drain(pending)) return -1;
                pending = -1;
                continue;
            }
            if (issue(b)) return -1;
            if (pending >= 0 && drain(pending)) return -1;
            pending = b;
            b ^= 1;
        }
        if (!failed.empty()) return fail(failed);
        return 0;
    }

    // Stops the threads (the writer first writes every output already handed to it) and frees the pool.
    int finish(int rc, RNNoiseCorpusStats* stats) {
        feed.shut(dw.st);
        const auto tw = Clock::now();
        writer.finish();
        st.write_wait_seconds += seconds_since(tw);
        if (dw.st) {
            const auto t0 = Clock::now();
            const cudaError_t e = cudaStreamSynchronize(dw.st);
            st.device_wait_seconds += seconds_since(t0);
            if (e != cudaSuccess && rc == 0) rc = fail("cudaStreamSynchronize", e);
        }
        if (rc == 0 && !writer.err.empty()) rc = fail(writer.err);
        st.files = writer.written;
        st.peak_pool_bytes = (long long)feed.peak;
        if (stats) *stats = st;
        return rc;
    }
};

// The one engine behind every file call.
int denoise_list(const char* who, bool one_file, int n_files, const char* const* in_paths, const char* const* out_paths,
                 const RNNoiseFileOptions* opt, int link_mode, const RNNoiseCorpusOptions* copt, RNNoiseCorpusStats* stats) {
    Settings cfg;
    if (check_options(who, one_file, n_files, in_paths, out_paths, opt, link_mode, copt, &cfg)) return -1;
    RNNoiseCorpusStats short_st{};
    if (stats) *stats = short_st;
    if (n_files == 0) return 0;
    if (!cfg.needs_device) {  // format errors are reported, and empty outputs written, on a machine without a GPU
        const int rc = write_short_outputs(cfg, &short_st);
        if (stats) *stats = short_st;
        return rc;
    }
    int device;
    if (open_device(cfg.o.device, &device)) return -1;
    ON_DEVICE(device);
    Corpus corpus(cfg, device);
    const int rc = corpus.run();
    return corpus.finish(rc, stats);
}

}  // namespace

extern "C" {

int rnnoise_denoise_corpus(int n_files, const char* const* in_paths, const char* const* out_paths, const RNNoiseFileOptions* opt,
                           int link_mode, const RNNoiseCorpusOptions* copt, RNNoiseCorpusStats* stats) {
    return denoise_list("rnnoise_denoise_corpus", false, n_files, in_paths, out_paths, opt, link_mode, copt, stats);
}

int rnnoise_denoise_files_linked(int n_files, const char* const* in_paths, const char* const* out_paths, const RNNoiseFileOptions* opt,
                                 int link_mode) {
    return denoise_list("rnnoise_denoise_files", true, n_files, in_paths, out_paths, opt, link_mode, nullptr, nullptr);
}

int rnnoise_denoise_files(int n_files, const char* const* in_paths, const char* const* out_paths, const RNNoiseFileOptions* opt) {
    return rnnoise_denoise_files_linked(n_files, in_paths, out_paths, opt, 0);
}

int rnnoise_denoise_file(const char* in_path, const char* out_path, const RNNoiseFileOptions* opt) {
    if (!in_path || !out_path) return fail("rnnoise_denoise_file: null path");
    return rnnoise_denoise_files(1, &in_path, &out_path, opt);
}

}  // extern "C"
