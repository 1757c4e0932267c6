"""rnnoise_denoise_corpus / files.denoise_corpus / --slots: a file corpus on a fixed set of recycled stream slots, the
engine behind every file call.

GPU: a seeded corpus of about 60 files (WAV of every sample format at 8, 16, 22.05, 44.1 and 48 kHz, 1-3 channels, raw
inputs, lengths from 0 samples to about 400 frames) gives, at every slot count, chunk length, list order and link mode,
outputs byte-identical to a reference built without the engine (decoder, resampler and one DenoiseBatch per file); so
does the one-file call; the stats hold; a small device pool still finishes; a late decoder refusal fails the call
naming the file, after every file before it is written and with no other output; the default slots are the list's
channels, and a file wider than 256 channels runs under defaults.
CPU: every up-front refusal leaves no output, the command line's and Python's argument checks, the C++ mirror."""
import ctypes as C
import os
import random
import re
import subprocess

import numpy as np
import pytest

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import files
from test_cli_files import _signal, _wav_bytes

F = 480
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RAW = dict(sample_rate=16000, channels=2)   # the raw inputs' options, passed to every call
FORMATS = [dict(bits=16), dict(bits=8), dict(bits=24), dict(bits=32), dict(fmt=3, bits=32)]
RATES = [8000, 16000, 22050, 44100, 48000]


def make_corpus(d, n_random=48, seed=7):
    """-> [(path, channels, rate, native frames)]: the edge lengths, then n_random files of random format and length."""
    rng = random.Random(seed)
    specs = [(0, 1, 48000), (1, 1, 48000), (479, 2, 48000), (480, 1, 48000), (960, 3, 48000), (960, 1, 16000),
             (2 * F + 1, 2, 44100), (3 * F, 1, 22050)]
    for _ in range(n_random):
        rate = rng.choice(RATES)
        specs.append((rng.randint(0, 400 * F) * rate // 48000, rng.choice([1, 1, 2, 3]), rate))
    out = []
    for i, (n, ch, rate) in enumerate(specs):
        x = _signal(max(n, 1), ch, seed=100 + i)[:n]
        if i % 9 == 4:                                     # raw inputs, all at the RAW options
            p = d / ("in%02d.raw" % i)
            x = _signal(max(n, 1), RAW["channels"], seed=100 + i)[:n]
            p.write_bytes(np.round(x).astype("<i2").tobytes())
            out.append((str(p), RAW["channels"], RAW["sample_rate"], n))
            continue
        p = d / ("in%02d.wav" % i)
        p.write_bytes(_wav_bytes(x, rate, **FORMATS[i % len(FORMATS)]))
        out.append((str(p), ch, rate, n))
    return out


def reference_output(path, out_path, mode=None):
    """What the file calls must write for one input, built without them: decode, resample to 48 kHz, a DenoiseBatch of
    the file's channels (linked as one group under a link mode) over its whole frames with float input and int16
    output, frame 0 dropped, written in the output's format.  Fewer than two whole frames give an empty output."""
    x, rate = files.read_audio(path, **RAW)
    if rate != 48000.0 and len(x):
        x = files.resample(x, rate / 48000.0)
    n_ch = x.shape[1]
    T = len(x) // F
    pcm = np.zeros((0, n_ch), np.int16)
    if T >= 2:
        import torch
        xd = torch.from_numpy(np.ascontiguousarray(x[:T * F])).cuda()      # [frame][sample][channel]
        out = torch.empty((T * F, n_ch), dtype=torch.int16, device="cuda")
        b = nb.DenoiseBatch(n_ch)
        if mode is not None and n_ch > 1:
            b.link_streams(list(range(n_ch)), mode)
        assert nb.lib().rnnoise_batch_process_device_strided(b._h, out.data_ptr(), xd.data_ptr(), 2, None, T, 1, n_ch, F * n_ch,
                                                             None) == 0, nb.last_error()
        pcm = out.cpu().numpy()[F:]
    files.write_audio(str(out_path), pcm)
    return open(out_path, "rb").read()


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """The corpus and each file's reference output, unlinked and under both link modes."""
    d = tmp_path_factory.mktemp("corpus")
    items = make_corpus(d)
    want = {}
    for mode in (None, "max", "mean"):
        for i, (p, ch, _, _) in enumerate(items):
            if mode is not None and ch == 1:
                want[(mode, i)] = want[(None, i)]
                continue
            want[(mode, i)] = reference_output(p, d / ("want_%s_%02d%s" % (mode, i, ".wav" if i % 2 else ".raw")), mode)
    return d, items, want


@pytest.mark.gpu
def test_one_file_calls_match_reference(corpus):
    d, items, want = corpus
    for mode in (None, "max", "mean"):
        for i, (p, ch, _, _) in enumerate(items):
            if mode is not None and ch == 1:
                continue
            o = d / ("one_%s_%02d%s" % (mode, i, ".wav" if i % 2 else ".raw"))
            if mode is None:
                files.denoise_file(p, str(o), **RAW)
            else:
                files.denoise_files([(p, str(o))], link_channels=mode, **RAW)
            assert o.read_bytes() == want[(mode, i)], (mode, i, items[i])


def run(d, items, order, tag, mode=None, **kw):
    """Denoises items[order] into fresh outputs (odd indices as WAV, as the wants) and returns (stats, {i: bytes})."""
    out = d / tag
    out.mkdir()
    pairs = [(items[i][0], str(out / ("o%02d%s" % (i, ".wav" if i % 2 else ".raw")))) for i in order]
    st = files.denoise_corpus(pairs, link_channels=mode, **RAW, **kw)
    return st, {i: open(p, "rb").read() for i, (_, p) in zip(order, pairs)}


def check_stats(st, items, order, want, mode=None, budget=None):
    useful, largest = 0, 0
    for i in order:
        w, ch = want[(mode, i)], items[i][1]
        n_out = int.from_bytes(w[w.index(b"data") + 4:][:4], "little") if w[:4] == b"RIFF" else len(w)
        frames = n_out // (2 * ch)
        if frames:
            useful += ch * (frames // F + 1)               # the discarded first frame ran too
        largest = max(largest, 4 * ch * max(items[i][3], 1))
    assert st["files"] == len(order)
    assert st["useful_stream_frames"] == useful
    assert st["issued_slot_frames"] >= useful and st["chunks"] > 0
    assert 0 < st["peak_pool_bytes"] <= (budget if budget else 1 << 30) + largest
    assert st["decode_wait_seconds"] >= 0 and st["device_wait_seconds"] >= 0 and st["write_wait_seconds"] >= 0


@pytest.mark.gpu
@pytest.mark.parametrize("slots,chunk", [(1, 64), (3, 1), (8, 5), (8, 64), (200, 64)])
def test_corpus_matches_one_file_calls(corpus, slots, chunk):
    d, items, want = corpus
    order = list(range(len(items)))
    if slots == 1:
        order = [i for i in order if items[i][1] == 1]
    if slots == 200:
        assert slots >= sum(it[1] for it in items)                   # every file has its own slots from the start
    st, got = run(d, items, order, "s%d_c%d" % (slots, chunk), slots=slots, chunk_frames=chunk, decode_threads=3)
    for i in order:
        assert got[i] == want[(None, i)], (i, items[i])
    check_stats(st, items, order, want)


@pytest.mark.gpu
def test_corpus_shuffled_order_and_small_pool(corpus):
    d, items, want = corpus
    order = list(range(len(items)))
    random.Random(3).shuffle(order)
    st, got = run(d, items, order, "shuffled", slots=8, chunk_frames=64)
    assert all(got[i] == want[(None, i)] for i in order)
    check_stats(st, items, order, want)
    # a budget of about three average files: decode waits for room, the call still finishes with the same bytes
    budget = 3 * 4 * 200 * F
    st, got = run(d, items, order, "pool", slots=8, chunk_frames=16, device_pool_bytes=budget, decode_threads=4)
    assert all(got[i] == want[(None, i)] for i in order)
    check_stats(st, items, order, want, budget=budget)
    # a budget of one byte: every source runs alone in the pool, and every output waits for the writer alone
    st, got = run(d, items, order, "one_byte", slots=8, chunk_frames=32, device_pool_bytes=1)
    assert all(got[i] == want[(None, i)] for i in order)
    check_stats(st, items, order, want, budget=1)


@pytest.mark.gpu
def test_corpus_write_failure_leaves_unopened_target(corpus, tmp_path):
    """An output the writer cannot open (here an existing directory) fails the call naming it and is left as it was."""
    d, items, want = corpus
    target = tmp_path / "taken.wav"
    target.mkdir()
    order = [8, 9, 10]
    pairs = [(items[i][0], str(tmp_path / ("o%02d%s" % (i, ".wav" if i % 2 else ".raw")))) for i in order]
    pairs[1] = (pairs[1][0], str(target))
    with pytest.raises(files.NnnoiselessError, match='Failed to open output file ".*taken.wav"'):
        files.denoise_corpus(pairs, slots=3, chunk_frames=8, **RAW)
    assert target.is_dir() and not any(target.iterdir())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["max", "mean"])
def test_corpus_linked_matches_one_file_calls(corpus, mode):
    d, items, want = corpus
    order = list(range(len(items)))
    st, got = run(d, items, order, "link_" + mode, mode=mode, slots=5, chunk_frames=5)
    for i in order:
        assert got[i] == want[(mode, i)], (mode, i, items[i])
    check_stats(st, items, order, want, mode=mode)


@pytest.mark.gpu
def test_corpus_cli_slots(corpus):
    d, items, want = corpus
    out = d / "cli"
    out.mkdir()
    lst = d / "cli.list"
    order = list(range(0, len(items), 3))
    lst.write_text("".join("%s\t%s\n" % (items[i][0], out / ("o%02d%s" % (i, ".wav" if i % 2 else ".raw"))) for i in order))
    r = subprocess.run([files.CLI_PATH, "--batch", str(lst), "--slots", "4", "--chunk-frames=7", "--sample-rate", "16000",
                        "--channels", "2"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for i in order:
        assert (out / ("o%02d%s" % (i, ".wav" if i % 2 else ".raw"))).read_bytes() == want[(None, i)]


@pytest.mark.gpu
def test_default_slots_follow_the_list(tmp_path):
    """Under defaults a short list runs on exactly its own channels, and a file wider than 256 channels is taken."""
    lengths = [2 * F + 5, 7 * F, 4 * F + 300]
    pairs = []
    for k, n in enumerate(lengths):
        p = tmp_path / ("m%d.wav" % k)
        files.write_audio(str(p), np.round(_signal(n, 1, seed=60 + k)).astype(np.int16), wav=True)
        pairs.append((str(p), str(tmp_path / ("o%d.raw" % k))))
    st = files.denoise_corpus(pairs)
    assert st["issued_slot_frames"] == 3 * (max(lengths) // F)
    for src, dst in pairs:
        assert open(dst, "rb").read() == reference_output(src, tmp_path / "want.raw")
    wide = tmp_path / "wide.wav"
    files.write_audio(str(wide), np.round(_signal(3 * F + 7, 300, seed=70)).astype(np.int16), wav=True)
    files.denoise_files([(str(wide), str(tmp_path / "wide_out.wav"))])
    assert (tmp_path / "wide_out.wav").read_bytes() == reference_output(str(wide), tmp_path / "wide_want.wav")


def odd_raw(path):
    path.write_bytes(bytes(2 * 3 * F + 1))                 # an odd number of bytes: refused by the raw decoder


def test_late_refusal_passes_the_checks(tmp_path):
    """The late failure below needs an input the up-front checks accept and the decoder refuses.  A WAV whose data
    chunk ends early does not do: the header probe already refuses it.  A raw file of an odd number of bytes does."""
    x = _signal(3 * F, 1, seed=5)
    short = tmp_path / "short.wav"
    short.write_bytes(_wav_bytes(x, 16000)[:-10])
    with pytest.raises(files.NnnoiselessError, match="Failed to read enough bytes"):
        files.probe_audio(str(short))
    with pytest.raises(files.NnnoiselessError, match="Failed to read enough bytes"):
        files.denoise_corpus([(str(short), str(tmp_path / "o.wav"))])
    assert not (tmp_path / "o.wav").exists()
    odd = tmp_path / "odd.raw"
    odd_raw(odd)
    with pytest.raises(files.NnnoiselessError, match="even number of bytes"):
        files.read_audio(str(odd))


@pytest.mark.gpu
def test_corpus_late_decoder_refusal(corpus, tmp_path):
    d, items, want = corpus
    bad = tmp_path / "bad.raw"
    odd_raw(bad)
    order = list(range(12))
    ins = [items[i][0] for i in order]
    ins.insert(10, str(bad))
    outs = [str(tmp_path / ("o%02d%s" % (k, ".wav" if k % 2 else ".raw"))) for k in range(len(ins))]
    with pytest.raises(files.NnnoiselessError) as e:
        files.denoise_corpus(list(zip(ins, outs)), slots=3, chunk_frames=4, **RAW)
    assert str(bad) in str(e.value) and "even number of bytes" in str(e.value)
    for i in order[:10]:                                   # every file before the refused one is written whole
        assert open(outs[i], "rb").read() == want[(None, i)], i
    assert not any(os.path.exists(p) for p in outs[10:])


# ---- CPU: refusals before any output or CUDA call -------------------------------------------------------------------
def _refused(pairs, match, **kw):
    with pytest.raises((files.NnnoiselessError, ValueError), match=match):
        files.denoise_corpus(pairs, **kw)
    for _, o in pairs:
        assert not os.path.exists(o) or o in [a for a, _ in pairs]


def test_corpus_refusals_leave_no_output(tmp_path):
    a, b = tmp_path / "a.wav", tmp_path / "b.raw"
    a.write_bytes(_wav_bytes(_signal(3 * F, 3, seed=1), 44100))
    b.write_bytes(bytes(4 * F))
    oa, ob = str(tmp_path / "oa.wav"), str(tmp_path / "ob.raw")
    _refused([(str(a), oa), (str(b), str(a))], "is also an input")
    _refused([(str(a), oa), (str(b), os.path.join(str(tmp_path), ".", "oa.wav"))], "listed twice")
    with pytest.raises(files.NnnoiselessError, match="listed twice"):
        files.denoise_files([(str(a), oa), (str(b), oa)])
    assert not os.path.exists(oa)
    _refused([(str(a), oa), (str(tmp_path / "missing.wav"), ob)], 'Failed to open input file ".*missing.wav"')
    (tmp_path / "junk.wav").write_bytes(bytes(100))
    _refused([(str(a), oa), (str(tmp_path / "junk.wav"), ob)], "no RIFF tag found")
    _refused([(str(a), oa), (str(b), ob)], "has 3 channels: more than the 2 slots", slots=2)
    _refused([(str(b), ob)], "has 4 channels: more than the 3 slots", slots=3, channels=4)
    wide = tmp_path / "wide.wav"
    files.write_audio(str(wide), np.zeros((2 * F, 65), np.int16), wav=True)
    _refused([(str(wide), oa)], "has 65 channels: linked channels are at most 64 per file", link_channels="max")
    for kw, match in [(dict(slots=0), "slots"), (dict(slots=1 << 21), "slots"), (dict(chunk_frames=-1), "chunk_frames"),
                      (dict(chunk_frames=1 << 17), "chunk_frames"), (dict(device_pool_bytes=0), "device_pool_bytes"),
                      (dict(decode_threads=300), "decode_threads"), (dict(slots=2.5), "slots"), (dict(slots=True), "slots"),
                      (dict(link_channels="sum"), "link mode")]:
        _refused([(str(a), oa)], match, **kw)
    assert files.denoise_corpus([]) == dict(files=0, useful_stream_frames=0, issued_slot_frames=0, chunks=0, peak_pool_bytes=0,
                                            decode_wait_seconds=0.0, device_wait_seconds=0.0, write_wait_seconds=0.0)


def test_corpus_c_argument_checks(tmp_path):
    """The C checks behind the Python ones: every option field, the link mode and the path arrays."""
    L = nb.lib()
    a = tmp_path / "a.raw"
    a.write_bytes(bytes(4 * F))
    o = tmp_path / "o.raw"
    ins = (C.c_char_p * 1)(os.fsencode(str(a)))
    outs = (C.c_char_p * 1)(os.fsencode(str(o)))
    cases = [(files.CorpusOptions(-1, 0, 0, 0), 0, "slots must be 1..1048576"),
             (files.CorpusOptions(0, 70000, 0, 0), 0, "chunk_frames must be 1..65536"),
             (files.CorpusOptions(0, 0, -5, 0), 0, "device_pool_bytes must be >= 0"),
             (files.CorpusOptions(0, 0, 0, -1), 0, "decode_threads must be 1..256"),
             (files.CorpusOptions(1 << 20, 64, 0, 0), 0, "slots \\* chunk_frames must be at most 2097152"),
             (files.CorpusOptions(0, 0, 0, 0), 3, "link mode 3 is neither")]
    for copt, link, match in cases:
        assert L.rnnoise_denoise_corpus(1, ins, outs, None, link, C.byref(copt), None) == -1
        assert re.search(match, nb.last_error()), nb.last_error()
    assert L.rnnoise_denoise_corpus(-1, ins, outs, None, 0, None, None) == -1 and "bad argument" in nb.last_error()
    assert L.rnnoise_denoise_corpus(1, None, outs, None, 0, None, None) == -1 and "bad argument" in nb.last_error()
    nul = (C.c_char_p * 1)(None)
    assert L.rnnoise_denoise_corpus(1, ins, nul, None, 0, None, None) == -1 and "null path at index 0" in nb.last_error()
    assert not o.exists()
    st = files.CorpusStats()
    assert L.rnnoise_denoise_corpus(0, None, None, None, 0, None, C.byref(st)) == 0 and st.files == 0


def test_corpus_cli_texts(tmp_path):
    h = subprocess.run([files.CLI_PATH, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--slots <N>" in h.stdout and "--chunk-frames <K>" in h.stdout
    for args, match in [(["--slots", "4", "a.wav", "b.wav"], "--slots is only valid with --batch"),
                        (["--batch", "x.list", "--chunk-frames", "4"], "--chunk-frames is only valid with --slots"),
                        (["--batch", "x.list", "--slots", "0"], "Invalid value for '--slots <N>'"),
                        (["--batch", "x.list", "--slots=4", "--chunk-frames=9x"], "Invalid value for '--chunk-frames <K>'"),
                        (["--batch", "x.list", "--slots"], "--slots needs a value")]:
        r = subprocess.run([files.CLI_PATH] + args, capture_output=True, text=True)
        assert r.returncode != 0 and match in r.stderr, (args, r.stderr)
    # a refusal through the binary: the list's output is also its input, and nothing is written
    a = tmp_path / "a.raw"
    a.write_bytes(bytes(4 * F))
    lst = tmp_path / "l.list"
    lst.write_text("%s\t%s\n%s\t%s\n" % (a, tmp_path / "o.raw", a, a))
    r = subprocess.run([files.CLI_PATH, "--batch", str(lst), "--slots", "2"], capture_output=True, text=True)
    assert r.returncode != 0 and "is also an input" in r.stderr and not (tmp_path / "o.raw").exists()


def test_corpus_cpp_mirror_compiles(tmp_path):
    src = tmp_path / "t.cpp"
    src.write_text('#include "nnnoiseless.hpp"\n'
                   "#include <string>\n"
                   "int main(int argc, char** argv) {\n"
                   "    RNNoiseCorpusOptions c{};\n"
                   "    c.slots = -1;\n"
                   "    try {\n"
                   "        nnnoiseless::denoise_corpus({{\"a.wav\", \"b.wav\"}}, nullptr, 0, &c);\n"
                   "    } catch (const std::runtime_error& e) {\n"
                   "        return std::string(e.what()).find(\"slots must be\") == std::string::npos;\n"
                   "    }\n"
                   "    return 2;\n}\n")
    exe = tmp_path / "t"
    libdir = os.path.join(ROOT, "nnnoiseless_b200", "lib")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir,
                        "-lnnnoiseless_b200", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0
