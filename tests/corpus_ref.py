"""A literal, frame-by-frame restatement of the reference's readers (src/training.rs): ``SignalReader::new``,
``next_reader`` and ``frame`` (:185-260) and the schedule of ``NoiseSimulator::next_frame`` (:388-395), for L lanes
stepped in lockstep and drawing from one generator in the order nnnoiseless_b200.training documents.  A reader is
reduced to what decides the rows: which file it has open and at which sample it stands.  tests/test_training_corpus.py
holds training.plan to it."""
import numpy as np

from nnnoiseless_b200.training import GAIN_CHANGE_COUNT, randomize

FRAME_SIZE = 480


class SignalReader:
    def __init__(self, lens, count, cur_idx):
        assert len(lens) > 0, "cannot read from an empty set of files"
        self.lens = lens
        self.frames_per_file = max(count // len(lens) + 1, 100)
        self.cur_idx = cur_idx
        self.frames_left = 0
        self.reader = None  # the open file's next sample, or None

    def next_reader(self, rng):
        if self.cur_idx >= len(self.lens):
            self.cur_idx = 0
        length = int(self.lens[self.cur_idx])
        num_samples = FRAME_SIZE * self.frames_per_file
        pos = 0
        if length > num_samples:
            pos = int(rng.integers(0, length - num_samples, endpoint=True))  # gen_range(0..=(len - num_samples))
            self.frames_left = self.frames_per_file
        else:
            self.frames_left = length // FRAME_SIZE
        if self.frames_left > 0:
            self.reader = pos

    def frame(self, rng):
        """-> (file index, first sample) of the frame it reads."""
        while self.reader is None:
            self.next_reader(rng)
        at = (self.cur_idx, self.reader)
        self.reader += FRAME_SIZE
        if self.frames_left <= 1:
            self.reader = None
            self.cur_idx += 1
        else:
            self.frames_left -= 1
        return at


def run(sig_lens, noise_lens, count, lanes, seed, shuffle):
    """-> (signal (file, offset) [F][L][2], noise [F][L][2], {frame: params [L]}, signal order, noise order)."""
    rng = np.random.default_rng(seed)
    ps, pn = np.arange(len(sig_lens)), np.arange(len(noise_lens))
    if shuffle:
        ps, pn = rng.permutation(len(sig_lens)), rng.permutation(len(noise_lens))
    sl, nl = np.asarray(sig_lens)[ps], np.asarray(noise_lens)[pn]
    F = -(-count // lanes)
    sig = [SignalReader(sl, count, (l * len(sl)) // lanes) for l in range(lanes)]
    noise = [SignalReader(nl, count, (l * len(nl)) // lanes) for l in range(lanes)]
    gain_change_count = 0
    at_s = np.zeros((F, lanes, 2), np.int64)
    at_n = np.zeros((F, lanes, 2), np.int64)
    params = {}
    for f in range(F):
        gain_change_count += 1  # next_frame: increment, then test
        if gain_change_count > GAIN_CHANGE_COUNT:
            gain_change_count = 0
            params[f] = randomize(lanes, rng)
        for l in range(lanes):
            at_n[f, l] = noise[l].frame(rng)  # read_noise before read_signal
            at_s[f, l] = sig[l].frame(rng)
    return at_s, at_n, params, ps, pn
