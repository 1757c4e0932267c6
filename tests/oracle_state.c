/*
 * oracle_state.c -- state records (the layout of rnnoise_batch_get_states, include/rnnoise.h) for the CPU oracle.
 *
 * TEST INFRASTRUCTURE ONLY.  Compiled together with oracle/nno_oracle.c, with the oracle's own flags, by
 * tests/oracle_state.py, so that tests can build and check records without a GPU.  The oracle itself is unchanged:
 * its nno_state keeps input_mem oldest first and cepstral_mem indexed by ring slot, exactly the record's order.
 * The analysis and synthesis stages of a frame can also be run on their own from given inputs (nno_analysis_frame,
 * nno_synthesis_from), so that tests can measure the oracle's own f32 error on the inputs the GPU saw.
 */
#include "../oracle/nno_oracle.c"

#define REC_MAGIC 0x54534E52u /* "RNST" */
#define REC_VERSION 1
#define OFF_INPUT 128
#define OFF_CEPS 7040
#define OFF_SYNTH 7744
#define OFF_GRU 9664

size_t nno_state_bytes(const nno_model *m) {
    return ((size_t)OFF_GRU + 4 * (size_t)(m->vad_gru.nn + m->noise_gru.nn + m->denoise_gru.nn) + 15) & ~(size_t)15;
}

/* rec: nno_state_bytes(model) bytes */
void nno_state_export(const nno_state *s, void *rec) {
    const nno_model *m = s->model;
    const int nv = m->vad_gru.nn, nn = m->noise_gru.nn, nd = m->denoise_gru.nn;
    unsigned char *r = (unsigned char *)rec;
    memset(r, 0, nno_state_bytes(m));
    const int32_t head[7] = {(int32_t)REC_MAGIC, REC_VERSION, nv, nn, nd, s->mem_id, s->last_period};
    memcpy(r, head, sizeof head);
    memcpy(r + 28, &s->last_gain, 4);
    memcpy(r + 32, s->mem_hp_x, sizeof s->mem_hp_x);
    memcpy(r + 40, s->lastg, sizeof s->lastg);
    memcpy(r + OFF_INPUT, s->input_mem, sizeof s->input_mem);
    memcpy(r + OFF_CEPS, s->cepstral_mem, sizeof s->cepstral_mem);
    memcpy(r + OFF_SYNTH, s->synthesis_mem, sizeof s->synthesis_mem);
    memcpy(r + OFF_GRU, s->vad_gru_state, 4 * (size_t)nv);
    memcpy(r + OFF_GRU + 4 * nv, s->noise_gru_state, 4 * (size_t)nn);
    memcpy(r + OFF_GRU + 4 * (nv + nn), s->denoise_gru_state, 4 * (size_t)nd);
}

/* 0: imported; -1: rejected by the same checks as rnnoise_batch_set_states (s unchanged) */
int nno_state_import(nno_state *s, const void *rec) {
    const nno_model *m = s->model;
    const int nv = m->vad_gru.nn, nn = m->noise_gru.nn, nd = m->denoise_gru.nn;
    const unsigned char *r = (const unsigned char *)rec;
    int32_t head[7];
    memcpy(head, r, sizeof head);
    if ((uint32_t)head[0] != REC_MAGIC || head[1] != REC_VERSION || head[2] != nv || head[3] != nn || head[4] != nd) return -1;
    if (head[5] < 0 || head[5] >= CEPS_MEM || head[6] < 0 || head[6] > PITCH_MAX_PERIOD) return -1;
    s->mem_id = head[5];
    s->last_period = head[6];
    memcpy(&s->last_gain, r + 28, 4);
    memcpy(s->mem_hp_x, r + 32, sizeof s->mem_hp_x);
    memcpy(s->lastg, r + 40, sizeof s->lastg);
    memcpy(s->input_mem, r + OFF_INPUT, sizeof s->input_mem);
    memcpy(s->cepstral_mem, r + OFF_CEPS, sizeof s->cepstral_mem);
    memcpy(s->synthesis_mem, r + OFF_SYNTH, sizeof s->synthesis_mem);
    memcpy(s->vad_gru_state, r + OFF_GRU, 4 * (size_t)nv);
    memcpy(s->noise_gru_state, r + OFF_GRU + 4 * nv, 4 * (size_t)nn);
    memcpy(s->denoise_gru_state, r + OFF_GRU + 4 * (nv + nn), 4 * (size_t)nd);
    return 0;
}

/* ---- the two spectral stages of nno_process_frame on their own, for tests of the GPU's analysis and synthesis kernels
 * one frame at a time.  Complex arrays are interleaved (re, im). ---- */

/* shift_and_filter then compute_frame_features on s (a state imported from a record taken before the frame): the
 * oracle's X, P (all 481 bins), ex, ep, exp, features, the cepstral ring and mem_id after the frame, the pitch it found
 * and input_mem after the high-pass.  Any output pointer may be NULL.  Returns the silence flag. */
int nno_analysis_frame(nno_state *s, const float *in, float *X, float *P, float *ex, float *ep, float *exp, float *features,
                       float *ceps, int32_t *mem_id, int32_t *pitch, float *input_mem) {
    shift_and_filter(s, in);
    const int silence = compute_frame_features(s);
    for (int k = 0; k < FREQ_SIZE; k++) {
        if (X) {
            X[2 * k] = s->x_re[k];
            X[2 * k + 1] = s->x_im[k];
        }
        if (P) {
            P[2 * k] = s->p_re[k];
            P[2 * k + 1] = s->p_im[k];
        }
    }
    if (ex) memcpy(ex, s->ex, sizeof s->ex);
    if (ep) memcpy(ep, s->ep, sizeof s->ep);
    if (exp) memcpy(exp, s->exp, sizeof s->exp);
    if (features) memcpy(features, s->features, sizeof s->features);
    if (ceps) memcpy(ceps, s->cepstral_mem, sizeof s->cepstral_mem);
    if (mem_id) *mem_id = s->mem_id;
    if (pitch) *pitch = s->taps.pitch;
    if (input_mem) memcpy(input_mem, s->input_mem, sizeof s->input_mem);
    return silence;
}

/* The statements of nno_process_frame after the network, on the given inputs: pitch_filter, the gain floor,
 * interp_band_gain, the gains applied, frame_synthesis (a silent frame goes straight to frame_synthesis).  X and P are
 * [481][2]; lastg [22] and synth_mem [480] are updated in place; out [480]. */
void nno_synthesis_from(const float *X, const float *P, const float *ex, const float *ep, const float *exp, const float *raw_gains,
                        float *lastg, float *synth_mem, int silence, float *out) {
    nno_state *s = (nno_state *)calloc(1, sizeof(*s));
    float g[NB_BANDS], gf[FREQ_SIZE];
    ensure_tables();
    for (int k = 0; k < FREQ_SIZE; k++) {
        s->x_re[k] = X[2 * k];
        s->x_im[k] = X[2 * k + 1];
        s->p_re[k] = P[2 * k];
        s->p_im[k] = P[2 * k + 1];
    }
    memcpy(s->ex, ex, sizeof s->ex);
    memcpy(s->ep, ep, sizeof s->ep);
    memcpy(s->exp, exp, sizeof s->exp);
    memcpy(s->lastg, lastg, sizeof s->lastg);
    memcpy(s->synthesis_mem, synth_mem, sizeof s->synthesis_mem);
    memcpy(g, raw_gains, sizeof g);
    if (!silence) {
        pitch_filter(s, g);
        for (int i = 0; i < NB_BANDS; i++) {
            g[i] = fmaxf(g[i], 0.6f * s->lastg[i]);
            s->lastg[i] = g[i];
        }
        interp_band_gain(gf, g);
        for (int i = 0; i < FREQ_SIZE; i++) {
            s->x_re[i] *= gf[i];
            s->x_im[i] *= gf[i];
        }
    }
    frame_synthesis(s, out);
    memcpy(lastg, s->lastg, sizeof s->lastg);
    memcpy(synth_mem, s->synthesis_mem, sizeof s->synthesis_mem);
    free(s);
}

/* ---- pitch_process (src/pitch.rs:45-221) in stages, for tests of the pitch kernel's decisions.  The oracle's own static
 * functions run in pitch_process's order on a 1728-sample buffer; every f32 value a decision is taken from is kept. ---- */
#define NL4 ((PITCH_MAX_PERIOD - 3 * PITCH_MIN_PERIOD) / 4) /* 147 coarse lags */
#define NL2 ((PITCH_MAX_PERIOD - 3 * PITCH_MIN_PERIOD) / 2) /* 294 fine lags */
#define NK 14                                              /* ladder steps k = 2..15 */

typedef struct {
    float pitch_buf[PITCH_BUF_SIZE / 2];   /* whitened, 2x decimated (pitch_downsample) */
    float xcorr4[NL4], ysq4[NL4];          /* coarse xcorr and find_best_pitch's y_sq_norm seen at each lag */
    int32_t best4, second4;
    float xcorr2[NL2], ysq2[NL2];          /* fine xcorr (0 outside the two windows) and its y_sq_norm at each lag */
    int32_t best2, offset2, pitch_idx;     /* fine best, pitch_search's +-1 offset, PITCH_MAX_PERIOD - (2 best - offset) */
    int32_t t0;
    float xx, xy0, g0;
    float yy_raw[PITCH_MAX_PERIOD / 2 + 1];    /* remove_doubling's running yy before the clamp */
    float yy_lookup[PITCH_MAX_PERIOD / 2 + 1]; /* ... and after it */
    int32_t nk;                            /* ladder steps run (k = 2 .. nk + 1) */
    int32_t t1[NK], t1b[NK], taken[NK];
    float xy[NK], yy[NK], g1[NK], cont[NK], thresh[NK];
    float xc[3];                           /* inner products at t - 1, t, t + 1 */
    int32_t t, offset, period;
    float gain;
} nno_pitch_stages_t;

size_t nno_pitch_stages_bytes(void) { return sizeof(nno_pitch_stages_t); }

/* pitch_process on buf [1728] with the given carried last_period / last_gain; returns the period. */
int32_t nno_pitch_stages(const float *buf, int32_t last_period, float last_gain, nno_pitch_stages_t *o) {
    memset(o, 0, sizeof *o);
    float *pb = o->pitch_buf;
    pitch_downsample(buf, pb);

    /* pitch_search (src/pitch.rs:63-115) */
    const float *x_lp = pb + PITCH_MAX_PERIOD / 2, *y = pb;
    const int len = PITCH_FRAME_SIZE, n4 = len / 4, ny4 = len / 4 + NL4;
    float x_lp4[PITCH_FRAME_SIZE / 4], y_lp4[PITCH_FRAME_SIZE / 4 + NL4];
    for (int j = 0; j < n4; j++) x_lp4[j] = x_lp[2 * j];
    for (int j = 0; j < ny4; j++) y_lp4[j] = y[2 * j];
    pitch_xcorr(x_lp4, n4, y_lp4, o->xcorr4, NL4);
    find_best_pitch(o->xcorr4, NL4, y_lp4, n4, &o->best4, &o->second4);
    float ys = 1.0f; /* find_best_pitch's running energy, the same statements */
    for (int j = 0; j < n4; j++) ys += y_lp4[j] * y_lp4[j];
    for (int i = 0; i < NL4; i++) {
        o->ysq4[i] = ys;
        ys += y_lp4[i + n4] * y_lp4[i + n4] - y_lp4[i] * y_lp4[i];
        ys = fmaxf(ys, 1.0f);
    }
    for (int i = 0; i < NL2; i++) {
        o->xcorr2[i] = 0.0f;
        if (abs(i - 2 * o->best4) > 2 && abs(i - 2 * o->second4) > 2) continue;
        o->xcorr2[i] = fmaxf(inner_prod(x_lp, y + i, len / 2), -1.0f);
    }
    int dummy;
    find_best_pitch(o->xcorr2, NL2, y, len / 2, &o->best2, &dummy);
    ys = 1.0f;
    for (int j = 0; j < len / 2; j++) ys += y[j] * y[j];
    for (int i = 0; i < NL2; i++) {
        o->ysq2[i] = ys;
        ys += y[i + len / 2] * y[i + len / 2] - y[i] * y[i];
        ys = fmaxf(ys, 1.0f);
    }
    const int best = o->best2;
    if (best > 0 && best < NL2 - 1) {
        float a = o->xcorr2[best - 1], b = o->xcorr2[best], c = o->xcorr2[best + 1];
        if (c - a > 0.7f * (b - a)) o->offset2 = 1;
        else if (a - c > 0.7f * (b - c)) o->offset2 = -1;
    }
    o->pitch_idx = PITCH_MAX_PERIOD - (2 * best - o->offset2);

    /* remove_doubling (src/pitch.rs:118-221) */
    const float *x = pb;
    const int min_period = PITCH_MIN_PERIOD / 2, max_period = PITCH_MAX_PERIOD / 2, n = PITCH_FRAME_SIZE / 2;
    int t0 = o->pitch_idx / 2;
    if (t0 > max_period - 1) t0 = max_period - 1;
    o->t0 = t0;
    const int prev_period = last_period / 2;
    float xx = inner_prod(x + max_period, x + max_period, n);
    float xy = inner_prod(x + max_period, x + max_period - t0, n);
    o->xx = xx;
    o->xy0 = xy;
    o->yy_raw[0] = o->yy_lookup[0] = xx;
    float yy = xx;
    for (int i = 1; i <= max_period; i++) {
        yy += x[max_period - i] * x[max_period - i] - x[max_period + n - i] * x[max_period + n - i];
        o->yy_raw[i] = yy;
        o->yy_lookup[i] = fmaxf(yy, 0.0f);
    }
    yy = o->yy_lookup[t0];
    float best_xy = xy, best_yy = yy;
    const float g0 = pitch_gain(xy, xx, yy);
    float g = g0;
    int t = t0;
    o->g0 = g0;
    for (int k = 2; k <= 15; k++) {
        int t1 = (2 * t0 + k) / (2 * k);
        if (t1 < min_period) break;
        int t1b;
        if (k == 2) t1b = (t1 + t0 > max_period) ? t0 : t0 + t1;
        else t1b = (2 * SECOND_CHECK[k] * t0 + k) / (2 * k);
        xy = inner_prod(x + max_period, x + max_period - t1, n);
        float xy2 = inner_prod(x + max_period, x + max_period - t1b, n);
        xy = (xy + xy2) / 2.0f;
        yy = (o->yy_lookup[t1] + o->yy_lookup[t1b]) / 2.0f;
        float g1 = pitch_gain(xy, xx, yy);
        float cont;
        int d = abs(t1 - prev_period);
        if (d <= 1) cont = last_gain;
        else if (d <= 2 && 5 * k * k < t0) cont = last_gain / 2.0f;
        else cont = 0.0f;
        float thresh;
        if (t1 < 3 * min_period) thresh = fmaxf(0.85f * g0 - cont, 0.4f);
        else if (t1 < 2 * min_period) thresh = fmaxf(0.9f * g0 - cont, 0.5f);
        else thresh = fmaxf(0.7f * g0 - cont, 0.3f);
        const int s = o->nk++;
        o->t1[s] = t1;
        o->t1b[s] = t1b;
        o->xy[s] = xy;
        o->yy[s] = yy;
        o->g1[s] = g1;
        o->cont[s] = cont;
        o->thresh[s] = thresh;
        o->taken[s] = g1 > thresh;
        if (g1 > thresh) {
            best_xy = xy;
            best_yy = yy;
            t = t1;
            g = g1;
        }
    }
    best_xy = fmaxf(best_xy, 0.0f);
    float pg = (best_yy <= best_xy) ? 1.0f : best_xy / (best_yy + 1.0f);
    for (int k = 0; k < 3; k++) o->xc[k] = inner_prod(x + max_period, x + max_period - (t + k - 1), n);
    int offset = 0;
    if (o->xc[2] - o->xc[0] > 0.7f * (o->xc[1] - o->xc[0])) offset = 1;
    else if (o->xc[0] - o->xc[2] > 0.7f * (o->xc[1] - o->xc[2])) offset = -1;
    pg = fminf(pg, g);
    int tf = 2 * t + offset;
    if (tf < PITCH_MIN_PERIOD) tf = PITCH_MIN_PERIOD;
    o->t = t;
    o->offset = offset;
    o->period = tf;
    o->gain = pg;
    return tf;
}

/* pitch_process through the oracle's own entry point, on a state carrying last_period / last_gain: (period, gain).
 * (The pitch path reads no model.) */
int32_t nno_pitch_only_from(const float *buf, int32_t last_period, float last_gain, float *gain) {
    nno_state *s = nno_state_new(NULL);
    s->last_period = last_period;
    s->last_gain = last_gain;
    const int32_t p = nno_pitch_only(s, buf);
    *gain = s->last_gain;
    nno_state_free(s);
    return p;
}

/* The input high-pass (src/util.rs:95-107) over n samples from the filter memory mem [2] (updated): the samples
 * shift_and_filter appends to input_mem. */
void nno_highpass(const float *in, int n, float *out, float *mem) { biquad_hp(out, mem, in, n); }

/* The state of a training lane after its most recent nno_train_frame: NoiseSimulator::vad_count, the random filters'
 * memories resp_mem [4] = (signal_resp_mem, noise_resp_mem), the band energies ex [3][22] and a state record (rec: 3
 * records of nno_state_bytes(m) bytes) of each of its clean, noise and combined feature extractors.  The extractors run
 * no network; m only gives the records their GRU widths. */
void nno_train_probe(const nno_trainer *t, const nno_model *m, int32_t *vad_count, float *resp_mem, float *ex, void *rec) {
    *vad_count = t->vad_count;
    memcpy(resp_mem, t->signal_resp_mem, sizeof t->signal_resp_mem);
    memcpy(resp_mem + 2, t->noise_resp_mem, sizeof t->noise_resp_mem);
    const nno_state *s[3] = {t->clean, t->noise, t->comb};
    for (int k = 0; k < 3; k++) {
        nno_state tmp = *s[k];
        tmp.model = m;
        memcpy(ex + k * NB_BANDS, tmp.ex, sizeof tmp.ex);
        nno_state_export(&tmp, (unsigned char *)rec + k * nno_state_bytes(m));
    }
}

/* transform_input's band energies of n given 960-sample windows (win [n][960]): each window is multiplied by the
 * analysis window, transformed by nno_rfft960 (under the current nno_set_fft_mode), scaled by wnorm and summed into
 * bands by compute_band_corr.  X [n][481][2] (interleaved re, im; may be NULL), ex [n][22]. */
void nno_band_energies(const float *win, int n, float *X, float *ex) {
    ensure_tables();
    float w[WINDOW_SIZE], re[FREQ_SIZE], im[FREQ_SIZE];
    for (int s = 0; s < n; s++) {
        const float *in = win + (size_t)s * WINDOW_SIZE;
        for (int i = 0; i < WINDOW_SIZE; i++) w[i] = in[i] * g_window[i];
        nno_rfft960(w, re, im);
        for (int i = 0; i < FREQ_SIZE; i++) {
            re[i] *= g_wnorm;
            im[i] *= g_wnorm;
            if (X) {
                X[((size_t)s * FREQ_SIZE + i) * 2] = re[i];
                X[((size_t)s * FREQ_SIZE + i) * 2 + 1] = im[i];
            }
        }
        compute_band_corr(ex + (size_t)s * NB_BANDS, re, im, re, im);
    }
}

/* The f32 tables the spectral stages use (src/lib.rs:107-127): window [960], dct [22][22], wnorm. */
void nno_spectral_tables(float *window, float *dct, float *wnorm) {
    ensure_tables();
    memcpy(window, g_window, sizeof g_window);
    memcpy(dct, g_dct, sizeof g_dct);
    *wnorm = g_wnorm;
}
