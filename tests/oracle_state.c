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

/* The f32 tables the spectral stages use (src/lib.rs:107-127): window [960], dct [22][22], wnorm. */
void nno_spectral_tables(float *window, float *dct, float *wnorm) {
    ensure_tables();
    memcpy(window, g_window, sizeof g_window);
    memcpy(dct, g_dct, sizeof g_dct);
    *wnorm = g_wnorm;
}
