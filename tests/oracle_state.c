/*
 * oracle_state.c -- state records (the layout of rnnoise_batch_get_states, include/rnnoise.h) for the CPU oracle.
 *
 * TEST INFRASTRUCTURE ONLY.  Compiled together with oracle/nno_oracle.c, with the oracle's own flags, by
 * tests/oracle_state.py, so that tests can build and check records without a GPU.  The oracle itself is unchanged:
 * its nno_state keeps input_mem oldest first and cepstral_mem indexed by ring slot, exactly the record's order.
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
