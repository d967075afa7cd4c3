// TEST INFRASTRUCTURE: compiles the device's callback signing (callback_sign.cuh: SHA-256, the HMAC midstates, the
// streaming base64 record path, the non-finite test and the kwargs walk) for the host, so that tests/test_callback_on_host.py
// can compare it with hashlib / hmac / base64 and json on a CPU.
#include <stdint.h>
#include <string.h>
#define __device__
#define __host__
#define __forceinline__ inline
#define __constant__ static const
#include "../../beta9_b200/csrc/callback_sign.cuh"

static void words_to_bytes(const uint32_t w[8], uint8_t out[32]) {
    for (int i = 0; i < 8; ++i) { out[4 * i] = (uint8_t)(w[i] >> 24); out[4 * i + 1] = (uint8_t)(w[i] >> 16); out[4 * i + 2] = (uint8_t)(w[i] >> 8); out[4 * i + 3] = (uint8_t)w[i]; }
}

extern "C" {

void b9_cb_sha256(const uint8_t* p, uint64_t n, uint8_t out[32]) { b9::sha256(p, n, out); }

// HMAC-SHA256(key, msg) through the midstates and the byte-stream path
void b9_cb_hmac(const uint8_t* key, uint32_t key_len, const uint8_t* msg, uint64_t n, uint8_t out[32]) {
    uint32_t mid[16];
    b9::cb_midstates(key, key_len, mid);
    b9::hmac_sha256(mid, msg, n, out);
}

// the record path: HMAC(key, "eyJkYXRhIjog" + base64(R + "}") + ":" + ts), fed word by word from R; *blocks = its inner blocks
void b9_cb_sign_record(const uint8_t* key, uint32_t key_len, int64_t ts, const uint8_t* r, uint32_t len, uint8_t out[32], uint32_t* blocks) {
    uint32_t mid[16], o[8];
    b9::cb_midstates(key, key_len, mid);
    b9::CbSign s;
    b9::cb_sign_init(s, mid, ts);
    b9::cb_sign_record(s, r, len, o);
    words_to_bytes(o, out);
    *blocks = b9::cb_inner_blocks(s, len);
}

int b9_cb_nonfinite(const uint8_t* r, uint32_t len) { return b9::cb_nonfinite(r, len) ? 1 : 0; }

// mode 0: an SDK put payload, 1: an HTTP body, 2: a TaskMessage record
int b9_cb_kwargs_have_callback_url(const uint8_t* p, uint32_t n, int mode) { return b9::cb_kwargs_have_callback_url(p, n, mode) ? 1 : 0; }

}
