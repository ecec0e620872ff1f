/* oracle/stubs/samplerate.h -- declaration-only stand-in for libsamplerate's header, enough for the reference's
 * sig_gen.c to compile into the oracle (oracle/ref_siggen.c).  TEST INFRASTRUCTURE.  The oracle drives only the CW loop,
 * which never reaches these; they are aborting stubs (oracle/ref_siggen_stubs.c). */
#ifndef ORACLE_STUB_SAMPLERATE_H
#define ORACLE_STUB_SAMPLERATE_H
typedef struct SRC_STATE_tag SRC_STATE;
typedef long (*src_callback_t)(void *cb_data, float **data);
enum { SRC_SINC_BEST_QUALITY = 0, SRC_SINC_MEDIUM_QUALITY = 1, SRC_SINC_FASTEST = 2, SRC_ZERO_ORDER_HOLD = 3, SRC_LINEAR = 4 };
SRC_STATE *src_callback_new(src_callback_t func, int converter_type, int channels, int *error, void *cb_data);
long src_callback_read(SRC_STATE *state, double src_ratio, long frames, float *data);
SRC_STATE *src_delete(SRC_STATE *state);
int src_error(SRC_STATE *state);
const char *src_strerror(int error);
void src_short_to_float_array(const short *in, float *out, int len);
#endif
