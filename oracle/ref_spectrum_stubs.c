/* oracle/ref_spectrum_stubs.c -- link-time stand-ins for what the reference's spectrum.c references but the oracle
 * never reaches (the status protocol, the channel loop, the demodulator plumbing).  TEST INFRASTRUCTURE.
 * Each aborts if it is ever called: the oracle only calls wideband_poll. */
#include <stdio.h>
#include <stdlib.h>
#define STUB(name)                                                     \
  void name(void) {                                                    \
    fprintf(stderr, "oracle/_ref: unexpected call of %s\n", #name);    \
    abort();                                                           \
  }
STUB(decode_radio_commands) STUB(downconvert) STUB(response)
/* globals radio.c and main.c own (radio.c:130, main.c) */
double Blocktime;
int Verbose;
