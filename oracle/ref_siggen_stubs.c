/* oracle/ref_siggen_stubs.c -- link-time stand-ins for what the reference's sig_gen.c references but the oracle never
 * reaches (libsamplerate, configuration, the front-end scaling of radio.c).  TEST INFRASTRUCTURE.  Each aborts if it is
 * ever called: the oracle only runs proc_sig_gen's CW loop.  The scheduling helpers of sched.c that the loop and
 * filter.c call are no-ops, so the oracle never changes thread priorities or pinning on the host that runs it. */
#include <stdio.h>
#include <stdlib.h>
#define STUB(name)                                                     \
  void name(void) {                                                    \
    fprintf(stderr, "oracle/_ref: unexpected call of %s\n", #name);    \
    abort();                                                           \
  }
STUB(src_callback_new) STUB(src_callback_read) STUB(src_delete) STUB(src_error) STUB(src_strerror)
STUB(src_short_to_float_array)
STUB(config_getstring) STUB(config_getint) STUB(config_getdouble) STUB(config_getboolean) STUB(config_validate)
STUB(config_validate_section) STUB(scale_AD)
/* sched.c:26-120, as no-ops */
int default_prio(void) { return 0; }
void realtime(int prio) { (void)prio; }
void norealtime(void) {}
void stick_core(void) {}
/* globals radio.c and main.c own */
double Blocktime;
int Verbose;
char const *Description;
