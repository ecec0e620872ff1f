/* oracle/ref_iqcorr_stubs.c -- link-time stand-ins for what the reference's hackrf.c and funcube.c reference but the
 * oracle never reaches (device control, configuration, the front-end scaling of radio.c).  TEST INFRASTRUCTURE.
 * Each aborts if it is ever called: the oracle only runs rx_callback and proc_funcube.  The scheduling helpers of
 * sched.c that the sample loops and filter.c call are no-ops, so the oracle never changes thread priorities or
 * pinning on the host that runs it. */
#include <stdio.h>
#include <stdlib.h>
#define STUB(name)                                                     \
  void name(void) {                                                    \
    fprintf(stderr, "oracle/_ref: unexpected call of %s\n", #name);    \
    abort();                                                           \
  }
STUB(hackrf_init) STUB(hackrf_exit) STUB(hackrf_error_name) STUB(hackrf_device_list) STUB(hackrf_device_list_open)
STUB(hackrf_device_list_free) STUB(hackrf_open) STUB(hackrf_start_rx) STUB(hackrf_stop_rx) STUB(hackrf_set_freq)
STUB(hackrf_set_sample_rate) STUB(hackrf_set_baseband_filter_bandwidth) STUB(hackrf_compute_baseband_filter_bw_round_down_lt)
STUB(hackrf_set_lna_gain) STUB(hackrf_set_vga_gain) STUB(hackrf_set_antenna_enable)
STUB(Pa_Initialize) STUB(Pa_Terminate) STUB(Pa_GetDeviceCount) STUB(Pa_GetDeviceInfo) STUB(Pa_OpenStream)
STUB(fcdOpen) STUB(fcdClose) STUB(fcdGetMode) STUB(fcdGetCapsStr) STUB(fcdAppSetFreq) STUB(fcdAppSetParam)
STUB(config_getstring) STUB(config_getint) STUB(config_getdouble) STUB(config_getboolean) STUB(config_validate)
STUB(config_validate_section) STUB(scale_AD) STUB(scale_ADpower2FS)
/* sched.c:26-120, as no-ops */
int default_prio(void) { return 0; }
void realtime(int prio) { (void)prio; }
void norealtime(void) {}
void stick_core(void) {}
/* globals radio.c and main.c own */
double Blocktime;
int Verbose;
char const *Description;
