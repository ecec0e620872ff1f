/* oracle/ref_raw16_stubs.c -- link-time stand-ins for what the reference's hydrasdr.c and bladerf.c reference but the
 * oracle never reaches (device control, configuration, the front-end scaling of radio.c).  TEST INFRASTRUCTURE.
 * Each aborts if it is ever called: the oracle only runs rx_callback (software AGC off) and bladerf_process.  The
 * scheduling helpers of sched.c are no-ops, so the oracle never changes thread priorities or pinning on the host that
 * runs it. */
#include <stdio.h>
#include <stdlib.h>
#define STUB(name)                                                     \
  void name(void) {                                                    \
    fprintf(stderr, "oracle/_ref: unexpected call of %s\n", #name);    \
    abort();                                                           \
  }
STUB(hydrasdr_lib_version) STUB(hydrasdr_list_devices) STUB(hydrasdr_open_sn) STUB(hydrasdr_close)
STUB(hydrasdr_error_name) STUB(hydrasdr_get_device_info) STUB(hydrasdr_set_packing) STUB(hydrasdr_set_sample_type)
STUB(hydrasdr_get_samplerates) STUB(hydrasdr_set_samplerate) STUB(hydrasdr_set_gain) STUB(hydrasdr_get_gain)
STUB(hydrasdr_set_rf_bias) STUB(hydrasdr_start_rx) STUB(hydrasdr_stop_rx) STUB(hydrasdr_is_streaming)
STUB(hydrasdr_set_freq)
STUB(bladerf_log_set_verbosity) STUB(bladerf_init_devinfo) STUB(bladerf_open_with_devinfo) STUB(bladerf_open)
STUB(bladerf_close) STUB(bladerf_strerror) STUB(bladerf_is_fpga_configured) STUB(bladerf_set_sample_rate)
STUB(bladerf_set_bandwidth) STUB(bladerf_set_gain_mode) STUB(bladerf_set_gain) STUB(bladerf_get_gain)
STUB(bladerf_set_bias_tee) STUB(bladerf_get_bias_tee) STUB(bladerf_set_frequency) STUB(bladerf_init_stream)
STUB(bladerf_enable_module) STUB(bladerf_stream) STUB(bladerf_deinit_stream)
STUB(config_getstring) STUB(config_getint) STUB(config_getdouble) STUB(config_getboolean)
STUB(config_validate_section) STUB(scale_AD) STUB(scale_ADpower2FS)
/* sched.c:26-120, as no-ops */
int default_prio(void) { return 0; }
void realtime(int prio) { (void)prio; }
void norealtime(void) {}
void stick_core(void) {}
/* globals main.c owns */
int Verbose;
char const *Description;
char const *Serial;
