/* oracle/ref_float_stubs.c -- link-time stand-ins for what the reference's airspyhf.c, fobos.c and hydrasdr.c reference
 * but the oracle never reaches (device control, configuration, the front-end scaling of radio.c).  TEST INFRASTRUCTURE.
 * Each aborts if it is ever called: the oracle only runs the three rx_callbacks (HydraSDR's software AGC off).  The
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
STUB(airspyhf_lib_version) STUB(airspyhf_list_devices) STUB(airspyhf_open_sn) STUB(airspyhf_close)
STUB(airspyhf_version_string_read) STUB(airspyhf_get_samplerates) STUB(airspyhf_set_samplerate) STUB(airspyhf_set_hf_agc)
STUB(airspyhf_set_hf_agc_threshold) STUB(airspyhf_set_hf_att) STUB(airspyhf_set_hf_lna) STUB(airspyhf_set_lib_dsp)
STUB(airspyhf_start) STUB(airspyhf_stop) STUB(airspyhf_is_streaming) STUB(airspyhf_set_freq)
STUB(fobos_rx_get_api_info) STUB(fobos_rx_list_devices) STUB(fobos_rx_open) STUB(fobos_rx_close)
STUB(fobos_rx_get_board_info) STUB(fobos_rx_set_frequency) STUB(fobos_rx_set_direct_sampling) STUB(fobos_rx_set_lna_gain)
STUB(fobos_rx_set_vga_gain) STUB(fobos_rx_get_samplerates) STUB(fobos_rx_set_samplerate) STUB(fobos_rx_set_clk_source)
STUB(fobos_rx_read_async) STUB(fobos_rx_cancel_async)
STUB(config_getstring) STUB(config_getint) STUB(config_getdouble) STUB(config_getboolean)
STUB(config_validate_section) STUB(scale_AD) STUB(scale_ADpower2FS)
/* sched.c:26-120, as no-ops */
int default_prio(void) { return 0; }
void realtime(int prio) { (void)prio; }
void norealtime(void) {}
void stick_core(void) {}
/* globals main.c owns; Blocktime at its default of 20 ms (main.c), which fobos.c's Power_alpha reads */
int Verbose;
char const *Description;
char const *Serial;
char const *App_path;
double Blocktime = 20.0e-3;
