/* oracle/stubs/libairspyhf/airspyhf.h -- declaration-only stand-in for libairspyhf's header, enough for the reference's
 * airspyhf.c to compile into the oracle (oracle/ref_airspyhf.c).  TEST INFRASTRUCTURE.  The oracle only calls rx_callback;
 * every function below is an aborting stub (oracle/ref_float_stubs.c). */
#ifndef ORACLE_STUB_LIBAIRSPYHF_H
#define ORACLE_STUB_LIBAIRSPYHF_H
#include <stdint.h>

enum airspyhf_error { AIRSPYHF_SUCCESS = 0, AIRSPYHF_ERROR = -1 };
typedef struct {
  float re, im;
} airspyhf_complex_float_t;
struct airspyhf_device;
typedef struct airspyhf_device airspyhf_device_t;
typedef struct {
  airspyhf_device_t *device;
  void *ctx;
  airspyhf_complex_float_t *samples;
  int sample_count;
  uint64_t dropped_samples;
} airspyhf_transfer_t;
typedef struct {
  uint32_t major_version, minor_version, revision;
} airspyhf_lib_version_t;
typedef int (*airspyhf_sample_block_cb_fn)(airspyhf_transfer_t *transfer);

void airspyhf_lib_version(airspyhf_lib_version_t *lib_version);
int airspyhf_list_devices(uint64_t *serials, int count);
int airspyhf_open_sn(airspyhf_device_t **device, uint64_t serial_number);
int airspyhf_close(airspyhf_device_t *device);
int airspyhf_version_string_read(airspyhf_device_t *device, char *version, uint8_t length);
int airspyhf_get_samplerates(airspyhf_device_t *device, uint32_t *buffer, const uint32_t len);
int airspyhf_set_samplerate(airspyhf_device_t *device, uint32_t samplerate);
int airspyhf_set_hf_agc(airspyhf_device_t *device, uint8_t flag);
int airspyhf_set_hf_agc_threshold(airspyhf_device_t *device, uint8_t flag);
int airspyhf_set_hf_att(airspyhf_device_t *device, uint8_t value);
int airspyhf_set_hf_lna(airspyhf_device_t *device, uint8_t flag);
int airspyhf_set_lib_dsp(airspyhf_device_t *device, uint8_t flag);
int airspyhf_start(airspyhf_device_t *device, airspyhf_sample_block_cb_fn callback, void *ctx);
int airspyhf_stop(airspyhf_device_t *device);
int airspyhf_is_streaming(airspyhf_device_t *device);
int airspyhf_set_freq(airspyhf_device_t *device, const uint32_t freq_hz);
#endif
