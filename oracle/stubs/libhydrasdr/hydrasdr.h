/* oracle/stubs/libhydrasdr/hydrasdr.h -- declaration-only stand-in for libhydrasdr's header, enough for the reference's
 * hydrasdr.c to compile into the oracle (oracle/ref_hydrasdr.c).  TEST INFRASTRUCTURE.  The oracle only calls
 * rx_callback with the software AGC off; every function below is an aborting stub (oracle/ref_raw16_stubs.c). */
#ifndef ORACLE_STUB_LIBHYDRASDR_H
#define ORACLE_STUB_LIBHYDRASDR_H
#include <stdbool.h>
#include <stdint.h>

#define HYDRASDR_VER_MAJOR 1
#define HYDRASDR_VER_MINOR 1
#define HYDRASDR_VER_REVISION 2
#define HYDRASDR_MAKE_VERSION(a, b, c) (((uint32_t)(a) << 16) | ((uint32_t)(b) << 8) | (uint32_t)(c))

enum hydrasdr_error { HYDRASDR_SUCCESS = 0, HYDRASDR_ERROR_OTHER = -9999 };
enum hydrasdr_sample_type {
  HYDRASDR_SAMPLE_FLOAT32_IQ = 0,
  HYDRASDR_SAMPLE_FLOAT32_REAL,
  HYDRASDR_SAMPLE_INT16_IQ,
  HYDRASDR_SAMPLE_INT16_REAL,
  HYDRASDR_SAMPLE_UINT16_REAL,
  HYDRASDR_SAMPLE_RAW,
  HYDRASDR_SAMPLE_INT8_IQ,
  HYDRASDR_SAMPLE_UINT8_IQ,
  HYDRASDR_SAMPLE_INT8_REAL,
  HYDRASDR_SAMPLE_UINT8_REAL,
  HYDRASDR_SAMPLE_END
};
enum hydrasdr_gain_type {
  HYDRASDR_GAIN_TYPE_LNA = 0,
  HYDRASDR_GAIN_TYPE_RF,
  HYDRASDR_GAIN_TYPE_MIXER,
  HYDRASDR_GAIN_TYPE_FILTER,
  HYDRASDR_GAIN_TYPE_VGA,
  HYDRASDR_GAIN_TYPE_LINEARITY,
  HYDRASDR_GAIN_TYPE_SENSITIVITY,
  HYDRASDR_GAIN_TYPE_LNA_AGC,
  HYDRASDR_GAIN_TYPE_RF_AGC,
  HYDRASDR_GAIN_TYPE_MIXER_AGC,
  HYDRASDR_GAIN_TYPE_FILTER_AGC
};
enum {
  HYDRASDR_CAP_LNA_GAIN = 1 << 0,
  HYDRASDR_CAP_RF_GAIN = 1 << 1,
  HYDRASDR_CAP_MIXER_GAIN = 1 << 2,
  HYDRASDR_CAP_FILTER_GAIN = 1 << 3,
  HYDRASDR_CAP_VGA_GAIN = 1 << 4,
  HYDRASDR_CAP_LINEARITY_GAIN = 1 << 5,
  HYDRASDR_CAP_SENSITIVITY_GAIN = 1 << 6,
  HYDRASDR_CAP_LNA_AGC = 1 << 7,
  HYDRASDR_CAP_RF_AGC = 1 << 8,
  HYDRASDR_CAP_MIXER_AGC = 1 << 9,
  HYDRASDR_CAP_FILTER_AGC = 1 << 10,
  HYDRASDR_CAP_BIAS_TEE = 1 << 11,
  HYDRASDR_CAP_PACKING = 1 << 12
};

struct hydrasdr_device;
typedef struct {
  struct hydrasdr_device *device;
  void *ctx;
  void *samples;
  int sample_count;
  uint64_t dropped_samples;
  enum hydrasdr_sample_type sample_type;
} hydrasdr_transfer;
typedef int (*hydrasdr_sample_block_cb_fn)(hydrasdr_transfer *transfer);
typedef struct {
  uint32_t major_version, minor_version, revision;
} hydrasdr_lib_version_t;
typedef struct {
  uint8_t min_value, max_value, default_value, value;
} hydrasdr_gain_info_t;
typedef struct {
  char board_name[64];
  char firmware_version[128];
  uint32_t features;
  uint32_t sample_types;
  uint8_t current_adc_bits;
  hydrasdr_gain_info_t lna_gain, rf_gain, mixer_gain, filter_gain, vga_gain, linearity_gain, sensitivity_gain;
} hydrasdr_device_info_t;

void hydrasdr_lib_version(hydrasdr_lib_version_t *lib_version);
int hydrasdr_list_devices(uint64_t *serials, int count);
int hydrasdr_open_sn(struct hydrasdr_device **device, uint64_t serial_number);
int hydrasdr_open(struct hydrasdr_device **device);
int hydrasdr_close(struct hydrasdr_device *device);
const char *hydrasdr_error_name(enum hydrasdr_error errcode);
int hydrasdr_get_device_info(struct hydrasdr_device *device, hydrasdr_device_info_t *info);
int hydrasdr_set_packing(struct hydrasdr_device *device, uint8_t value);
int hydrasdr_set_sample_type(struct hydrasdr_device *device, enum hydrasdr_sample_type sample_type);
int hydrasdr_get_samplerates(struct hydrasdr_device *device, uint32_t *buffer, const uint32_t len);
int hydrasdr_set_samplerate(struct hydrasdr_device *device, uint32_t samplerate);
int hydrasdr_set_gain(struct hydrasdr_device *device, enum hydrasdr_gain_type type, uint8_t value);
int hydrasdr_get_gain(struct hydrasdr_device *device, enum hydrasdr_gain_type type, hydrasdr_gain_info_t *info);
int hydrasdr_set_rf_bias(struct hydrasdr_device *device, uint8_t value);
int hydrasdr_start_rx(struct hydrasdr_device *device, hydrasdr_sample_block_cb_fn callback, void *rx_ctx);
int hydrasdr_stop_rx(struct hydrasdr_device *device);
int hydrasdr_is_streaming(struct hydrasdr_device *device);
int hydrasdr_set_freq(struct hydrasdr_device *device, const uint64_t freq_hz);
#endif
