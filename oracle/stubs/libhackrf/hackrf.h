/* oracle/stubs/libhackrf/hackrf.h -- declaration-only stand-in for libhackrf's header, enough for the reference's
 * hackrf.c to compile into the oracle (oracle/ref_hackrf.c).  TEST INFRASTRUCTURE.  The oracle only calls rx_callback;
 * every function below is an aborting stub (oracle/ref_iqcorr_stubs.c). */
#ifndef ORACLE_STUB_LIBHACKRF_H
#define ORACLE_STUB_LIBHACKRF_H
#include <stdint.h>

enum hackrf_error { HACKRF_SUCCESS = 0, HACKRF_TRUE = 1, HACKRF_ERROR_OTHER = -9999 };

typedef struct hackrf_device hackrf_device;
typedef struct {
  hackrf_device *device;
  uint8_t *buffer;
  int buffer_length;
  int valid_length;
  void *rx_ctx;
  void *tx_ctx;
} hackrf_transfer;
typedef struct {
  const char **serial_numbers;
  int *usb_board_ids;
  int *usb_device_index;
  int devicecount;
  void **usb_devices;
  int usb_devicecount;
} hackrf_device_list_t;
typedef int (*hackrf_sample_block_cb_fn)(hackrf_transfer *transfer);

int hackrf_init(void);
int hackrf_exit(void);
const char *hackrf_error_name(enum hackrf_error errcode);
hackrf_device_list_t *hackrf_device_list(void);
int hackrf_device_list_open(hackrf_device_list_t *list, int idx, hackrf_device **device);
void hackrf_device_list_free(hackrf_device_list_t *list);
int hackrf_open(hackrf_device **device);
int hackrf_start_rx(hackrf_device *device, hackrf_sample_block_cb_fn callback, void *rx_ctx);
int hackrf_stop_rx(hackrf_device *device);
int hackrf_set_freq(hackrf_device *device, const uint64_t freq_hz);
int hackrf_set_sample_rate(hackrf_device *device, const double freq_hz);
int hackrf_set_baseband_filter_bandwidth(hackrf_device *device, const uint32_t bandwidth_hz);
uint32_t hackrf_compute_baseband_filter_bw_round_down_lt(const uint32_t bandwidth_hz);
int hackrf_set_lna_gain(hackrf_device *device, uint32_t value);
int hackrf_set_vga_gain(hackrf_device *device, uint32_t value);
int hackrf_set_antenna_enable(hackrf_device *device, const uint8_t value);
#endif
