/* oracle/stubs/libbladeRF.h -- declaration-only stand-in for libbladeRF's header, enough for the reference's bladerf.c to
 * compile into the oracle (oracle/ref_bladerf.c).  TEST INFRASTRUCTURE.  The oracle only calls bladerf_process; every
 * function below is an aborting stub (oracle/ref_raw16_stubs.c). */
#ifndef ORACLE_STUB_LIBBLADERF_H
#define ORACLE_STUB_LIBBLADERF_H
#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

struct bladerf;
struct bladerf_stream;
struct bladerf_metadata {
  uint64_t timestamp;
  uint32_t flags, status;
  unsigned int actual_count;
};
struct bladerf_devinfo {
  int backend;
  char serial[33];
  uint8_t usb_bus, usb_addr;
  unsigned int instance;
};
typedef int bladerf_channel;
typedef int bladerf_gain;
#define BLADERF_MODULE_RX ((bladerf_channel)0)
typedef enum { BLADERF_GAIN_DEFAULT, BLADERF_GAIN_MGC, BLADERF_GAIN_FASTATTACK_AGC, BLADERF_GAIN_SLOWATTACK_AGC,
               BLADERF_GAIN_HYBRID_AGC } bladerf_gain_mode;
#define BLADERF_GAIN_AUTOMATIC BLADERF_GAIN_DEFAULT
typedef enum { BLADERF_FORMAT_SC16_Q11, BLADERF_FORMAT_SC16_Q11_META } bladerf_format;
typedef enum { BLADERF_LOG_LEVEL_VERBOSE, BLADERF_LOG_LEVEL_DEBUG, BLADERF_LOG_LEVEL_INFO } bladerf_log_level;
typedef void *(*bladerf_stream_cb)(struct bladerf *dev, struct bladerf_stream *stream, struct bladerf_metadata *meta,
                                   void *samples, size_t num_samples, void *user_data);

void bladerf_log_set_verbosity(bladerf_log_level level);
void bladerf_init_devinfo(struct bladerf_devinfo *info);
int bladerf_open_with_devinfo(struct bladerf **device, struct bladerf_devinfo *devinfo);
int bladerf_open(struct bladerf **device, const char *device_identifier);
void bladerf_close(struct bladerf *device);
const char *bladerf_strerror(int error);
int bladerf_is_fpga_configured(struct bladerf *dev);
int bladerf_set_sample_rate(struct bladerf *dev, bladerf_channel ch, uint32_t rate, uint32_t *actual);
int bladerf_set_bandwidth(struct bladerf *dev, bladerf_channel ch, uint32_t bandwidth, uint32_t *actual);
int bladerf_set_gain_mode(struct bladerf *dev, bladerf_channel ch, bladerf_gain_mode mode);
int bladerf_set_gain(struct bladerf *dev, bladerf_channel ch, bladerf_gain gain);
int bladerf_get_gain(struct bladerf *dev, bladerf_channel ch, bladerf_gain *gain);
int bladerf_set_bias_tee(struct bladerf *dev, bladerf_channel ch, bool enable);
int bladerf_get_bias_tee(struct bladerf *dev, bladerf_channel ch, bool *enable);
int bladerf_set_frequency(struct bladerf *dev, bladerf_channel ch, uint64_t frequency);
int bladerf_init_stream(struct bladerf_stream **stream, struct bladerf *dev, bladerf_stream_cb callback, void ***buffers,
                        size_t num_buffers, bladerf_format format, size_t samples_per_buffer, size_t num_transfers,
                        void *user_data);
int bladerf_enable_module(struct bladerf *dev, bladerf_channel ch, bool enable);
int bladerf_stream(struct bladerf_stream *stream, bladerf_channel layout);
void bladerf_deinit_stream(struct bladerf_stream *stream);
#endif
