/* oracle/stubs/fobos.h -- declaration-only stand-in for libfobos's header, enough for the reference's fobos.c to compile
 * into the oracle (oracle/ref_fobos.c).  TEST INFRASTRUCTURE.  The oracle only calls rx_callback; every function below is
 * an aborting stub (oracle/ref_float_stubs.c). */
#ifndef ORACLE_STUB_FOBOS_H
#define ORACLE_STUB_FOBOS_H
#include <stdint.h>

#define FOBOS_ERR_OK 0
struct fobos_dev_t;
typedef void (*fobos_rx_cb_t)(float *buf, uint32_t buf_length, void *ctx);

int fobos_rx_get_api_info(char *lib_version, char *drv_version);
int fobos_rx_list_devices(char *serials);
int fobos_rx_open(struct fobos_dev_t **out_dev, uint32_t index);
int fobos_rx_close(struct fobos_dev_t *dev);
int fobos_rx_get_board_info(struct fobos_dev_t *dev, char *hw_revision, char *fw_version, char *manufacturer, char *product,
                            char *serial);
int fobos_rx_set_frequency(struct fobos_dev_t *dev, double value, double *actual);
int fobos_rx_set_direct_sampling(struct fobos_dev_t *dev, unsigned int enabled);
int fobos_rx_set_lna_gain(struct fobos_dev_t *dev, unsigned int value);
int fobos_rx_set_vga_gain(struct fobos_dev_t *dev, unsigned int value);
int fobos_rx_get_samplerates(struct fobos_dev_t *dev, double *values, unsigned int *count);
int fobos_rx_set_samplerate(struct fobos_dev_t *dev, double value, double *actual);
int fobos_rx_set_clk_source(struct fobos_dev_t *dev, int value);
int fobos_rx_read_async(struct fobos_dev_t *dev, fobos_rx_cb_t cb, void *ctx, uint32_t buf_count, uint32_t buf_length);
int fobos_rx_cancel_async(struct fobos_dev_t *dev);
#endif
