/*
 * barb200_shim_env.h -- the GPUs a shim's engine context drives, from the environment; shared by cactus_bar_shim.c (POA mode)
 * and cactus_pecan_shim.c (cPecan mode) so that both modes read the same settings the same way:
 *
 *   BARB200_DEVICE=<ordinal>           one GPU for this process
 *   BARB200_DEVICES=all | 0,1,2,3      several GPUs behind ONE context (up to 8; the list wins over BARB200_DEVICE)
 */
#ifndef BARB200_SHIM_ENV_H
#define BARB200_SHIM_ENV_H
#include <stdlib.h>
#include <string.h>
#include "barb200.h"

static void barb200_devices_from_env(barb200_params *p) {
    const char *dev = getenv("BARB200_DEVICE");
    if (dev) p->device = atoi(dev);
    const char *devs = getenv("BARB200_DEVICES");
    if (devs) {
        if (strcmp(devs, "all") == 0) {
            p->n_devices = -1;
        } else {
            p->n_devices = 0;
            for (const char *c = devs; *c && p->n_devices < 8; ) {
                p->devices[p->n_devices++] = atoi(c);
                while (*c && *c != ',') c++;
                if (*c == ',') c++;
            }
        }
    }
}

#endif
