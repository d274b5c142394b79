/*
 * device_b200_component.c -- MCA glue of the b200 device component (parsec/mca/device/b200).
 *
 * Fills parsec_device_base_component_t the way every PaRSEC device component has to (device.h:54-58; the contract is
 * spelled out in SURVEY.md 8b; the reference's CUDA component is parsec/mca/device/cuda/device_cuda_component.c):
 * register -> MCA parameters; open -> count devices; query -> NULL-terminated array of modules, priority;
 * close -> finalise and remove the modules.  Everything device specific is in device_b200_module.c.
 *
 * Selection: the component is enabled with  --mca device_b200_enabled N  (or PARSEC_MCA_device_b200_enabled=N; -1 = all
 * GPUs; default 0 = off so that an unmodified installation keeps the reference's cuda component).  When it is enabled
 * it turns device_cuda_enabled off: both components answer to PARSEC_DEV_CUDA chores and must not drive the same GPU.
 */
#include "parsec/parsec_config.h"
#include "parsec/parsec_internal.h"
#include "parsec/utils/mca_param.h"
#include "parsec/utils/debug.h"
#include "parsec/constants.h"
#include "parsec/mca/device/device.h"
#include "parsec/mca/device/device_gpu.h"
#include "parsec/mca/device/b200/device_b200.h"
#include "parsec/mca/device/b200/device_b200_internal.h"

#include <stdlib.h>

int parsec_device_b200_enabled = 0;
int parsec_device_b200_enabled_index = -1;
int parsec_b200_dry_run = 0;
int parsec_b200_memory_block_size = 512 * 1024;
int parsec_b200_memory_percentage = 95;
int parsec_b200_memory_number_of_blocks = -1;
int parsec_b200_cmd_slots = 65536;
int parsec_b200_idle_us = 2000;
int parsec_b200_max_workers = 0;
char *parsec_b200_trace = NULL;
int parsec_b200_nvtx = 0;
int parsec_b200_parallel_completion = 1;
int parsec_b200_stage_window = 32 * 1024 * 1024;
int parsec_b200_registration_cache = 1;
static int b200_mask = -1;

#if !defined(PARSEC_HAVE_MPI)
/* read by the shared GPU code (device_gpu.c:261, :3261); parsec_mpi_funnelled.c, its home, is only built with MPI */
int parsec_mpi_allow_gpu_memory_communications = 0;
#endif

static int device_b200_component_open(void);
static int device_b200_component_close(void);
static int device_b200_component_query(mca_base_module_2_0_0_t **module, int *priority);
static int device_b200_component_register(void);

parsec_device_base_component_t parsec_device_b200_component = {
    {
        PARSEC_DEVICE_BASE_VERSION_2_0_0,
        "b200",
        "+persistent_kernel+device_release+tma",
        PARSEC_VERSION_MAJOR,
        PARSEC_VERSION_MINOR,
        device_b200_component_open,
        device_b200_component_close,
        device_b200_component_query,
        device_b200_component_register,
        "",
    },
    {
        MCA_BASE_METADATA_PARAM_NONE,
        "",
    },
    NULL
};

mca_base_component_t *device_b200_static_component(void)
{
    return (mca_base_component_t *)&parsec_device_b200_component;
}

static int device_b200_component_register(void)
{
    parsec_device_b200_enabled_index =
        parsec_mca_param_reg_int_name("device_b200", "enabled",
                                      "Number of GPUs driven by the b200 engine (-1: all available, 0: component off)",
                                      false, false, 0, &parsec_device_b200_enabled);
    (void)parsec_mca_param_reg_int_name("device_b200", "mask", "Bit mask of the CUDA devices the component may use",
                                        false, false, -1, &b200_mask);
    (void)parsec_mca_param_reg_int_name("device_b200", "dry_run",
                                        "Host-logic test mode: build modules without touching CUDA; tasks retire in dependency order "
                                        "without running their bodies (the value is the number of pretend devices)",
                                        false, false, 0, &parsec_b200_dry_run);
    (void)parsec_mca_param_reg_int_name("device_b200", "memory_block_size", "Unit of the device heap in bytes",
                                        false, false, 512 * 1024, &parsec_b200_memory_block_size);
    (void)parsec_mca_param_reg_int_name("device_b200", "memory_use", "Percentage of the free GPU memory given to the device heap",
                                        false, false, 95, &parsec_b200_memory_percentage);
    (void)parsec_mca_param_reg_int_name("device_b200", "memory_number_of_blocks",
                                        "Exact number of heap blocks instead of a percentage (-1: use device_b200_memory_use)",
                                        false, false, -1, &parsec_b200_memory_number_of_blocks);
    (void)parsec_mca_param_reg_int_name("device_b200", "cmd_slots", "Capacity of the host->device command ring (tasks in flight)",
                                        false, false, 65536, &parsec_b200_cmd_slots);
    (void)parsec_mca_param_reg_int_name("device_b200", "idle_us", "The persistent kernel parks after this many idle microseconds",
                                        false, false, 2000, &parsec_b200_idle_us);
    (void)parsec_mca_param_reg_int_name("device_b200", "parallel_completion",
                                        "Let the worker pool run __parsec_complete_execution of finished GPU tasks instead of the manager thread",
                                        false, false, 1, &parsec_b200_parallel_completion);
    (void)parsec_mca_param_reg_int_name("device_b200", "stage_window",
                                        "Bytes of stage-in (host or peer to device) allowed in flight before further cold tasks wait",
                                        false, false, 32 * 1024 * 1024, &parsec_b200_stage_window);
    (void)parsec_mca_param_reg_int_name("device_b200", "registration_cache",
                                        "Keep host ranges pinned after memory_unregister and revive them at the next registration of the same range",
                                        false, false, 1, &parsec_b200_registration_cache);
    (void)parsec_mca_param_reg_int_name("device_b200", "max_workers", "Debug: limit the worker CTAs of the persistent kernel (0: all)",
                                        false, false, 0, &parsec_b200_max_workers);
    (void)parsec_mca_param_reg_string_name("device_b200", "trace",
                                           "Write one Chrome-trace JSON file <value>.<device index>.json per device at finalize: every task with the "
                                           "device-clock time a worker CTA started and finished it and the SM it ran on (empty: off)",
                                           false, false, "", &parsec_b200_trace);
    (void)parsec_mca_param_reg_int_name("device_b200", "nvtx",
                                        "Wrap the host side of the device in NVTX ranges (domain \"parsec_b200\": start pass, retire pass, "
                                        "epilog batch) and mark every manager election; what profiling_nvtx.c does for the profiling keys "
                                        "of the reference's stream engine",
                                        false, false, 0, &parsec_b200_nvtx);
    return (0 == parsec_device_b200_enabled && 0 == parsec_b200_dry_run) ? MCA_ERROR : MCA_SUCCESS;
}

static int device_b200_component_open(void)
{
    int ndev = 0;
    if( 0 == parsec_device_b200_enabled && 0 == parsec_b200_dry_run ) return MCA_ERROR;
    if( parsec_b200_dry_run > 0 ) {
        ndev = parsec_b200_dry_run;
    } else {
        ndev = parsec_b200_device_count();
        if( ndev <= 0 ) {
            parsec_warning("device_b200: enabled but no sm_90 CUDA device is usable on %s; component disabled", parsec_hostname);
            parsec_device_b200_enabled = 0;
            return MCA_ERROR;
        }
        if( parsec_device_b200_enabled > 0 && parsec_device_b200_enabled < ndev ) ndev = parsec_device_b200_enabled;
    }
    parsec_device_b200_enabled = ndev;
    /* both components answer PARSEC_DEV_CUDA chores: never let the reference's stream engine drive the same GPUs.
     * Components are registered and opened one after the other in list order (mca_repository.c:128-141) and "b200"
     * sorts before "cuda": its parameters are not registered yet, so the switch is thrown where it will look. */
    setenv("PARSEC_MCA_device_cuda_enabled", "0", 1);
    {
        int idx = parsec_mca_param_find("device_cuda", NULL, "enabled");
        if( idx >= 0 ) parsec_mca_param_set_int(idx, 0);
    }
    return MCA_SUCCESS;
}

static int device_b200_component_query(mca_base_module_2_0_0_t **module, int *priority)
{
    int i, j;
    *module = NULL;
    *priority = 0;
    if( parsec_device_b200_enabled <= 0 ) return MCA_SUCCESS;
    parsec_device_b200_component.modules = (parsec_device_module_t**)calloc(parsec_device_b200_enabled + 1, sizeof(parsec_device_module_t*));
    for( i = j = 0; i < parsec_device_b200_enabled; i++ ) {
        if( !((1 << i) & b200_mask) ) continue;
        if( PARSEC_SUCCESS != parsec_b200_module_init(i, &parsec_device_b200_component.modules[j]) ) continue;
        parsec_device_b200_component.modules[j]->component = &parsec_device_b200_component;
        j++;
        parsec_device_b200_component.modules[j] = NULL;
    }
    *priority = 20;     /* above the cuda component (10): when both could run, the engine wins */
    *module = (mca_base_module_2_0_0_t*)(void*)parsec_device_b200_component.modules;
    return MCA_SUCCESS;
}

static int device_b200_component_close(void)
{
    parsec_device_module_t *dev;
    if( NULL == parsec_device_b200_component.modules ) return MCA_SUCCESS;
    for( int i = 0; NULL != (dev = parsec_device_b200_component.modules[i]); i++ ) {
        parsec_device_b200_component.modules[i] = NULL;
        parsec_b200_module_fini(dev);
        (void)parsec_mca_device_remove(dev);
        free(dev);
    }
    free(parsec_device_b200_component.modules);
    parsec_device_b200_component.modules = NULL;
    return MCA_SUCCESS;
}
