// sat_internal.h — the few hooks sat_train.cu needs into the (private) handle of sat_api.cu.
#pragma once
#include "../../include/sat_b200.h"

int sat_fail(int code, const char* fmt, ...);
const sat_dims* sat_handle_dims(sat_handle* h);
void** sat_handle_train_slot(sat_handle* h);
void sat_handle_set_train_free(sat_handle* h, void (*fn)(void*));

// dense product on the wgmma kernel from packed operands (see sat_api.cu); epi = sat::kEpi* of sat_linear.cuh.
// weights_dynamic: the packed weight was produced by the kernel launched just before (it must not be prefetched
// ahead of the dependency wait).
int sat_dense_packed(sat_handle* h, const uint8_t* x_pa, int rows, int row_tile, int K, const uint8_t* wpack,
                     const float* bias_packed, int n_out, int epi, float* out, int ldo, int accumulate, int splits,
                     void* stream, int weights_dynamic = 0);
int sat_handle_layout_mode(sat_handle* h);
int sat_handle_train_tc(sat_handle* h);
// device the handle is bound to (entry points re-select it: the caller may have switched devices since sat_create)
int sat_handle_device(sat_handle* h);
// training-side keys of sat_get_info ("train_bad_ids": word ids outside [0, V) met by the last forward pass);
// returns 1 if the key was handled
int sat_train_info(sat_handle* h, const char* key, int64_t* value, int* rc);
