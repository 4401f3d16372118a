/*
 * Arrow C Data / C Stream / C Device Data / C Device Stream Interface structure
 * definitions.  These are the published, frozen ABI structs of the Apache Arrow
 * format specification (docs: "The Arrow C data interface", "C stream interface",
 * "C device data interface" and its "device stream interface"); every Arrow
 * implementation (arrow-rs `ffi`,
 * pyarrow `_import_from_c/_export_to_c`) binds to exactly this layout.
 * The guards are the ones the specification mandates so this header can be
 * included next to any other copy.
 */
#ifndef DFD_ARROW_C_ABI_H
#define DFD_ARROW_C_ABI_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE

#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4

struct ArrowSchema {
    const char* format;
    const char* name;
    const char* metadata;
    int64_t flags;
    int64_t n_children;
    struct ArrowSchema** children;
    struct ArrowSchema* dictionary;
    void (*release)(struct ArrowSchema*);
    void* private_data;
};

struct ArrowArray {
    int64_t length;
    int64_t null_count;
    int64_t offset;
    int64_t n_buffers;
    int64_t n_children;
    const void** buffers;
    struct ArrowArray** children;
    struct ArrowArray* dictionary;
    void (*release)(struct ArrowArray*);
    void* private_data;
};

#endif /* ARROW_C_DATA_INTERFACE */

#ifndef ARROW_C_STREAM_INTERFACE
#define ARROW_C_STREAM_INTERFACE

struct ArrowArrayStream {
    int (*get_schema)(struct ArrowArrayStream*, struct ArrowSchema* out);
    int (*get_next)(struct ArrowArrayStream*, struct ArrowArray* out);
    const char* (*get_last_error)(struct ArrowArrayStream*);
    void (*release)(struct ArrowArrayStream*);
    void* private_data;
};

#endif /* ARROW_C_STREAM_INTERFACE */

#ifndef ARROW_C_DEVICE_DATA_INTERFACE
#define ARROW_C_DEVICE_DATA_INTERFACE

typedef int32_t ArrowDeviceType;
#define ARROW_DEVICE_CPU 1
#define ARROW_DEVICE_CUDA 2
#define ARROW_DEVICE_CUDA_HOST 3

struct ArrowDeviceArray {
    struct ArrowArray array;
    int64_t device_id;
    ArrowDeviceType device_type;
    void* sync_event; /* cudaEvent_t* for ARROW_DEVICE_CUDA, or NULL */
    int64_t reserved[3];
};

#endif /* ARROW_C_DEVICE_DATA_INTERFACE */

#ifndef ARROW_C_DEVICE_STREAM_INTERFACE
#define ARROW_C_DEVICE_STREAM_INTERFACE

struct ArrowDeviceArrayStream {
    ArrowDeviceType device_type;
    int (*get_schema)(struct ArrowDeviceArrayStream*, struct ArrowSchema* out);
    int (*get_next)(struct ArrowDeviceArrayStream*, struct ArrowDeviceArray* out);
    const char* (*get_last_error)(struct ArrowDeviceArrayStream*);
    void (*release)(struct ArrowDeviceArrayStream*);
    void* private_data;
};

#endif /* ARROW_C_DEVICE_STREAM_INTERFACE */

#ifdef __cplusplus
}
#endif
#endif
