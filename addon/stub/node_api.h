/* NOT node_api.h: a declaration-only stand-in for the handful of N-API entry points addon/amgpu_napi.cc uses, so that the
 * addon can be syntax- and type-checked (`make -C addon check`) in a build image without Node. Signatures follow the Node
 * documentation (N-API version 3). Never used to build the real addon: node-gyp supplies the real header. */
#ifndef AMG_NODE_API_STUB_H
#define AMG_NODE_API_STUB_H
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#ifdef __cplusplus
extern "C" {
#endif
typedef struct napi_env__* napi_env;
typedef struct napi_value__* napi_value;
typedef struct napi_callback_info__* napi_callback_info;
typedef enum { napi_ok, napi_invalid_arg, napi_generic_failure } napi_status;
typedef enum { napi_int8_array, napi_uint8_array, napi_uint8_clamped_array, napi_int16_array, napi_uint16_array, napi_int32_array, napi_uint32_array, napi_float32_array, napi_float64_array } napi_typedarray_type;
typedef napi_value (*napi_callback)(napi_env env, napi_callback_info info);
typedef void (*napi_finalize)(napi_env env, void* finalize_data, void* finalize_hint);
#define NAPI_AUTO_LENGTH ((size_t)-1)
napi_status napi_throw_error(napi_env env, const char* code, const char* msg);
napi_status napi_throw_type_error(napi_env env, const char* code, const char* msg);
napi_status napi_throw_range_error(napi_env env, const char* code, const char* msg);
napi_status napi_create_external(napi_env env, void* data, napi_finalize finalize_cb, void* finalize_hint, napi_value* result);
napi_status napi_get_value_external(napi_env env, napi_value value, void** result);
napi_status napi_is_typedarray(napi_env env, napi_value value, bool* result);
napi_status napi_is_array(napi_env env, napi_value value, bool* result);
napi_status napi_get_typedarray_info(napi_env env, napi_value typedarray, napi_typedarray_type* type, size_t* length, void** data, napi_value* arraybuffer, size_t* byte_offset);
napi_status napi_create_arraybuffer(napi_env env, size_t byte_length, void** data, napi_value* result);
napi_status napi_create_typedarray(napi_env env, napi_typedarray_type type, size_t length, napi_value arraybuffer, size_t byte_offset, napi_value* result);
napi_status napi_get_undefined(napi_env env, napi_value* result);
napi_status napi_create_array_with_length(napi_env env, size_t length, napi_value* result);
napi_status napi_create_object(napi_env env, napi_value* result);
napi_status napi_set_element(napi_env env, napi_value object, uint32_t index, napi_value value);
napi_status napi_get_element(napi_env env, napi_value object, uint32_t index, napi_value* result);
napi_status napi_get_array_length(napi_env env, napi_value value, uint32_t* result);
napi_status napi_get_cb_info(napi_env env, napi_callback_info cbinfo, size_t* argc, napi_value* argv, napi_value* this_arg, void** data);
napi_status napi_get_value_bool(napi_env env, napi_value value, bool* result);
napi_status napi_get_value_double(napi_env env, napi_value value, double* result);
napi_status napi_create_double(napi_env env, double value, napi_value* result);
napi_status napi_create_string_utf8(napi_env env, const char* str, size_t length, napi_value* result);
napi_status napi_create_error(napi_env env, napi_value code, napi_value msg, napi_value* result);
napi_status napi_create_range_error(napi_env env, napi_value code, napi_value msg, napi_value* result);
napi_status napi_create_type_error(napi_env env, napi_value code, napi_value msg, napi_value* result);
napi_status napi_throw(napi_env env, napi_value error);
napi_status napi_remove_wrap(napi_env env, napi_value js_object, void** result);
napi_status napi_create_function(napi_env env, const char* utf8name, size_t length, napi_callback cb, void* data, napi_value* result);
napi_status napi_set_named_property(napi_env env, napi_value object, const char* utf8name, napi_value value);
napi_status napi_get_named_property(napi_env env, napi_value object, const char* utf8name, napi_value* result);
napi_status napi_get_value_uint32(napi_env env, napi_value value, uint32_t* result);
#define NAPI_MODULE(modname, regfunc) extern "C" napi_value napi_register_module_v1(napi_env env, napi_value exports) { return regfunc(env, exports); }
#define NODE_GYP_MODULE_NAME amgpu_napi
#ifdef __cplusplus
}
#endif
#endif
