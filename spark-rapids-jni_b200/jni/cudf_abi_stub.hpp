// cudf_abi_stub.hpp -- stand-ins for the libcudf / rmm declarations the shim touches, so that it can be
// syntax-checked without libcudf (this image has neither libcudf nor rmm headers).  Field meanings follow
// thirdparty/cudf/cpp/include/cudf/column/column_view.hpp:237-244 and types.hpp:191-224; a real build includes
// <cudf/column/column_view.hpp>, <cudf/table/table_view.hpp>, <cudf/column/column_factories.hpp>,
// <cudf/lists/lists_column_view.hpp>, <cudf/scalar/scalar.hpp>, <rmm/device_buffer.hpp>, <rmm/cuda_stream_view.hpp> instead.
#pragma once
#include <cstddef>
#include <cstdint>
#include <memory>
#include <vector>

namespace rmm {
struct cuda_stream_view { void* value() const; void synchronize() const; };
struct device_buffer {
  device_buffer();
  device_buffer(std::size_t bytes, cuda_stream_view stream);
  device_buffer(void const* source, std::size_t bytes, cuda_stream_view stream);   // a device-to-device copy
  void* data();
  std::size_t size() const;
};
}  // namespace rmm

namespace cudf {
using size_type     = int32_t;
using bitmask_type  = uint32_t;
enum class type_id : int32_t { EMPTY = 0, INT8 = 1, INT16 = 2, UINT8 = 5, INT32 = 3, INT64 = 4, FLOAT32 = 9, FLOAT64 = 10, BOOL8 = 11, TIMESTAMP_DAYS = 12, TIMESTAMP_MICROSECONDS = 15,
                              STRING = 23, LIST = 24, DECIMAL32 = 25, DECIMAL64 = 26, DECIMAL128 = 27,
                              STRUCT = 28 };
struct data_type {
  data_type(type_id id, int32_t scale = 0);
  type_id id() const;
  int32_t scale() const;
};
struct column_view {
  column_view(data_type type, size_type size, void const* data, bitmask_type const* null_mask, size_type null_count, size_type offset = 0,
              std::vector<column_view> const& children = {});
  data_type type() const;
  size_type size() const;
  size_type offset() const;
  size_type num_children() const;
  size_type null_count() const;
  column_view child(size_type i) const;
  bitmask_type const* null_mask() const;
  template <typename T> T const* head() const;     // base pointer, offset not applied
};
struct mutable_column_view : column_view {
  template <typename T> T* head() const;
  bitmask_type* null_mask() const;
};
struct table_view {
  size_type num_columns() const;
  size_type num_rows() const;
  column_view column(size_type i) const;
};
struct column {
  column(data_type type, size_type size, rmm::device_buffer&& data, rmm::device_buffer&& null_mask, size_type null_count);
  mutable_column_view mutable_view();
  void set_null_count(size_type n);
};
struct lists_column_view {                           // lists/lists_column_view.hpp
  explicit lists_column_view(column_view const& lists);
  column_view offsets() const;
  column_view child() const;
  size_type size() const;
};
struct scalar {                                      // scalar/scalar.hpp: a device value and a device validity flag
  data_type type() const;
  bool const* validity_data() const;
};
namespace detail {
template <typename T>
struct fixed_width_scalar : scalar {
  T const* data() const;
};
}  // namespace detail
struct string_scalar : scalar {                      // scalar/scalar.hpp: the string's bytes on the device
  char const* data() const;
  size_type size() const;
  bool is_valid(rmm::cuda_stream_view stream) const;
};
struct list_scalar {                                 // scalar/scalar.hpp: one row of a LIST column, held by its child
  list_scalar(column&& data, bool is_valid, rmm::cuda_stream_view stream);
  column_view view() const;
};
std::unique_ptr<column> make_lists_column(size_type num_rows, std::unique_ptr<column> offsets, std::unique_ptr<column> child,
                                          size_type null_count, rmm::device_buffer&& null_mask);
std::unique_ptr<column> make_strings_column(size_type num_rows, std::unique_ptr<column> offsets, rmm::device_buffer&& chars,
                                            size_type null_count, rmm::device_buffer&& null_mask);
std::unique_ptr<column> make_structs_column(size_type num_rows, std::vector<std::unique_ptr<column>>&& child_columns, size_type null_count,
                                            rmm::device_buffer&& null_mask, rmm::cuda_stream_view stream);
rmm::cuda_stream_view get_default_stream();
namespace jni {
void auto_set_device(JNIEnv* env);
}  // namespace jni
}  // namespace cudf
