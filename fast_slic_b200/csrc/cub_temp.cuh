// fast_slic_b200/csrc/cub_temp.cuh -- the temporary-storage sizes of the CUB calls that several entry points make.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

// cub::DeviceRadixSort::SortPairs of `items` pairs over key bits [0, end_bit)
template <typename Key, typename Value>
static size_t radix_pairs_temp_bytes(long long items, int end_bit) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const Key*)nullptr, (Key*)nullptr, (const Value*)nullptr,
                                    (Value*)nullptr, (int)items, 0, end_bit);
    return bytes;
}

// cub::DeviceScan::ExclusiveSum of `items` values
template <typename T>
static size_t exclusive_sum_temp_bytes(long long items) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const T*)nullptr, (T*)nullptr, (int)items);
    return bytes;
}
