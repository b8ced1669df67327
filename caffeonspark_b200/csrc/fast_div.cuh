// fast_div.cuh -- integer division by a divisor fixed at launch, for the kernels that split a flat index into
// coordinates (caffe_layers.cu, native_producer.cu).
#ifndef COS_FAST_DIV_CUH_
#define COS_FAST_DIV_CUH_

namespace cosb {

// n / d for 0 <= n < 2^31 with a multiply-high and a shift instead of an integer division (a division per
// element costs more issue slots than the element's memory traffic takes time)
struct FastDiv {
  unsigned d, m, s;
  explicit FastDiv(unsigned div) : d(div), m(0), s(0) {
    while (s < 31 && (1u << s) < d) ++s;
    m = (unsigned)((((1ull << 32) * ((1ull << s) - d)) / d) + 1);
  }
  __device__ __forceinline__ unsigned div(unsigned n) const { return (__umulhi(n, m) + n) >> s; }
};

}  // namespace cosb
#endif
