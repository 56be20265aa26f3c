// Host-side harness for tests/test_panel_start_rhs.py: the right-hand side k_panel_start forms for a pairs panel
// (pair_rhs_at, the function the kernel calls per element), over a whole n_pad x kt panel, with its fp32 copy.
#include "../circuitscape_b200/csrc/kernels.cuh"

namespace {

template <typename T, int KT>
void fill(const csb::PanelCtl* ctl, long long n_pad, T* R, float* R32) {
  for (size_t e = 0; e < (size_t)n_pad * KT; ++e) {
    const T r = csb::pair_rhs_at<T, KT>(ctl, e);
    R[e] = r;
    R32[e] = (float)r;
  }
}

template <typename T>
int fill_kt(int kt, const csb::PanelCtl* ctl, long long n_pad, void* R, float* R32) {
  switch (kt) {
    case 1: fill<T, 1>(ctl, n_pad, (T*)R, R32); return 0;
    case 2: fill<T, 2>(ctl, n_pad, (T*)R, R32); return 0;
    case 4: fill<T, 4>(ctl, n_pad, (T*)R, R32); return 0;
    case 8: fill<T, 8>(ctl, n_pad, (T*)R, R32); return 0;
    default: return 1;
  }
}

}  // namespace

// R (n_pad x kt, double if dbl else float) and R32 (n_pad x kt floats) of the pairs panel src / dst
extern "C" int panel_start_pairs(int kt, int dbl, long long n_pad, const long long* src, const long long* dst,
                                 void* R, float* R32) {
  csb::PanelCtl ctl{};
  for (int c = 0; c < kt && c < csb::MAXKT; ++c) {
    ctl.src[c] = src[c];
    ctl.dst[c] = dst[c];
  }
  return dbl ? fill_kt<double>(kt, &ctl, n_pad, R, R32) : fill_kt<float>(kt, &ctl, n_pad, R, R32);
}
