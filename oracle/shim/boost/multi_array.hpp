/* Stand-in for boost::multi_array (TEST INFRASTRUCTURE, see oracle/shim/Eigen/Core): the 3-D subset that planning_ros_utils'
 * voxel_grid.cpp uses — construction from boost::extents[a][b][c], resize, data, num_elements, m[i][j][k] and assignment.
 * Storage is C order (last index fastest) like Boost's default.  resize() here does not keep the old elements, unlike Boost's;
 * voxel_grid.cpp assigns a whole new array right after every resize (vg:161-164), so nothing observes the difference. */
#ifndef MPLB_SHIM_BOOST_MULTI_ARRAY
#define MPLB_SHIM_BOOST_MULTI_ARRAY
#include <cstddef>
#include <vector>
namespace boost {
struct extent_gen {
  std::size_t e[3];
  int n;
  extent_gen operator[](long long v) const {
    extent_gen g = *this;
    g.e[g.n++] = (std::size_t)v;
    return g;
  }
};
static const extent_gen extents = {{0, 0, 0}, 0};

template <class T, std::size_t N>
class multi_array;

template <class T>
class multi_array<T, 3> {
  std::vector<T> d_;
  std::size_t e_[3] = {0, 0, 0};

 public:
  struct Row2 {
    T *p;
    T &operator[](long long k) const { return p[k]; }
  };
  struct Row1 {
    T *p;
    std::size_t e2;
    Row2 operator[](long long j) const { return Row2{p + j * e2}; }
  };
  multi_array() {}
  explicit multi_array(const extent_gen &g) { resize(g); }
  void resize(const extent_gen &g) {
    for (int i = 0; i < 3; i++) e_[i] = g.e[i];
    d_.assign(e_[0] * e_[1] * e_[2], T());
  }
  T *data() { return d_.data(); }
  const T *data() const { return d_.data(); }
  std::size_t num_elements() const { return d_.size(); }
  Row1 operator[](long long i) { return Row1{d_.data() + i * e_[1] * e_[2], e_[2]}; }
};
}  // namespace boost
#endif
