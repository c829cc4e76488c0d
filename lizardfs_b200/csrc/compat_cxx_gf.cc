// compat_cxx_gf.cc — C++-LINKAGE twins of the Galois-field names.
//
// The reference has two spellings of this layer: <isa-l/erasure_code.h> declares gf_gen_rs_matrix ... ec_encode_data with C
// linkage (what engine.cu / host_math.cc export), while its own src/common/galois_field.h:35-88 declares the same names
// WITHOUT extern "C" (they are defined in galois_field_isal.cc / galois_field_encode.cc as C++ functions).  A build of the
// reference that does not define LIZARDFS_HAVE_ISA_L_ERASURE_CODE_H therefore references the mangled names
// (_Z16gf_gen_rs_matrixPhii, _Z14ec_encode_dataiiiPhPS_S0_, ...).  This translation unit defines those, forwarding to the C
// symbols through their lzgpu_isal_* aliases — it must not see the extern "C" declarations of the same names, which is why it
// is a file of its own and does not include lzgpu.h.  Tested by oracle/_ref/test_link_substitution_cxx (the reference's
// reed_solomon_unittest.cc compiled against galois_field.h).
#include <cstdint>

extern "C" {
void lzgpu_isal_gf_gen_rs_matrix(unsigned char *a, int m, int k);
void lzgpu_isal_gf_gen_cauchy1_matrix(unsigned char *a, int m, int k);
int lzgpu_isal_gf_invert_matrix(unsigned char *in, unsigned char *out, const int n);
void lzgpu_isal_ec_init_tables(int k, int rows, unsigned char *a, unsigned char *gftbls);
void lzgpu_isal_ec_encode_data(int len, int srcs, int dests, unsigned char *v, unsigned char **src, unsigned char **dest);
}

void gf_gen_rs_matrix(uint8_t *a, int m, int k) { lzgpu_isal_gf_gen_rs_matrix(a, m, k); }
void gf_gen_cauchy1_matrix(uint8_t *a, int m, int k) { lzgpu_isal_gf_gen_cauchy1_matrix(a, m, k); }
int gf_invert_matrix(uint8_t *in_mat, uint8_t *out_mat, const int n) { return lzgpu_isal_gf_invert_matrix(in_mat, out_mat, n); }
void ec_init_tables(int k, int rows, uint8_t *a, uint8_t *g_tbls) { lzgpu_isal_ec_init_tables(k, rows, a, g_tbls); }
void ec_encode_data(int len, int srcs, int dests, uint8_t *v, uint8_t **src, uint8_t **dest) { lzgpu_isal_ec_encode_data(len, srcs, dests, v, src, dest); }
