/* ref_rand_shim.c -- linked into oracle/_ref/libpvnet_refextend.so next to the reference's unmodified
 * farthest_point_sampling.cpp (oracle/extend.mk).  Its random-start mode begins at rand() % pn after
 * srand(time(0)); with -Wl,-Bsymbolic the library's own calls bind to these definitions, so that start is the value
 * set by pvnet_ref_set_start() and the reference's output can be recorded and compared. */
static int start_value;

__attribute__((visibility("default"))) int rand(void) { return start_value; }

__attribute__((visibility("default"))) void srand(unsigned seed) { (void)seed; }

__attribute__((visibility("default"))) void pvnet_ref_set_start(int s) { start_value = s; }
