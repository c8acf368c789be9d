// alz_pow2.h -- CPython 3.12's float `k ** 2` on x86-64 glibc 2.39, restated for host and device.
//
// CPython's float_pow settles NaN, +-inf, 0 and |k| == 1 itself and hands the rest to libm's pow(|k|, 2.0); a result
// that is infinite raises OverflowError.  glibc's pow is not correctly rounded, so `k ** 2 != k * k` for about one
// double in 1400: the bits of pow are those of glibc's table-driven algorithm (a log in double-double from a 128-entry
// table, times y, then a 128-entry exp), as compiled for CPUs with FMA, which glibc selects at load time on any x86-64
// with FMA and AVX2.  alz_pow2_glibc restates that compiled code operation for operation: every fma below is one the
// compiler emitted (including the contractions of a product into an add it chose), and every other operation is a
// single IEEE rounding.  With y == 2 the products y * hi and y * lo are exact, so only the log, the exp and the exp's
// special paths remain.  The tables are the words of __pow_log_data (invc, logc, logctail) and __exp_data's tab in
// that libm's .rodata; the scalar constants are spelled as hexadecimal floats.
//
// On the device the tables are read with __ldg: lanes of a warp index them divergently, which __constant__ memory
// would serialize.  Units that include this file must not contract (nvcc -fmad=false, host -ffp-contract=off); the
// device path spells every operation with an explicit round-to-nearest intrinsic anyway.
#pragma once

#include <stdint.h>
#include <string.h>
#include <math.h>

#ifdef __CUDACC__
#define ALZ_POW2_HD __host__ __device__ __forceinline__
#else
#define ALZ_POW2_HD static inline
#endif

#define ALZ_POW2_LOG_TAB { \
  0x3ff6a00000000000ULL, 0xbfd62c82f2b9c800ULL, 0x3cfab42428375680ULL, \
  0x3ff6800000000000ULL, 0xbfd5d1bdbf580800ULL, 0xbd1ca508d8e0f720ULL, \
  0x3ff6600000000000ULL, 0xbfd5767717455800ULL, 0xbd2362a4d5b6506dULL, \
  0x3ff6400000000000ULL, 0xbfd51aad872df800ULL, 0xbce684e49eb067d5ULL, \
  0x3ff6200000000000ULL, 0xbfd4be5f95777800ULL, 0xbd041b6993293ee0ULL, \
  0x3ff6000000000000ULL, 0xbfd4618bc21c6000ULL, 0x3d13d82f484c84ccULL, \
  0x3ff5e00000000000ULL, 0xbfd404308686a800ULL, 0x3cdc42f3ed820b3aULL, \
  0x3ff5c00000000000ULL, 0xbfd3a64c55694800ULL, 0x3d20b1c686519460ULL, \
  0x3ff5a00000000000ULL, 0xbfd347dd9a988000ULL, 0x3d25594dd4c58092ULL, \
  0x3ff5800000000000ULL, 0xbfd2e8e2bae12000ULL, 0x3d267b1e99b72bd8ULL, \
  0x3ff5600000000000ULL, 0xbfd2895a13de8800ULL, 0x3d15ca14b6cfb03fULL, \
  0x3ff5600000000000ULL, 0xbfd2895a13de8800ULL, 0x3d15ca14b6cfb03fULL, \
  0x3ff5400000000000ULL, 0xbfd22941fbcf7800ULL, 0xbd165a242853da76ULL, \
  0x3ff5200000000000ULL, 0xbfd1c898c1699800ULL, 0xbd1fafbc68e75404ULL, \
  0x3ff5000000000000ULL, 0xbfd1675cababa800ULL, 0x3d1f1fc63382a8f0ULL, \
  0x3ff4e00000000000ULL, 0xbfd1058bf9ae4800ULL, 0xbd26a8c4fd055a66ULL, \
  0x3ff4c00000000000ULL, 0xbfd0a324e2739000ULL, 0xbd0c6bee7ef4030eULL, \
  0x3ff4a00000000000ULL, 0xbfd0402594b4d000ULL, 0xbcf036b89ef42d7fULL, \
  0x3ff4a00000000000ULL, 0xbfd0402594b4d000ULL, 0xbcf036b89ef42d7fULL, \
  0x3ff4800000000000ULL, 0xbfcfb9186d5e4000ULL, 0x3d0d572aab993c87ULL, \
  0x3ff4600000000000ULL, 0xbfcef0adcbdc6000ULL, 0x3d2b26b79c86af24ULL, \
  0x3ff4400000000000ULL, 0xbfce27076e2af000ULL, 0xbd172f4f543fff10ULL, \
  0x3ff4200000000000ULL, 0xbfcd5c216b4fc000ULL, 0x3d21ba91bbca681bULL, \
  0x3ff4000000000000ULL, 0xbfcc8ff7c79aa000ULL, 0x3d27794f689f8434ULL, \
  0x3ff4000000000000ULL, 0xbfcc8ff7c79aa000ULL, 0x3d27794f689f8434ULL, \
  0x3ff3e00000000000ULL, 0xbfcbc286742d9000ULL, 0x3d194eb0318bb78fULL, \
  0x3ff3c00000000000ULL, 0xbfcaf3c94e80c000ULL, 0x3cba4e633fcd9066ULL, \
  0x3ff3a00000000000ULL, 0xbfca23bc1fe2b000ULL, 0xbd258c64dc46c1eaULL, \
  0x3ff3a00000000000ULL, 0xbfca23bc1fe2b000ULL, 0xbd258c64dc46c1eaULL, \
  0x3ff3800000000000ULL, 0xbfc9525a9cf45000ULL, 0xbd2ad1d904c1d4e3ULL, \
  0x3ff3600000000000ULL, 0xbfc87fa06520d000ULL, 0x3d2bbdbf7fdbfa09ULL, \
  0x3ff3400000000000ULL, 0xbfc7ab890210e000ULL, 0x3d2bdb9072534a58ULL, \
  0x3ff3400000000000ULL, 0xbfc7ab890210e000ULL, 0x3d2bdb9072534a58ULL, \
  0x3ff3200000000000ULL, 0xbfc6d60fe719d000ULL, 0xbd10e46aa3b2e266ULL, \
  0x3ff3000000000000ULL, 0xbfc5ff3070a79000ULL, 0xbd1e9e439f105039ULL, \
  0x3ff3000000000000ULL, 0xbfc5ff3070a79000ULL, 0xbd1e9e439f105039ULL, \
  0x3ff2e00000000000ULL, 0xbfc526e5e3a1b000ULL, 0xbd20de8b90075b8fULL, \
  0x3ff2c00000000000ULL, 0xbfc44d2b6ccb8000ULL, 0x3d170cc16135783cULL, \
  0x3ff2c00000000000ULL, 0xbfc44d2b6ccb8000ULL, 0x3d170cc16135783cULL, \
  0x3ff2a00000000000ULL, 0xbfc371fc201e9000ULL, 0x3cf178864d27543aULL, \
  0x3ff2800000000000ULL, 0xbfc29552f81ff000ULL, 0xbd248d301771c408ULL, \
  0x3ff2600000000000ULL, 0xbfc1b72ad52f6000ULL, 0xbd2e80a41811a396ULL, \
  0x3ff2600000000000ULL, 0xbfc1b72ad52f6000ULL, 0xbd2e80a41811a396ULL, \
  0x3ff2400000000000ULL, 0xbfc0d77e7cd09000ULL, 0x3d0a699688e85bf4ULL, \
  0x3ff2400000000000ULL, 0xbfc0d77e7cd09000ULL, 0x3d0a699688e85bf4ULL, \
  0x3ff2200000000000ULL, 0xbfbfec9131dbe000ULL, 0xbd2575545ca333f2ULL, \
  0x3ff2000000000000ULL, 0xbfbe27076e2b0000ULL, 0x3d2a342c2af0003cULL, \
  0x3ff2000000000000ULL, 0xbfbe27076e2b0000ULL, 0x3d2a342c2af0003cULL, \
  0x3ff1e00000000000ULL, 0xbfbc5e548f5bc000ULL, 0xbd1d0c57585fbe06ULL, \
  0x3ff1c00000000000ULL, 0xbfba926d3a4ae000ULL, 0x3d253935e85baac8ULL, \
  0x3ff1c00000000000ULL, 0xbfba926d3a4ae000ULL, 0x3d253935e85baac8ULL, \
  0x3ff1a00000000000ULL, 0xbfb8c345d631a000ULL, 0x3d137c294d2f5668ULL, \
  0x3ff1a00000000000ULL, 0xbfb8c345d631a000ULL, 0x3d137c294d2f5668ULL, \
  0x3ff1800000000000ULL, 0xbfb6f0d28ae56000ULL, 0xbd269737c93373daULL, \
  0x3ff1600000000000ULL, 0xbfb51b073f062000ULL, 0x3d1f025b61c65e57ULL, \
  0x3ff1600000000000ULL, 0xbfb51b073f062000ULL, 0x3d1f025b61c65e57ULL, \
  0x3ff1400000000000ULL, 0xbfb341d7961be000ULL, 0x3d2c5edaccf913dfULL, \
  0x3ff1400000000000ULL, 0xbfb341d7961be000ULL, 0x3d2c5edaccf913dfULL, \
  0x3ff1200000000000ULL, 0xbfb16536eea38000ULL, 0x3d147c5e768fa309ULL, \
  0x3ff1000000000000ULL, 0xbfaf0a30c0118000ULL, 0x3d2d599e83368e91ULL, \
  0x3ff1000000000000ULL, 0xbfaf0a30c0118000ULL, 0x3d2d599e83368e91ULL, \
  0x3ff0e00000000000ULL, 0xbfab42dd71198000ULL, 0x3d1c827ae5d6704cULL, \
  0x3ff0e00000000000ULL, 0xbfab42dd71198000ULL, 0x3d1c827ae5d6704cULL, \
  0x3ff0c00000000000ULL, 0xbfa77458f632c000ULL, 0xbd2cfc4634f2a1eeULL, \
  0x3ff0c00000000000ULL, 0xbfa77458f632c000ULL, 0xbd2cfc4634f2a1eeULL, \
  0x3ff0a00000000000ULL, 0xbfa39e87b9fec000ULL, 0x3cf502b7f526feaaULL, \
  0x3ff0a00000000000ULL, 0xbfa39e87b9fec000ULL, 0x3cf502b7f526feaaULL, \
  0x3ff0800000000000ULL, 0xbf9f829b0e780000ULL, 0xbd2980267c7e09e4ULL, \
  0x3ff0800000000000ULL, 0xbf9f829b0e780000ULL, 0xbd2980267c7e09e4ULL, \
  0x3ff0600000000000ULL, 0xbf97b91b07d58000ULL, 0xbd288d5493faa639ULL, \
  0x3ff0400000000000ULL, 0xbf8fc0a8b0fc0000ULL, 0xbcdf1e7cf6d3a69cULL, \
  0x3ff0400000000000ULL, 0xbf8fc0a8b0fc0000ULL, 0xbcdf1e7cf6d3a69cULL, \
  0x3ff0200000000000ULL, 0xbf7fe02a6b100000ULL, 0xbd19e23f0dda40e4ULL, \
  0x3ff0200000000000ULL, 0xbf7fe02a6b100000ULL, 0xbd19e23f0dda40e4ULL, \
  0x3ff0000000000000ULL, 0x0000000000000000ULL, 0x0000000000000000ULL, \
  0x3ff0000000000000ULL, 0x0000000000000000ULL, 0x0000000000000000ULL, \
  0x3fefc00000000000ULL, 0x3f80101575890000ULL, 0xbd10c76b999d2be8ULL, \
  0x3fef800000000000ULL, 0x3f90205658938000ULL, 0xbd23dc5b06e2f7d2ULL, \
  0x3fef400000000000ULL, 0x3f98492528c90000ULL, 0xbd2aa0ba325a0c34ULL, \
  0x3fef000000000000ULL, 0x3fa0415d89e74000ULL, 0x3d0111c05cf1d753ULL, \
  0x3feec00000000000ULL, 0x3fa466aed42e0000ULL, 0xbd2c167375bdfd28ULL, \
  0x3fee800000000000ULL, 0x3fa894aa149fc000ULL, 0xbd197995d05a267dULL, \
  0x3fee400000000000ULL, 0x3faccb73cdddc000ULL, 0xbd1a68f247d82807ULL, \
  0x3fee200000000000ULL, 0x3faeea31c006c000ULL, 0xbd0e113e4fc93b7bULL, \
  0x3fede00000000000ULL, 0x3fb1973bd1466000ULL, 0xbd25325d560d9e9bULL, \
  0x3feda00000000000ULL, 0x3fb3bdf5a7d1e000ULL, 0x3d2cc85ea5db4ed7ULL, \
  0x3fed600000000000ULL, 0x3fb5e95a4d97a000ULL, 0xbd2c69063c5d1d1eULL, \
  0x3fed400000000000ULL, 0x3fb700d30aeac000ULL, 0x3cec1e8da99ded32ULL, \
  0x3fed000000000000ULL, 0x3fb9335e5d594000ULL, 0x3d23115c3abd47daULL, \
  0x3fecc00000000000ULL, 0x3fbb6ac88dad6000ULL, 0xbd1390802bf768e5ULL, \
  0x3feca00000000000ULL, 0x3fbc885801bc4000ULL, 0x3d2646d1c65aacd3ULL, \
  0x3fec600000000000ULL, 0x3fbec739830a2000ULL, 0xbd2dc068afe645e0ULL, \
  0x3fec400000000000ULL, 0x3fbfe89139dbe000ULL, 0xbd2534d64fa10afdULL, \
  0x3fec000000000000ULL, 0x3fc1178e8227e000ULL, 0x3d21ef78ce2d07f2ULL, \
  0x3febe00000000000ULL, 0x3fc1aa2b7e23f000ULL, 0x3d2ca78e44389934ULL, \
  0x3feba00000000000ULL, 0x3fc2d1610c868000ULL, 0x3d039d6ccb81b4a1ULL, \
  0x3feb800000000000ULL, 0x3fc365fcb0159000ULL, 0x3cc62fa8234b7289ULL, \
  0x3feb400000000000ULL, 0x3fc4913d8333b000ULL, 0x3d25837954fdb678ULL, \
  0x3feb200000000000ULL, 0x3fc527e5e4a1b000ULL, 0x3d2633e8e5697dc7ULL, \
  0x3feae00000000000ULL, 0x3fc6574ebe8c1000ULL, 0x3d19cf8b2c3c2e78ULL, \
  0x3feac00000000000ULL, 0x3fc6f0128b757000ULL, 0xbd25118de59c21e1ULL, \
  0x3feaa00000000000ULL, 0x3fc7898d85445000ULL, 0xbd1c661070914305ULL, \
  0x3fea600000000000ULL, 0x3fc8beafeb390000ULL, 0xbd073d54aae92cd1ULL, \
  0x3fea400000000000ULL, 0x3fc95a5adcf70000ULL, 0x3d07f22858a0ff6fULL, \
  0x3fea000000000000ULL, 0x3fca93ed3c8ae000ULL, 0xbd28724350562169ULL, \
  0x3fe9e00000000000ULL, 0x3fcb31d8575bd000ULL, 0xbd0c358d4eace1aaULL, \
  0x3fe9c00000000000ULL, 0x3fcbd087383be000ULL, 0xbd2d4bc4595412b6ULL, \
  0x3fe9a00000000000ULL, 0x3fcc6ffbc6f01000ULL, 0xbcf1ec72c5962bd2ULL, \
  0x3fe9600000000000ULL, 0x3fcdb13db0d49000ULL, 0xbd2aff2af715b035ULL, \
  0x3fe9400000000000ULL, 0x3fce530effe71000ULL, 0x3cc212276041f430ULL, \
  0x3fe9200000000000ULL, 0x3fcef5ade4dd0000ULL, 0xbcca211565bb8e11ULL, \
  0x3fe9000000000000ULL, 0x3fcf991c6cb3b000ULL, 0x3d1bcbecca0cdf30ULL, \
  0x3fe8c00000000000ULL, 0x3fd07138604d5800ULL, 0x3cf89cdb16ed4e91ULL, \
  0x3fe8a00000000000ULL, 0x3fd0c42d67616000ULL, 0x3d27188b163ceae9ULL, \
  0x3fe8800000000000ULL, 0x3fd1178e8227e800ULL, 0xbd2c210e63a5f01cULL, \
  0x3fe8600000000000ULL, 0x3fd16b5ccbacf800ULL, 0x3d2b9acdf7a51681ULL, \
  0x3fe8400000000000ULL, 0x3fd1bf99635a6800ULL, 0x3d2ca6ed5147bdb7ULL, \
  0x3fe8200000000000ULL, 0x3fd214456d0eb800ULL, 0x3d0a87deba46baeaULL, \
  0x3fe7e00000000000ULL, 0x3fd2bef07cdc9000ULL, 0x3d2a9cfa4a5004f4ULL, \
  0x3fe7c00000000000ULL, 0x3fd314f1e1d36000ULL, 0xbd28e27ad3213cb8ULL, \
  0x3fe7a00000000000ULL, 0x3fd36b6776be1000ULL, 0x3d116ecdb0f177c8ULL, \
  0x3fe7800000000000ULL, 0x3fd3c25277333000ULL, 0x3d183b54b606bd5cULL, \
  0x3fe7600000000000ULL, 0x3fd419b423d5e800ULL, 0x3d08e436ec90e09dULL, \
  0x3fe7400000000000ULL, 0x3fd4718dc271c800ULL, 0xbd2f27ce0967d675ULL, \
  0x3fe7200000000000ULL, 0x3fd4c9e09e173000ULL, 0xbd2e20891b0ad8a4ULL, \
  0x3fe7000000000000ULL, 0x3fd522ae0738a000ULL, 0x3d2ebe708164c759ULL, \
  0x3fe6e00000000000ULL, 0x3fd57bf753c8d000ULL, 0x3d1fadedee5d40efULL, \
  0x3fe6c00000000000ULL, 0x3fd5d5bddf596000ULL, 0xbd0a0b2a08a465dcULL, \
}
#define ALZ_POW2_EXP_TAB { \
  0x0000000000000000ULL, 0x3ff0000000000000ULL, 0x3c9b3b4f1a88bf6eULL, 0x3feff63da9fb3335ULL, \
  0xbc7160139cd8dc5dULL, 0x3fefec9a3e778061ULL, 0xbc905e7a108766d1ULL, 0x3fefe315e86e7f85ULL, \
  0x3c8cd2523567f613ULL, 0x3fefd9b0d3158574ULL, 0xbc8bce8023f98efaULL, 0x3fefd06b29ddf6deULL, \
  0x3c60f74e61e6c861ULL, 0x3fefc74518759bc8ULL, 0x3c90a3e45b33d399ULL, 0x3fefbe3ecac6f383ULL, \
  0x3c979aa65d837b6dULL, 0x3fefb5586cf9890fULL, 0x3c8eb51a92fdeffcULL, 0x3fefac922b7247f7ULL, \
  0x3c3ebe3d702f9cd1ULL, 0x3fefa3ec32d3d1a2ULL, 0xbc6a033489906e0bULL, 0x3fef9b66affed31bULL, \
  0xbc9556522a2fbd0eULL, 0x3fef9301d0125b51ULL, 0xbc5080ef8c4eea55ULL, 0x3fef8abdc06c31ccULL, \
  0xbc91c923b9d5f416ULL, 0x3fef829aaea92de0ULL, 0x3c80d3e3e95c55afULL, 0x3fef7a98c8a58e51ULL, \
  0xbc801b15eaa59348ULL, 0x3fef72b83c7d517bULL, 0xbc8f1ff055de323dULL, 0x3fef6af9388c8deaULL, \
  0x3c8b898c3f1353bfULL, 0x3fef635beb6fcb75ULL, 0xbc96d99c7611eb26ULL, 0x3fef5be084045cd4ULL, \
  0x3c9aecf73e3a2f60ULL, 0x3fef54873168b9aaULL, 0xbc8fe782cb86389dULL, 0x3fef4d5022fcd91dULL, \
  0x3c8a6f4144a6c38dULL, 0x3fef463b88628cd6ULL, 0x3c807a05b0e4047dULL, 0x3fef3f49917ddc96ULL, \
  0x3c968efde3a8a894ULL, 0x3fef387a6e756238ULL, 0x3c875e18f274487dULL, 0x3fef31ce4fb2a63fULL, \
  0x3c80472b981fe7f2ULL, 0x3fef2b4565e27cddULL, 0xbc96b87b3f71085eULL, 0x3fef24dfe1f56381ULL, \
  0x3c82f7e16d09ab31ULL, 0x3fef1e9df51fdee1ULL, 0xbc3d219b1a6fbffaULL, 0x3fef187fd0dad990ULL, \
  0x3c8b3782720c0ab4ULL, 0x3fef1285a6e4030bULL, 0x3c6e149289cecb8fULL, 0x3fef0cafa93e2f56ULL, \
  0x3c834d754db0abb6ULL, 0x3fef06fe0a31b715ULL, 0x3c864201e2ac744cULL, 0x3fef0170fc4cd831ULL, \
  0x3c8fdd395dd3f84aULL, 0x3feefc08b26416ffULL, 0xbc86a3803b8e5b04ULL, 0x3feef6c55f929ff1ULL, \
  0xbc924aedcc4b5068ULL, 0x3feef1a7373aa9cbULL, 0xbc9907f81b512d8eULL, 0x3feeecae6d05d866ULL, \
  0xbc71d1e83e9436d2ULL, 0x3feee7db34e59ff7ULL, 0xbc991919b3ce1b15ULL, 0x3feee32dc313a8e5ULL, \
  0x3c859f48a72a4c6dULL, 0x3feedea64c123422ULL, 0xbc9312607a28698aULL, 0x3feeda4504ac801cULL, \
  0xbc58a78f4817895bULL, 0x3feed60a21f72e2aULL, 0xbc7c2c9b67499a1bULL, 0x3feed1f5d950a897ULL, \
  0x3c4363ed60c2ac11ULL, 0x3feece086061892dULL, 0x3c9666093b0664efULL, 0x3feeca41ed1d0057ULL, \
  0x3c6ecce1daa10379ULL, 0x3feec6a2b5c13cd0ULL, 0x3c93ff8e3f0f1230ULL, 0x3feec32af0d7d3deULL, \
  0x3c7690cebb7aafb0ULL, 0x3feebfdad5362a27ULL, 0x3c931dbdeb54e077ULL, 0x3feebcb299fddd0dULL, \
  0xbc8f94340071a38eULL, 0x3feeb9b2769d2ca7ULL, 0xbc87deccdc93a349ULL, 0x3feeb6daa2cf6642ULL, \
  0xbc78dec6bd0f385fULL, 0x3feeb42b569d4f82ULL, 0xbc861246ec7b5cf6ULL, 0x3feeb1a4ca5d920fULL, \
  0x3c93350518fdd78eULL, 0x3feeaf4736b527daULL, 0x3c7b98b72f8a9b05ULL, 0x3feead12d497c7fdULL, \
  0x3c9063e1e21c5409ULL, 0x3feeab07dd485429ULL, 0x3c34c7855019c6eaULL, 0x3feea9268a5946b7ULL, \
  0x3c9432e62b64c035ULL, 0x3feea76f15ad2148ULL, 0xbc8ce44a6199769fULL, 0x3feea5e1b976dc09ULL, \
  0xbc8c33c53bef4da8ULL, 0x3feea47eb03a5585ULL, 0xbc845378892be9aeULL, 0x3feea34634ccc320ULL, \
  0xbc93cedd78565858ULL, 0x3feea23882552225ULL, 0x3c5710aa807e1964ULL, 0x3feea155d44ca973ULL, \
  0xbc93b3efbf5e2228ULL, 0x3feea09e667f3bcdULL, 0xbc6a12ad8734b982ULL, 0x3feea012750bdabfULL, \
  0xbc6367efb86da9eeULL, 0x3fee9fb23c651a2fULL, 0xbc80dc3d54e08851ULL, 0x3fee9f7df9519484ULL, \
  0xbc781f647e5a3ecfULL, 0x3fee9f75e8ec5f74ULL, 0xbc86ee4ac08b7db0ULL, 0x3fee9f9a48a58174ULL, \
  0xbc8619321e55e68aULL, 0x3fee9feb564267c9ULL, 0x3c909ccb5e09d4d3ULL, 0x3feea0694fde5d3fULL, \
  0xbc7b32dcb94da51dULL, 0x3feea11473eb0187ULL, 0x3c94ecfd5467c06bULL, 0x3feea1ed0130c132ULL, \
  0x3c65ebe1abd66c55ULL, 0x3feea2f336cf4e62ULL, 0xbc88a1c52fb3cf42ULL, 0x3feea427543e1a12ULL, \
  0xbc9369b6f13b3734ULL, 0x3feea589994cce13ULL, 0xbc805e843a19ff1eULL, 0x3feea71a4623c7adULL, \
  0xbc94d450d872576eULL, 0x3feea8d99b4492edULL, 0x3c90ad675b0e8a00ULL, 0x3feeaac7d98a6699ULL, \
  0x3c8db72fc1f0eab4ULL, 0x3feeace5422aa0dbULL, 0xbc65b6609cc5e7ffULL, 0x3feeaf3216b5448cULL, \
  0x3c7bf68359f35f44ULL, 0x3feeb1ae99157736ULL, 0xbc93091fa71e3d83ULL, 0x3feeb45b0b91ffc6ULL, \
  0xbc5da9b88b6c1e29ULL, 0x3feeb737b0cdc5e5ULL, 0xbc6c23f97c90b959ULL, 0x3feeba44cbc8520fULL, \
  0xbc92434322f4f9aaULL, 0x3feebd829fde4e50ULL, 0xbc85ca6cd7668e4bULL, 0x3feec0f170ca07baULL, \
  0x3c71affc2b91ce27ULL, 0x3feec49182a3f090ULL, 0x3c6dd235e10a73bbULL, 0x3feec86319e32323ULL, \
  0xbc87c50422622263ULL, 0x3feecc667b5de565ULL, 0x3c8b1c86e3e231d5ULL, 0x3feed09bec4a2d33ULL, \
  0xbc91bbd1d3bcbb15ULL, 0x3feed503b23e255dULL, 0x3c90cc319cee31d2ULL, 0x3feed99e1330b358ULL, \
  0x3c8469846e735ab3ULL, 0x3feede6b5579fdbfULL, 0xbc82dfcd978e9db4ULL, 0x3feee36bbfd3f37aULL, \
  0x3c8c1a7792cb3387ULL, 0x3feee89f995ad3adULL, 0xbc907b8f4ad1d9faULL, 0x3feeee07298db666ULL, \
  0xbc55c3d956dcaebaULL, 0x3feef3a2b84f15fbULL, 0xbc90a40e3da6f640ULL, 0x3feef9728de5593aULL, \
  0xbc68d6f438ad9334ULL, 0x3feeff76f2fb5e47ULL, 0xbc91eee26b588a35ULL, 0x3fef05b030a1064aULL, \
  0x3c74ffd70a5fddcdULL, 0x3fef0c1e904bc1d2ULL, 0xbc91bdfbfa9298acULL, 0x3fef12c25bd71e09ULL, \
  0x3c736eae30af0cb3ULL, 0x3fef199bdd85529cULL, 0x3c8ee3325c9ffd94ULL, 0x3fef20ab5fffd07aULL, \
  0x3c84e08fd10959acULL, 0x3fef27f12e57d14bULL, 0x3c63cdaf384e1a67ULL, 0x3fef2f6d9406e7b5ULL, \
  0x3c676b2c6c921968ULL, 0x3fef3720dcef9069ULL, 0xbc808a1883ccb5d2ULL, 0x3fef3f0b555dc3faULL, \
  0xbc8fad5d3ffffa6fULL, 0x3fef472d4a07897cULL, 0xbc900dae3875a949ULL, 0x3fef4f87080d89f2ULL, \
  0x3c74a385a63d07a7ULL, 0x3fef5818dcfba487ULL, 0xbc82919e2040220fULL, 0x3fef60e316c98398ULL, \
  0x3c8e5a50d5c192acULL, 0x3fef69e603db3285ULL, 0x3c843a59ac016b4bULL, 0x3fef7321f301b460ULL, \
  0xbc82d52107b43e1fULL, 0x3fef7c97337b9b5fULL, 0xbc892ab93b470dc9ULL, 0x3fef864614f5a129ULL, \
  0x3c74b604603a88d3ULL, 0x3fef902ee78b3ff6ULL, 0x3c83c5ec519d7271ULL, 0x3fef9a51fbc74c83ULL, \
  0xbc8ff7128fd391f0ULL, 0x3fefa4afa2a490daULL, 0xbc8dae98e223747dULL, 0x3fefaf482d8e67f1ULL, \
  0x3c8ec3bc41aa2008ULL, 0x3fefba1bee615a27ULL, 0x3c842b94c3a9eb32ULL, 0x3fefc52b376bba97ULL, \
  0x3c8a64a931d185eeULL, 0x3fefd0765b6e4540ULL, 0xbc8e37bae43be3edULL, 0x3fefdbfdad9cbe14ULL, \
  0x3c77893b4d91cd9dULL, 0x3fefe7c1819e90d8ULL, 0x3c5305c14160cc89ULL, 0x3feff3c22b8f71f1ULL, \
}

#ifdef __CUDACC__
__device__ const uint64_t alz_pow2_log_tab_dev[3 * 128] = ALZ_POW2_LOG_TAB;
__device__ const uint64_t alz_pow2_exp_tab_dev[256] = ALZ_POW2_EXP_TAB;
#endif
static const uint64_t alz_pow2_log_tab_host[3 * 128] = ALZ_POW2_LOG_TAB;
static const uint64_t alz_pow2_exp_tab_host[256] = ALZ_POW2_EXP_TAB;

ALZ_POW2_HD uint64_t alz_pow2_log_word(int i) {
#ifdef __CUDA_ARCH__
  return __ldg((const unsigned long long*)&alz_pow2_log_tab_dev[i]);
#else
  return alz_pow2_log_tab_host[i];
#endif
}

ALZ_POW2_HD uint64_t alz_pow2_exp_word(int i) {
#ifdef __CUDA_ARCH__
  return __ldg((const unsigned long long*)&alz_pow2_exp_tab_dev[i]);
#else
  return alz_pow2_exp_tab_host[i];
#endif
}

ALZ_POW2_HD double alz_pow2_asdouble(uint64_t u) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)u);
#else
  double d;
  memcpy(&d, &u, 8);
  return d;
#endif
}

ALZ_POW2_HD uint64_t alz_pow2_asuint(double d) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(d);
#else
  uint64_t u;
  memcpy(&u, &d, 8);
  return u;
#endif
}

// One IEEE operation each, rounded to nearest.
#ifdef __CUDA_ARCH__
#define ALZ_P2_ADD(a, b) __dadd_rn((a), (b))
#define ALZ_P2_SUB(a, b) __dsub_rn((a), (b))
#define ALZ_P2_MUL(a, b) __dmul_rn((a), (b))
#define ALZ_P2_FMA(a, b, c) __fma_rn((a), (b), (c))
#else
#define ALZ_P2_ADD(a, b) ((a) + (b))
#define ALZ_P2_SUB(a, b) ((a) - (b))
#define ALZ_P2_MUL(a, b) ((a) * (b))
#define ALZ_P2_FMA(a, b, c) fma((a), (b), (c))
#endif

// glibc's pow(x, 2.0) for a finite x > 0.
ALZ_POW2_HD double alz_pow2_glibc(double x) {
  uint64_t ix = alz_pow2_asuint(x);
  if ((ix >> 52) == 0) {                          // subnormal: normalize so that the exponent becomes negative
    ix = alz_pow2_asuint(ALZ_P2_MUL(x, 0x1p52)) & 0x7fffffffffffffffULL;
    ix -= 52ULL << 52;
  }
  // log(x) = k ln2 + log(c) + log1p(z / c - 1) in double-double (hi, tail)
  const uint64_t tmp = ix - 0x3fe6955500000000ULL;
  const int i = (int)((tmp >> 45) & 127);
  const int64_t k = (int64_t)tmp >> 52;
  const double z = alz_pow2_asdouble(ix - (tmp & (0xfffULL << 52)));
  const double kd = (double)k;
  const double invc = alz_pow2_asdouble(alz_pow2_log_word(3 * i));
  const double logc = alz_pow2_asdouble(alz_pow2_log_word(3 * i + 1));
  const double logctail = alz_pow2_asdouble(alz_pow2_log_word(3 * i + 2));
  const double r = ALZ_P2_FMA(z, invc, -1.0);
  const double t1 = ALZ_P2_FMA(kd, 0x1.62e42fefa38p-1, logc);            // k Ln2hi + logc
  const double lo1 = ALZ_P2_FMA(kd, 0x1.ef35793c7673p-45, logctail);      // k Ln2lo + logctail
  const double ar = ALZ_P2_MUL(r, -0x1p-1);
  const double p1 = ALZ_P2_FMA(r, 0x1.0000000000006p-1, -0x1.555555555556p-1);
  const double p3 = ALZ_P2_FMA(r, -0x1.555555529a47ap-1, 0x1.999999959554ep-1);
  const double t2 = ALZ_P2_ADD(r, t1);
  const double lo2 = ALZ_P2_ADD(ALZ_P2_SUB(t1, t2), r);
  const double ar2 = ALZ_P2_MUL(r, ar);
  const double ar3 = ALZ_P2_MUL(r, ar2);
  const double lo3 = ALZ_P2_FMA(ar, r, -ar2);
  const double hi = ALZ_P2_ADD(t2, ar2);
  const double p5 = ALZ_P2_FMA(r, 0x1.0002b8b263fc3p+0, -0x1.2495b9b4845e9p+0);
  const double lo4 = ALZ_P2_ADD(ALZ_P2_SUB(t2, hi), ar2);
  const double q = ALZ_P2_FMA(p5, ar2, p3);
  const double s = ALZ_P2_FMA(ar2, q, p1);
  double lo = ALZ_P2_ADD(ALZ_P2_ADD(ALZ_P2_ADD(lo1, lo2), lo3), lo4);
  lo = ALZ_P2_FMA(ar3, s, lo);
  const double lhi = ALZ_P2_ADD(hi, lo);
  const double ltail = ALZ_P2_ADD(ALZ_P2_SUB(hi, lhi), lo);
  // times y = 2: ehi + elo
  const double ehi = ALZ_P2_MUL(2.0, lhi);
  const double elo = ALZ_P2_FMA(2.0, ltail, ALZ_P2_FMA(lhi, 2.0, -ehi));
  // exp(ehi + elo) = 2^(ki / 128) exp(r)
  uint32_t abstop = (uint32_t)(alz_pow2_asuint(ehi) >> 52) & 0x7ff;
  if (abstop - 0x3c9u >= 0x3fu) {
    if ((int32_t)(abstop - 0x3c9u) < 0) return ALZ_P2_ADD(ehi, 1.0);    // |ehi| < 2^-54
    if (abstop >= 0x409u) return (alz_pow2_asuint(ehi) >> 63) ? 0.0 : INFINITY;   // |ehi| >= 1024
    abstop = 0;                                   // the final scaling is done by the special case below
  }
  double kx = ALZ_P2_FMA(ehi, 0x1.71547652b82fep+7, 0x1.8p52);           // InvLn2N ehi + Shift
  const uint64_t ki = alz_pow2_asuint(kx);
  kx = ALZ_P2_SUB(kx, 0x1.8p52);
  double er = ALZ_P2_FMA(kx, -0x1.62e42fefa0000p-8, ehi);
  er = ALZ_P2_FMA(kx, -0x1.cf79abc9e3b3ap-47, er);
  er = ALZ_P2_ADD(elo, er);
  const int idx = (int)(2 * (ki & 127));
  uint64_t sbits = alz_pow2_exp_word(idx + 1) + (ki << 45);
  const double p23 = ALZ_P2_FMA(er, 0x1.555555555543cp-3, 0x1.ffffffffffdbdp-2);
  const double tr = ALZ_P2_ADD(er, alz_pow2_asdouble(alz_pow2_exp_word(idx)));
  const double r2 = ALZ_P2_MUL(er, er);
  const double p45 = ALZ_P2_FMA(er, 0x1.1111167a4d017p-7, 0x1.55555cf172b91p-5);
  double t = ALZ_P2_FMA(p23, r2, tr);
  t = ALZ_P2_FMA(p45, ALZ_P2_MUL(r2, r2), t);
  if (abstop != 0) {
    const double scale = alz_pow2_asdouble(sbits);
    return ALZ_P2_FMA(t, scale, scale);
  }
  if ((ki & 0x80000000ULL) == 0) {                // k > 0: the scale's exponent may have overflowed
    sbits -= 1009ULL << 52;
    const double scale = alz_pow2_asdouble(sbits);
    return ALZ_P2_MUL(ALZ_P2_FMA(scale, t, scale), 0x1p1009);
  }
  sbits += 1022ULL << 52;                         // k < 0: round once before scaling into the subnormal range
  const double scale = alz_pow2_asdouble(sbits);
  const double st = ALZ_P2_MUL(t, scale);
  double y = ALZ_P2_ADD(scale, st);
  if (fabs(y) < 1.0) {
    const double one = y < 0.0 ? -1.0 : 1.0;
    double l = ALZ_P2_ADD(ALZ_P2_SUB(scale, y), st);
    const double h = ALZ_P2_ADD(y, one);
    l = ALZ_P2_ADD(ALZ_P2_ADD(ALZ_P2_SUB(one, h), y), l);
    y = ALZ_P2_SUB(ALZ_P2_ADD(l, h), one);
    if (y == 0.0) y = alz_pow2_asdouble(sbits & 0x8000000000000000ULL);
  }
  return ALZ_P2_MUL(y, 0x1p-1022);
}

// CPython 3.12's `k ** 2` for a float k; *overflow is set to 1 where it raises OverflowError (a finite k whose square
// is infinite), and the result is then +inf.
ALZ_POW2_HD double alz_py_pow2(double k, int* overflow) {
  *overflow = 0;
  if (k != k) return k;                           // nan ** 2 is the nan
  double a = fabs(k);
  if (a == INFINITY) return INFINITY;
  if (a == 0.0) return 0.0;
  if (a == 1.0) return 1.0;
  const double p = alz_pow2_glibc(a);
  if (p == INFINITY) *overflow = 1;
  return p;
}
